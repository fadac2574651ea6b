"""Batch vs serial local_laplacian on one GPU: one halide_b200_local_laplacian_batch call of N frames against N
single-frame local_laplacian calls on the same device-resident frames, for N = 1, 2, 4, 8 at 1920x1080x3 and
3840x2160x3 (levels 8, alpha 1/7, beta 1).

    python tools/ll_batch_bench.py OUT_DIR [--window-ms 300] [--rounds 3]

Every shape is warmed up first; each arm is then timed with CUDA events on one stream over enough calls to fill the
window, batch and serial alternating, `rounds` times each.  The two arms' outputs are compared bit for bit at every timed
size.  Writes OUT_DIR/ll_batch_bench.json (Mpx/s of both arms per round, and the per-kernel profile of one batch call)
and prints one line per shape.  The GPU's name, power limit and top SM clock are read in the same run."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters

SIZES = [(1920, 1080), (3840, 2160)]
FRAMES = [1, 2, 4, 8]
LEVELS, ALPHA, BETA = 8, 1.0 / 7.0, 1.0


def main():
    args = timing.common_args().parse_args()
    timing.setup("ll_batch_bench")

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "levels": LEVELS, "alpha": ALPHA, "beta": BETA, "window_ms": args.window_ms,
              "rounds": args.rounds, "shapes": []}
    gen = torch.Generator(device="cuda")
    for (w, h) in SIZES:
        for n in FRAMES:
            gen.manual_seed(1000 * n + w)
            x = torch.randint(-32768, 32768, (n, 3, h, w), dtype=torch.int16, device="cuda", generator=gen).view(torch.uint16)
            out_b, out_s = torch.zeros_like(x), torch.zeros_like(x)
            bi, bo = HalideBuffer.from_torch(x), HalideBuffer.from_torch(out_b)
            si = [HalideBuffer.from_torch(x[k]) for k in range(n)]
            so = [HalideBuffer.from_torch(out_s[k]) for k in range(n)]

            def batch():
                filters.local_laplacian_batch(bi, LEVELS, ALPHA, BETA, bo)

            def serial():
                for k in range(n):
                    filters.local_laplacian(si[k], LEVELS, ALPHA, BETA, so[k])

            arms = {"batch": batch, "serial": serial}
            timing.warm_up(arms)
            assert torch.equal(out_b, out_s), f"batch and serial outputs differ at {w}x{h} N={n}"
            iters, ms = timing.measure(arms, args.window_ms, args.rounds)
            assert torch.equal(out_b, out_s), f"batch and serial outputs differ at {w}x{h} N={n} after timing"
            prof = timing.profile(batch)
            mpx = n * w * h / 1e6
            entry = {"w": w, "h": h, "n": n, "iters": iters,
                     "ms_per_call": ms, "mpx_s": {k: [mpx / (t / 1e3) for t in v] for k, v in ms.items()},
                     "median_mpx_s": {k: mpx / (statistics.median(v) / 1e3) for k, v in ms.items()},
                     "ms_per_frame_median": {k: statistics.median(v) / n for k, v in ms.items()},
                     "outputs_identical": True,
                     "batch_profile_ms": {k: {"launches": c, "ms": t} for k, (c, t) in sorted(prof.items())}}
            result["shapes"].append(entry)
            print(f"{w}x{h} N={n}: batch {entry['median_mpx_s']['batch']:.0f} Mpx/s "
                  f"({min(ms['batch']):.3f}-{max(ms['batch']):.3f} ms/call), serial {entry['median_mpx_s']['serial']:.0f} Mpx/s "
                  f"({min(ms['serial']):.3f}-{max(ms['serial']):.3f} ms/call); profile "
                  + ", ".join(f"{k} {t:.3f}" for k, (c, t) in sorted(prof.items())), flush=True)
            del x, out_b, out_s, bi, bo, si, so
    timing.write_json(args.out_dir, "ll_batch_bench.json", result)


if __name__ == "__main__":
    main()
