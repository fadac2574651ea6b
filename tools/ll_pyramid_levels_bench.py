"""local_laplacian at every pyramid depth: what halide_b200_local_laplacian_pyramid_levels costs per call as J moves, on
device-resident uint16 RGB frames (levels 8, alpha 1/7, beta 1).

    python tools/ll_pyramid_levels_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--J 1,2,3,5,8,11,14,20] [--sizes 4k,16k]

Frames: 3840 x 2160 x 3 and 16384 x 16384 x 3 (smooth content + noise, seeded).  Arms per frame: one per J, each followed
in every round by `local_laplacian` itself on the same frame, so every arm is compared with the fixed-8 filter timed right
next to it.  Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window,
`rounds` times; the median round is reported.  Per J the script also records the per-kernel times of one profiled call
(the library's profile mode) and, for J = 1, the achieved bandwidth of the tone kernel (12 B/px: three uint16 samples
read, three written) against the H100 SXM data sheet's 3.35 TB/s.  The J = 8 output must equal local_laplacian's byte for
byte.  The GPU's name, power limit and top SM clock are read in the same run.  Writes OUT_DIR/ll_pyramid_levels_bench.json
and prints one line per (frame, J)."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters

SIZES = {"4k": (3840, 2160), "16k": (16384, 16384)}
LEVELS, ALPHA, BETA = 8, 1.0 / 7.0, 1.0
HBM_BYTES_PER_S = 3.35e12


def main():
    ap = timing.common_args()
    ap.add_argument("--J", default="1,2,3,5,8,11,14,20")
    ap.add_argument("--sizes", default="4k,16k")
    args = ap.parse_args()
    js = [int(v) for v in args.J.split(",")]
    timing.setup("ll_pyramid_levels_bench")

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "levels": LEVELS, "alpha": ALPHA, "beta": BETA, "window_ms": args.window_ms,
              "rounds": args.rounds, "frames": []}
    for size in args.sizes.split(","):
        W, H = SIZES[size]
        gen = torch.Generator(device="cuda")
        gen.manual_seed(W)
        yy = torch.linspace(0, 1, H, device="cuda").view(H, 1)
        xx = torch.linspace(0, 1, W, device="cuda").view(1, W)
        base = torch.stack([0.5 + 0.4 * torch.sin(6.0 * xx + c) * torch.cos(5.0 * yy - c) for c in range(3)])
        noise = 0.03 * torch.rand((3, H, W), device="cuda", generator=gen)
        x = ((base + noise).clamp(0, 1) * 65535).to(torch.int32).to(torch.int16).view(torch.uint16)  # (int32 -> int16 wraps)
        del base, noise
        bx = HalideBuffer.from_torch(x)
        y_ref = torch.zeros_like(x)
        b_ref = HalideBuffer.from_torch(y_ref)
        y = torch.zeros_like(x)
        b_y = HalideBuffer.from_torch(y)
        plain = lambda: filters.local_laplacian(bx, LEVELS, ALPHA, BETA, b_ref)  # noqa: E731
        frame = {"size": size, "w": W, "h": H, "J": []}
        for J in js:
            arm = lambda J=J: filters.local_laplacian_pyramid_levels(bx, J, LEVELS, ALPHA, BETA, b_y)  # noqa: E731
            arms = {"J": arm, "ll": plain}
            timing.warm_up(arms)
            eq8 = None
            if J == 8:
                eq8 = bool(timing.same(y, y_ref))
                assert eq8, "J = 8 differs from local_laplacian"
            iters, ms = timing.measure(arms, args.window_ms, args.rounds)
            if J == 8:
                assert timing.same(y, y_ref), "J = 8 differs from local_laplacian after timing"
            prof = {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(arm).items())}
            entry = {"J": J, "iters": iters["J"], "ms_per_call": ms["J"], "median_ms": statistics.median(ms["J"]),
                     "local_laplacian_ms_per_call": ms["ll"], "local_laplacian_median_ms": statistics.median(ms["ll"]),
                     "equals_local_laplacian": eq8, "profile_ms": prof}
            if "ll_tone" in prof:
                t = prof["ll_tone"]["ms"] / prof["ll_tone"]["launches"] * 1e-3
                entry["tone_bytes"] = 12 * W * H
                entry["tone_tb_per_s"] = 12 * W * H / t / 1e12
                entry["tone_share_of_3_35_tb_per_s"] = 12 * W * H / t / HBM_BYTES_PER_S
            frame["J"].append(entry)
            extra = f", tone {entry['tone_tb_per_s']:.2f} TB/s" if "tone_tb_per_s" in entry else ""
            print(f"{size} J {J}: {entry['median_ms']:.3f} ms (local_laplacian {entry['local_laplacian_median_ms']:.3f} ms){extra}; " +
                  ", ".join(f"{n} {v['launches']}x {v['ms']:.3f}" for n, v in prof.items()), flush=True)
        result["frames"].append(frame)
        del x, y, y_ref, bx, b_y, b_ref
        torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "ll_pyramid_levels_bench.json", result)


if __name__ == "__main__":
    main()
