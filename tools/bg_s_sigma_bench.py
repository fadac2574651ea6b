"""bilateral_grid at every cell size: what halide_b200_bilateral_grid_s_sigma costs per call as s_sigma moves, on one
7680 x 4320 float32 noise frame (BASELINE.json config 3) with r_sigma = 0.1, device-resident.

    python tools/bg_s_sigma_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--s 1,2,4,8,16,32,64,128]

Arms: one per s_sigma, plus `bilateral_grid` itself (the fixed-8 entry point) on the same frame.  Every arm is warmed up,
then timed with CUDA events on one stream over enough calls to fill the window, the arms alternating, `rounds` times
each; the median round is reported.  For each s_sigma the script also records the per-kernel times of one profiled call,
the algorithmic bytes (4 B read + 4 B written per pixel) and the bytes of one grid array (stored cells x planes x 2
channels x 4 B; the histogram writes one, bg_blur_xy reads it and writes the second, the slice reads that).  The s_sigma = 8
output must equal bilateral_grid's byte for byte.  The GPU's name, power limit and top SM clock are read in the same run.
Writes OUT_DIR/bg_s_sigma_bench.json and prints one line per s_sigma."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters

W, H, R_SIGMA = 7680, 4320, 0.1


def grid_shape(s, w=W, h=H, ox=0, oy=0, r_sigma=R_SIGMA):
    """(stored cell columns, cell rows, planes) of one grid array, as bilateral_grid.cu lays it out."""
    import numpy as np
    inv_r = np.float32(1.0) / np.float32(r_sigma)
    zmax = int(np.float32(np.float32(1.0) * inv_r) + np.float32(0.5))
    gw = (ox + w - 1) // s + 1 + 2 - (ox // s - 2) + 1
    gh = (oy + h - 1) // s + 1 + 2 - (oy // s - 2) + 1
    return gw, gh, zmax + 2


def main():
    ap = timing.common_args()
    ap.add_argument("--s", default="1,2,4,8,16,32,64,128")
    args = ap.parse_args()
    s_values = [int(v) for v in args.s.split(",")]
    timing.setup("bg_s_sigma_bench")

    def profile(fn):
        return {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(fn).items())}

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7680)
    x = torch.rand((H, W), dtype=torch.float32, device="cuda", generator=gen)
    bx = HalideBuffer.from_torch(x)
    outs = {s: torch.zeros_like(x) for s in s_values}
    bouts = {s: HalideBuffer.from_torch(o) for s, o in outs.items()}
    y_ref = torch.zeros_like(x)
    b_ref = HalideBuffer.from_torch(y_ref)

    arms = {}
    for s in s_values:
        arms[f"s{s}"] = (lambda s=s: filters.bilateral_grid_s_sigma(bx, s, R_SIGMA, bouts[s]))
    arms["bilateral_grid"] = lambda: filters.bilateral_grid(bx, R_SIGMA, b_ref)
    timing.warm_up(arms)
    same8 = None
    if 8 in outs:
        same8 = bool(torch.equal(outs[8].view(torch.int32), y_ref.view(torch.int32)))
        assert same8, "s_sigma = 8 differs from bilateral_grid"
    iters, ms = timing.measure(arms, args.window_ms, args.rounds)
    med = {k: statistics.median(v) for k, v in ms.items()}
    if 8 in outs:
        assert torch.equal(outs[8].view(torch.int32), y_ref.view(torch.int32)), "s_sigma = 8 differs after timing"

    result = {"gpu": info, "w": W, "h": H, "r_sigma": R_SIGMA, "window_ms": args.window_ms, "rounds": args.rounds,
              "bilateral_grid": {"iters": iters["bilateral_grid"], "ms_per_call": ms["bilateral_grid"],
                                 "median_ms": med["bilateral_grid"], "profile_ms": profile(arms["bilateral_grid"])},
              "s8_equals_bilateral_grid": same8, "s_sigma": []}
    print(f"bilateral_grid: {med['bilateral_grid']:.3f} ms", flush=True)
    for s in s_values:
        k = f"s{s}"
        gw, gh, nz = grid_shape(s)
        grid_bytes = gw * gh * nz * 2 * 4
        prof = profile(arms[k])
        entry = {"s_sigma": s, "iters": iters[k], "ms_per_call": ms[k], "median_ms": med[k],
                 "algorithmic_bytes": 8 * W * H, "grid_cells": [gw, gh, nz], "grid_bytes": grid_bytes,
                 "profile_ms": prof}
        result["s_sigma"].append(entry)
        print(f"s_sigma {s}: {med[k]:.3f} ms (x{med[k] / med.get('s8', med['bilateral_grid']):.2f} of s_sigma 8), "
              f"grid {grid_bytes / 1e6:.1f} MB; " + ", ".join(f"{n} {v['ms']:.3f}" for n, v in prof.items()), flush=True)
    timing.write_json(args.out_dir, "bg_s_sigma_bench.json", result)


if __name__ == "__main__":
    main()
