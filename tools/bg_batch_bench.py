"""Batch bilateral_grid on one GPU: what a clip costs through the batch entry points next to one call per frame.  Two arms
on the same device-resident frames:

  batch    halide_b200_bilateral_grid_batch / _u8_batch / _s_sigma_batch on the (N, H, W) clip
  singles  bilateral_grid / halide_b200_bilateral_grid_u8 / halide_b200_bilateral_grid_s_sigma on each of its N frames

for three cases (float at s_sigma 8, uint8 at s_sigma 8, float at s_sigma 32; r_sigma 0.1) at 640 x 480, 1280 x 720,
1920 x 1080 and 3840 x 2160 with N = 8, and 7680 x 4320 with N = 4.

    python tools/bg_batch_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--sizes 480p,720p,...] [--cases f32_s8,...]
    python tools/bg_batch_bench.py OUT_DIR --compare-lib OTHER.so [--runs 3]

Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window, the arms
alternating, `rounds` times each; the median round is reported with the spread of the rounds.  The two arms' outputs are
compared bit for bit in every case.  Writes OUT_DIR/bg_batch_bench.json and prints one line per case.

--compare-lib times bilateral_grid on one 7680 x 4320 frame with another build of the library (e.g. the parent commit's)
and with this tree's, in alternating processes, `runs` of each, and checks that both give the same bytes; it writes
OUT_DIR/bg_batch_bench_compare.json.  The GPU's name, power limit and top SM clock are read in the same run."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import torch

import timing
from halide_b200 import HalideBuffer, bilateral_grid_video, filters

SIZES = {"480p": (480, 640, 8), "720p": (720, 1280, 8), "1080p": (1080, 1920, 8), "4k": (2160, 3840, 8),
         "8k": (4320, 7680, 4)}
# name: (element type, s_sigma)
CASES = {"f32_s8": (torch.float32, 8), "u8_s8": (torch.uint8, 8), "f32_s32": (torch.float32, 32)}
R_SIGMA = 0.1


def make_clip(dtype, n, h, w, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    if dtype == torch.uint8:
        return torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=gen)
    return torch.rand((n, h, w), dtype=torch.float32, device="cuda", generator=gen)


def calls(dtype, s):
    """(batch call, one-frame call), each taking (input buffer, output buffer)."""
    if dtype == torch.uint8:
        return (lambda i, o: bilateral_grid_video.bilateral_grid_u8_batch(i, R_SIGMA, o),
                lambda i, o: filters.bilateral_grid_u8(i, R_SIGMA, o))
    if s == 8:
        return (lambda i, o: bilateral_grid_video.bilateral_grid_batch(i, R_SIGMA, o),
                lambda i, o: filters.bilateral_grid(i, R_SIGMA, o))
    return (lambda i, o: bilateral_grid_video.bilateral_grid_s_sigma_batch(i, s, R_SIGMA, o),
            lambda i, o: filters.bilateral_grid_s_sigma(i, s, R_SIGMA, o))


def batch_vs_singles(args):
    timing.setup("bg_batch_bench")
    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "window_ms": args.window_ms, "rounds": args.rounds, "r_sigma": R_SIGMA, "cases": []}
    for size in args.sizes.split(","):
        h, w, n = SIZES[size]
        for case in args.cases.split(","):
            dtype, s = CASES[case]
            x = make_clip(dtype, n, h, w, h * 100003 + w + s)
            yb, ys = torch.zeros_like(x), torch.zeros_like(x)
            bi, bo = HalideBuffer.from_torch(x), HalideBuffer.from_torch(yb)
            fi = [HalideBuffer.from_torch(x[k]) for k in range(n)]
            fo = [HalideBuffer.from_torch(ys[k]) for k in range(n)]
            batch, one = calls(dtype, s)

            def arm_batch():
                batch(bi, bo)

            def arm_singles():
                for k in range(n):
                    one(fi[k], fo[k])

            arms = {"batch": arm_batch, "singles": arm_singles}
            timing.warm_up(arms)
            assert timing.same(yb, ys), f"batch and single calls differ at {size} {case}"
            iters, ms = timing.measure(arms, args.window_ms, args.rounds)
            med = {k: statistics.median(v) for k, v in ms.items()}
            ratio = med["batch"] / med["singles"]
            # the spread: the ratio's range over the rounds (each round's batch against each round's singles)
            lo = min(ms["batch"]) / max(ms["singles"])
            hi = max(ms["batch"]) / min(ms["singles"])
            launches = {k: c for k, (c, _) in timing.profile(arm_batch).items()}
            entry = {"size": size, "h": h, "w": w, "n": n, "case": case, "s_sigma": s, "iters": iters, "ms_per_clip": ms,
                     "median_ms": med, "batch_over_singles": ratio, "ratio_range": [lo, hi], "outputs_equal": True,
                     "batch_launches": launches}
            result["cases"].append(entry)
            print(f"{size} N={n} {case}: batch {med['batch']:.3f} ms, {n} singles {med['singles']:.3f} ms, "
                  f"batch/singles {ratio:.3f} (rounds {lo:.3f}-{hi:.3f}); batch launches {launches}; outputs equal",
                  flush=True)
            del x, yb, ys, bi, bo, fi, fo
            torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "bg_batch_bench.json", result)


def one_8k_frame(args):
    """(child process) bilateral_grid on one 7680 x 4320 float frame with the library at args.lib: one JSON line."""
    import halide_b200.lib as hlib
    if args.lib:
        hlib.LIB_PATH = os.path.abspath(args.lib)
    timing.setup("bg_batch_bench")
    x = make_clip(torch.float32, 1, 4320, 7680, 8)[0]
    y = torch.zeros_like(x)
    bi, bo = HalideBuffer.from_torch(x), HalideBuffer.from_torch(y)
    arms = {"bilateral_grid": lambda: filters.bilateral_grid(bi, R_SIGMA, bo)}
    timing.warm_up(arms)
    _, ms = timing.measure(arms, args.window_ms, args.rounds)
    digest = hashlib.sha256(y.cpu().numpy().tobytes()).hexdigest()
    print(json.dumps({"lib": hlib.LIB_PATH, "median_ms": statistics.median(ms["bilateral_grid"]),
                      "ms": ms["bilateral_grid"], "sha256": digest}), flush=True)


def compare_libs(args):
    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    libs = {"other": os.path.abspath(args.compare_lib), "this": ""}
    runs = {k: [] for k in libs}
    for i in range(args.runs):
        for name, path in libs.items():
            cmd = [sys.executable, os.path.abspath(__file__), args.out_dir, "--one-8k-frame", "--window-ms",
                   str(args.window_ms), "--rounds", str(args.rounds)] + (["--lib", path] if path else [])
            out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
            r = json.loads(out.strip().splitlines()[-1])
            runs[name].append(r)
            print(f"run {i} {name}: {r['median_ms']:.4f} ms", flush=True)
    digests = {r["sha256"] for rs in runs.values() for r in rs}
    assert len(digests) == 1, "the two libraries give different bytes"
    med = {k: statistics.median(r["median_ms"] for r in rs) for k, rs in runs.items()}
    spread = {k: [min(r["median_ms"] for r in rs), max(r["median_ms"] for r in rs)] for k, rs in runs.items()}
    print(f"bilateral_grid 7680x4320: other {med['other']:.4f} ms (runs {spread['other'][0]:.4f}-{spread['other'][1]:.4f}), "
          f"this {med['this']:.4f} ms (runs {spread['this'][0]:.4f}-{spread['this'][1]:.4f}), this/other "
          f"{med['this'] / med['other']:.3f}; outputs equal", flush=True)
    timing.write_json(args.out_dir, "bg_batch_bench_compare.json",
                      {"gpu": info, "runs": runs, "median_ms": med, "spread_ms": spread, "outputs_equal": True})


def main():
    ap = timing.common_args()
    ap.add_argument("--sizes", default=",".join(SIZES))
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--compare-lib", default=None)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--one-8k-frame", action="store_true", help=argparse.SUPPRESS)  # (the child processes of --compare-lib)
    ap.add_argument("--lib", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one_8k_frame:
        one_8k_frame(args)
    elif args.compare_lib:
        compare_libs(args)
    else:
        batch_vs_singles(args)


if __name__ == "__main__":
    main()
