"""Batch halide_blur and stencil_chain on one GPU: what a clip costs through the batch entry points next to one call per
frame.  Two arms on the same device-resident uint16 frames:

  batch    halide_b200_blur_batch / _stencil_chain_batch / _stencil_chain_stencils_batch on the (N, H, W) clip
  singles  halide_blur / stencil_chain / halide_b200_stencil_chain_stencils on each of its N frames

for four cases (blur; stencil_chain, S = 32; stencil_chain_stencils at S = 4 and S = 100) at 640 x 480, 1920 x 1080 and
3840 x 2160 with N = 8, and 7680 x 4320 with N = 4.  A blur frame's input is the output grown by 2 in x and y.

    python tools/blur_sc_batch_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--sizes 480p,...] [--cases blur,...]
    python tools/blur_sc_batch_bench.py OUT_DIR --compare-lib OTHER.so [--runs 3]

Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window, the arms
alternating, `rounds` times each; the median round is reported with the spread of the rounds.  The two arms' outputs are
compared bit for bit in every case.  For blur it also reports the batch's achieved rate at 4 bytes per output pixel
(a 2-byte read and a 2-byte write) as a fraction of 3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth (a figure from the
data sheet, not one measured here).  Writes OUT_DIR/blur_sc_batch_bench.json and prints one line per case.

--compare-lib times the one-frame halide_blur (3840 x 2160) and stencil_chain (2560 x 1536) with another build of the
library (e.g. the parent commit's) and with this tree's, in alternating processes, `runs` of each, and checks that both
give the same bytes; it writes OUT_DIR/blur_sc_batch_bench_compare.json.  The GPU's name, power limit and top SM clock
are read in the same run."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import torch

import timing
from halide_b200 import HalideBuffer, blur_video, filters, stencil_chain_video

SIZES = {"480p": (480, 640, 8), "1080p": (1080, 1920, 8), "4k": (2160, 3840, 8), "8k": (4320, 7680, 4)}
# name: (batch call, one-frame call), each taking (input buffer, output buffer)
CASES = {
    "blur": (blur_video.blur_batch, filters.halide_blur),
    "sc32": (stencil_chain_video.stencil_chain_batch, filters.stencil_chain),
    "scs4": (lambda i, o: stencil_chain_video.stencil_chain_stencils_batch(i, 4, o),
             lambda i, o: filters.stencil_chain_stencils(i, 4, o)),
    "scs100": (lambda i, o: stencil_chain_video.stencil_chain_stencils_batch(i, 100, o),
               lambda i, o: filters.stencil_chain_stencils(i, 100, o)),
}
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
COMPARE = {"halide_blur": (2160, 3840), "stencil_chain": (1536, 2560)}


def make_clip(n, h, w, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    return torch.randint(0, 1 << 16, (n, h, w), dtype=torch.int32, device="cuda", generator=gen).to(torch.uint16)


def batch_vs_singles(args):
    timing.setup("blur_sc_batch_bench")
    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "window_ms": args.window_ms, "rounds": args.rounds, "cases": []}
    for size in args.sizes.split(","):
        h, w, n = SIZES[size]
        for case in args.cases.split(","):
            a = 2 if case == "blur" else 0
            x = make_clip(n, h + a, w + a, h * 100003 + w + len(case))
            yb = torch.zeros((n, h, w), dtype=torch.uint16, device="cuda")
            ys = torch.zeros_like(yb)
            bi, bo = HalideBuffer.from_torch(x), HalideBuffer.from_torch(yb)
            fi = [HalideBuffer.from_torch(x[k]) for k in range(n)]
            fo = [HalideBuffer.from_torch(ys[k]) for k in range(n)]
            batch, one = CASES[case]

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
            entry = {"size": size, "h": h, "w": w, "n": n, "case": case, "iters": iters, "ms_per_clip": ms,
                     "median_ms": med, "batch_over_singles": ratio, "ratio_range": [lo, hi], "outputs_equal": True,
                     "batch_launches": launches}
            rate = ""
            if case == "blur":
                frac = 4.0 * n * h * w / (med["batch"] * 1e-3) / HBM_BYTES_PER_S
                entry["batch_fraction_of_datasheet_hbm"] = frac
                rate = f"; batch at 4 B/px: {frac:.2f} of the data-sheet 3.35 TB/s"
            result["cases"].append(entry)
            print(f"{size} N={n} {case}: batch {med['batch']:.4f} ms, {n} singles {med['singles']:.4f} ms, "
                  f"batch/singles {ratio:.3f} (rounds {lo:.3f}-{hi:.3f}); batch launches {launches}{rate}; "
                  f"outputs equal", flush=True)
            del x, yb, ys, bi, bo, fi, fo
            torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "blur_sc_batch_bench.json", result)


def one_frame_calls(args):
    """(child process) the one-frame halide_blur and stencil_chain with the library at args.lib: one JSON line."""
    import halide_b200.lib as hlib
    if args.lib:
        hlib.LIB_PATH = os.path.abspath(args.lib)
    timing.setup("blur_sc_batch_bench")
    out = {"lib": hlib.LIB_PATH}
    for name, (h, w) in COMPARE.items():
        a = 2 if name == "halide_blur" else 0
        x = make_clip(1, h + a, w + a, h + w)[0]
        y = torch.zeros((h, w), dtype=torch.uint16, device="cuda")
        bi, bo = HalideBuffer.from_torch(x), HalideBuffer.from_torch(y)
        fn = getattr(filters, name)
        arms = {name: lambda: fn(bi, bo)}
        timing.warm_up(arms)
        _, ms = timing.measure(arms, args.window_ms, args.rounds)
        out[name] = {"median_ms": statistics.median(ms[name]), "ms": ms[name],
                     "sha256": hashlib.sha256(y.cpu().numpy().tobytes()).hexdigest()}
    print(json.dumps(out), flush=True)


def compare_libs(args):
    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    libs = {"other": os.path.abspath(args.compare_lib), "this": ""}
    runs = {k: [] for k in libs}
    for i in range(args.runs):
        for name, path in libs.items():
            cmd = [sys.executable, os.path.abspath(__file__), args.out_dir, "--one-frame-calls", "--window-ms",
                   str(args.window_ms), "--rounds", str(args.rounds)] + (["--lib", path] if path else [])
            out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
            r = json.loads(out.strip().splitlines()[-1])
            runs[name].append(r)
            print(f"run {i} {name}: " + ", ".join(f"{f} {r[f]['median_ms']:.4f} ms" for f in COMPARE), flush=True)
    summary = {}
    for f, (h, w) in COMPARE.items():
        digests = {r[f]["sha256"] for rs in runs.values() for r in rs}
        assert len(digests) == 1, f"the two libraries give different bytes for {f}"
        med = {k: statistics.median(r[f]["median_ms"] for r in rs) for k, rs in runs.items()}
        spread = {k: [min(r[f]["median_ms"] for r in rs), max(r[f]["median_ms"] for r in rs)] for k, rs in runs.items()}
        summary[f] = {"h": h, "w": w, "median_ms": med, "spread_ms": spread, "outputs_equal": True}
        print(f"{f} {w}x{h}: other {med['other']:.4f} ms (runs {spread['other'][0]:.4f}-{spread['other'][1]:.4f}), "
              f"this {med['this']:.4f} ms (runs {spread['this'][0]:.4f}-{spread['this'][1]:.4f}), this/other "
              f"{med['this'] / med['other']:.3f}; outputs equal", flush=True)
    timing.write_json(args.out_dir, "blur_sc_batch_bench_compare.json", {"gpu": info, "runs": runs, "summary": summary})


def main():
    ap = timing.common_args()
    ap.add_argument("--sizes", default=",".join(SIZES))
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--compare-lib", default=None)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--one-frame-calls", action="store_true", help=argparse.SUPPRESS)  # (the children of --compare-lib)
    ap.add_argument("--lib", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one_frame_calls:
        one_frame_calls(args)
    elif args.compare_lib:
        compare_libs(args)
    else:
        batch_vs_singles(args)


if __name__ == "__main__":
    main()
