"""How the tools/ benchmarks measure, kept in one place so that their numbers (DESIGN §9, the README tables) stay
comparable: every arm is warmed up, each arm's calls per round are probed to fill the window, then `rounds` rounds are
timed with CUDA events, the arms alternating in a fixed order inside each round; the scripts report the median round.

Importing this module puts the repository root on sys.path, so the scripts import halide_b200 from the tree."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import halide_b200.lib as hlib  # noqa: E402


def gpu_info():
    """The GPU's name, power limit and top SM clock, which belong beside any number measured on it."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def setup(tool_name):
    """Exit unless there is a CUDA GPU; otherwise select device 0, put the library on torch's current stream (so the
    CUDA events bracket its kernels) and return the library handle."""
    if not torch.cuda.is_available():
        sys.exit(f"{tool_name} needs a CUDA GPU")
    torch.cuda.set_device(0)
    l = hlib.load_library()
    l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return l


def timed(fn, iters):
    """Milliseconds per call of `iters` back-to-back calls of fn."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def warm_up(arms):
    """Three calls of every arm of the ordered dict `arms` (name -> callable), then a synchronize."""
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()


def measure(arms, window_ms, rounds):
    """Probes every arm for the calls that fill `window_ms`, then times `rounds` rounds, the arms alternating in dict
    order.  Returns ({name: calls per round}, {name: [ms per call of each round]})."""
    iters = {k: max(3, int(window_ms / max(timed(fn, 3), 1e-3))) for k, fn in arms.items()}
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(timed(fn, iters[k]))
    return iters, ms


def profile(fn, calls=1):
    """The library's per-kernel profile of `calls` calls of fn: {kernel: (launches, total ms)}."""
    hlib.profile(True)
    hlib.profile_reset()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    prof = hlib.profile_report()
    hlib.profile(False)
    return prof


def same(a, b):
    """Bit-for-bit equality; uint16 tensors are compared as int16 views (torch's uint16 has copies, not comparisons)."""
    if a.dtype == torch.uint16:
        a, b = a.view(torch.int16), b.view(torch.int16)
    return torch.equal(a, b)


def common_args(window_ms=300.0):
    """The arguments every benchmark takes: OUT_DIR, --window-ms and --rounds."""
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window-ms", type=float, default=window_ms)
    ap.add_argument("--rounds", type=int, default=3)
    return ap


def write_json(out_dir, filename, result):
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, filename)
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {path}")
