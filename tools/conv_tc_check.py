"""Checks conv_layer's wgmma contraction through the C ABI: on the harness's two input scales (rand() in [0, 1) and up to
2^31), the largest relative error against the CPU oracle, and the kernel's and the oracle's own against float64; on
those and tests/conv_exact.py's signed and channel-scaled data, the largest error over the bound
tests/test_conv_layer_exact_gpu.py allows; and the mean time per call on device-resident buffers (CUDA events over 50
calls after warm-up).
    python tools/conv_tc_check.py"""
import json
import os
import sys

import numpy as np
import torch

import timing

sys.path.insert(0, os.path.join(timing.ROOT, "tests"))
import conv_exact  # noqa: E402
import halide_b200 as hb  # noqa: E402
from oracle import pyoracle  # noqa: E402
from test_conv_layer_gpu import make, run  # noqa: E402


def time_call(calls=50):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    bi, bf, bb = (hb.HalideBuffer.from_torch(torch.rand(s, dtype=torch.float32, device=dev, generator=g))
                  for s in ((5, 82, 102, 128), (128, 3, 3, 128), (128,)))
    bo = hb.HalideBuffer.from_torch(torch.zeros((5, 80, 100, 128), dtype=torch.float32, device=dev))

    def call():
        hb.filters.conv_layer(bi, bf, bb, bo)

    for _ in range(5):
        call()
    torch.cuda.synchronize()
    return timing.timed(call, calls) * 1e3


def rel_err(got, want):
    return float((np.abs(got.astype(np.float64) - want) / np.maximum(np.abs(want), 1e-30)).max())


def main():
    hb.load_library()
    pyoracle.set_threads(min(16, pyoracle.use_all_cores()))
    errs, kernel_f64, oracle_f64 = [], [], []
    for seed, scale in ((0, 1.0), (1, 2147483648.0)):
        inp, filt, bias = make(seed, scale)
        want = pyoracle.conv_layer(inp, filt, bias)
        got = run(hb, inp, filt, bias)
        want64 = np.maximum(conv_exact.ref64(inp, filt, bias), 0.0)
        errs.append(rel_err(got, want))
        kernel_f64.append(rel_err(got, want64))
        oracle_f64.append(rel_err(want, want64))
    err_over_bound = {}
    for case in conv_exact.HARNESS_CASES:
        inp, filt, bias = conv_exact.harness(case)
        want64, bound = conv_exact.harness_bound(inp, filt, bias)
        err_over_bound[case] = float((np.abs(conv_exact.run(hb, inp, filt, bias) - want64) / bound).max())
    print(json.dumps({"device": torch.cuda.get_device_name(0), "max_rel_err": errs, "kernel_max_rel_err_vs_f64": kernel_f64,
                      "oracle_max_rel_err_vs_f64": oracle_f64, "kernel_max_err_over_bound": err_over_bound,
                      "us_per_call": time_call()}), flush=True)


if __name__ == "__main__":
    main()
