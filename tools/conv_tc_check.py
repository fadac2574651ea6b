"""Compares conv_layer's two contractions through the C ABI: the wgmma path (the default) and the FP32 SIMT kernel.
For each path: the largest relative error against the CPU oracle on the harness's two input scales (rand() in [0, 1)
and up to 2^31), and the mean time per call on device-resident buffers (CUDA events over 50 calls after warm-up).
    python tools/conv_tc_check.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import halide_b200 as hb  # noqa: E402
from oracle import pyoracle  # noqa: E402
from test_conv_layer_gpu import make, run  # noqa: E402


def time_path(l, use_tc, calls=50):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    bi, bf, bb = (hb.HalideBuffer.from_torch(torch.rand(s, dtype=torch.float32, device=dev, generator=g))
                  for s in ((5, 82, 102, 128), (128, 3, 3, 128), (128,)))
    bo = hb.HalideBuffer.from_torch(torch.zeros((5, 80, 100, 128), dtype=torch.float32, device=dev))
    l.halide_b200_conv_use_tensor_cores(1 if use_tc else 0)
    for _ in range(5):
        hb.filters.conv_layer(bi, bf, bb, bo)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        hb.filters.conv_layer(bi, bf, bb, bo)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls * 1e3


def main():
    l = hb.load_library()
    pyoracle.set_threads(min(16, pyoracle.use_all_cores()))
    result = {"device": torch.cuda.get_device_name(0)}
    for use_tc, name in ((1, "wgmma"), (0, "simt")):
        errs = []
        for seed, scale in ((0, 1.0), (1, 2147483648.0)):
            inp, filt, bias = make(seed, scale)
            want = pyoracle.conv_layer(inp, filt, bias)
            l.halide_b200_conv_use_tensor_cores(use_tc)
            got = run(hb, inp, filt, bias)
            errs.append(float((np.abs(got - want) / np.maximum(np.abs(want), 1e-30)).max()))
        result[name] = {"max_rel_err": errs, "us_per_call": time_path(l, use_tc)}
    l.halide_b200_conv_use_tensor_cores(1)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
