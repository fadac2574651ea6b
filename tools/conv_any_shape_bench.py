"""halide_b200_conv_layer_any_shape across layer shapes: time per call, useful TFLOP/s and the per-kernel split, on
device-resident buffers.

    python tools/conv_any_shape_bench.py OUT_DIR [--window-ms 200] [--rounds 3]

Shapes (N, CI, CO, W, H): conv_layer's fixed one, a first layer (3 input channels), four ResNet-like stages, a
1024-channel layer (288 K steps: the accumulators fold 7 times) and an odd one.  Arms, all warmed up, then timed with
CUDA events on one stream over enough calls to fill the window, alternating, `rounds` times each; the median round is
reported:

  any_shape   halide_b200_conv_layer_any_shape: split of the input, re-lay of the filter and the GEMM, every call
  conv_layer  (fixed shape only) the drop-in filter on the same buffers; the outputs must be equal byte for byte
  torch       context, not a like-for-like arm: torch.nn.functional.conv2d on channels_last tensors with
              allow_tf32 = False (cuDNN's fp32 kernels; no 3xTF32), then + bias and relu as two more elementwise
              kernels.  Its input is the same padded tensor (padding = 0), its weight is already in cuDNN's layout, so
              it includes no filter re-lay, and its algorithm search happens in the warm-up.

Per shape: microseconds per call, useful TFLOP/s = 2 * 9 * CI * CO * W * H * N / t, that over 165 TFLOP/s (the 3xTF32
bound: a third of the H100 SXM data sheet's 495 dense TF32 TFLOP/s, because three MMAs are issued per product; a
compute bound of the GEMM alone, which the split and re-lay kernels and a power limit below 700 W both lower), the
mean per-kernel times of 20 profiled calls, and the largest error over the derived float64 bound on signed data
(tests/conv_any_exact.py: harness_bound).  The GPU's name, power limit and top SM clock are read in the same run.
Writes OUT_DIR/conv_any_shape_bench.json and prints one line per shape.  Fails without a GPU."""
import os
import statistics
import sys

import torch

import timing
from halide_b200 import HalideBuffer, filters

sys.path.insert(0, os.path.join(timing.ROOT, "tests"))

FIXED = (5, 128, 128, 100, 80)
SHAPES = [FIXED, (1, 3, 64, 224, 224), (8, 64, 64, 56, 56), (8, 128, 128, 28, 28), (8, 256, 256, 14, 14), (32, 512, 512, 7, 7),
          (1, 1024, 1024, 14, 14), (3, 37, 75, 29, 17)]
BOUND_TFLOPS = 495.0 / 3.0


def main():
    args = timing.common_args(window_ms=200.0).parse_args()
    timing.setup("conv_any_shape_bench")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    import numpy as np
    import conv_any_exact as cx

    def profile(fn, calls=20):
        """Microseconds per launch of each kernel, the mean over `calls` profiled calls (every launch bracketed by events,
        which keeps the kernels from overlapping: the times add up to more than an unprofiled call)."""
        return {k: round(t * 1e3 / c, 2) for k, (c, t) in sorted(timing.profile(fn, calls).items())}

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "window_ms": args.window_ms, "rounds": args.rounds, "bound_tflops": BOUND_TFLOPS, "shapes": []}
    for shape in SHAPES:
        n, ci, co, w, h = shape
        inp, filt, bias = cx.harness("signed", shape)
        ti, tf, tb = (torch.from_numpy(a).cuda() for a in (inp, filt, bias))
        to = torch.full((n, h, w, co), float("nan"), device="cuda")
        bufs = [HalideBuffer.from_torch(t) for t in (ti, tf, tb, to)]
        arms = {"any_shape": lambda: filters.conv_layer_any_shape(*bufs)}
        if shape == FIXED:
            to_fixed = torch.full_like(to, float("nan"))
            bufs_fixed = bufs[:3] + [HalideBuffer.from_torch(to_fixed)]
            arms["conv_layer"] = lambda: filters.conv_layer(*bufs_fixed)
        # torch: NCHW logical shape in channels_last memory = the same NHWC bytes; weight [CO, CI, 3, 3] channels_last
        x_t = ti.permute(0, 3, 1, 2)
        w_t = tf.permute(3, 0, 1, 2).contiguous(memory_format=torch.channels_last)
        b_t = tb.view(1, co, 1, 1)
        arms["torch"] = lambda: torch.relu_(torch.nn.functional.conv2d(x_t, w_t).add_(b_t))
        timing.warm_up(arms)
        got = to.cpu().numpy()
        ratio = cx.worst_ratio(got, inp, filt, bias)
        assert np.isfinite(got).all() and ratio <= 1.0, (shape, ratio)
        if shape == FIXED:
            assert torch.equal(to.view(torch.int32), to_fixed.view(torch.int32)), "any_shape differs from conv_layer at its shape"
        iters, ms = timing.measure(arms, args.window_ms, args.rounds)
        us = {k: statistics.median(v) * 1e3 for k, v in ms.items()}
        flop = 2.0 * 9 * ci * co * w * h * n
        tflops = flop / (us["any_shape"] * 1e-6) / 1e12
        entry = {"shape": shape, "gflop": flop / 1e9, "iters": iters, "us_rounds": {k: [v * 1e3 for v in r] for k, r in ms.items()},
                 "us": us, "useful_tflops": tflops, "share_of_3xtf32_bound": tflops / BOUND_TFLOPS,
                 "kernels_us": profile(arms["any_shape"]), "max_err_over_bound": ratio, "folds": cx.folds(ci)}
        if shape == FIXED:
            entry["conv_layer_kernels_us"] = profile(arms["conv_layer"])
        result["shapes"].append(entry)
        print(f"{shape}: any_shape {us['any_shape']:.1f} us, {tflops:.1f} useful TFLOP/s = {100 * tflops / BOUND_TFLOPS:.0f}% of the "
              f"3xTF32 bound; " + (f"conv_layer {us['conv_layer']:.1f} us; " if shape == FIXED else "") +
              f"torch fp32 {us['torch']:.1f} us; kernels " + ", ".join(f"{k} {v}" for k, v in entry["kernels_us"].items()) +
              f"; err/bound {ratio:.2f}", flush=True)
    timing.write_json(args.out_dir, "conv_any_shape_bench.json", result)


if __name__ == "__main__":
    main()
