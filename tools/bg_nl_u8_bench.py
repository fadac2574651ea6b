"""8-bit bilateral_grid and nl_means on one GPU: what the 8-bit entry points cost next to the float filters and next to
what an 8-bit torch caller does without them.  Three arms on the same device-resident content:

  u8     halide_b200_bilateral_grid_u8 / halide_b200_nl_means_u8 on the uint8 frame
  f32    bilateral_grid / nl_means on the float32 frame to_f32(in8)
  torch  torch's conversion to float32, the float call, and torch's conversion back to uint8

for bilateral_grid (r_sigma 0.1) at 1536 x 2560 (the apps' gray.png), 3840 x 2160 and 7680 x 4320, and nl_means (sigma
0.12) at 1536 x 2560 x 3 (rgb.png) and 3840 x 2160 x 3 with patch / search 3/7 and 7/7.

    python tools/bg_nl_u8_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--cases bg_gray,bg_4k,...]

Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window, the arms
alternating, `rounds` times each; the median round is reported.  The u8 and torch outputs are compared byte for byte in
every case.  Writes OUT_DIR/bg_nl_u8_bench.json (ms per call of every round, and the per-kernel profile of one call of
each arm) and prints one line per case.  The GPU's name, power limit and top SM clock are read in the same run."""
import statistics

import numpy as np
import torch

import timing
from halide_b200 import HalideBuffer, filters

# name: (filter, (channels or 0 for 2-D, height, width), parameters after the input)
CASES = {
    "bg_gray": ("bg", (0, 2560, 1536), (0.1,)),
    "bg_4k": ("bg", (0, 2160, 3840), (0.1,)),
    "bg_8k": ("bg", (0, 4320, 7680), (0.1,)),
    "nl_rgb_3_7": ("nl", (3, 2560, 1536), (3, 7, 0.12)),
    "nl_rgb_7_7": ("nl", (3, 2560, 1536), (7, 7, 0.12)),
    "nl_4k_3_7": ("nl", (3, 2160, 3840), (3, 7, 0.12)),
    "nl_4k_7_7": ("nl", (3, 2160, 3840), (7, 7, 0.12)),
}


def main():
    ap = timing.common_args()
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    timing.setup("bg_nl_u8_bench")

    # to_f32(v) = v / 255.0f as an IEEE division.  The divisor is a device tensor: torch turns division by a Python
    # scalar into a multiply by its reciprocal, which gives another float for 126 of the 256 codes.
    d255 = torch.tensor(255.0, dtype=torch.float32, device="cuda")

    def to_f32(t8):
        return t8.to(torch.float32) / d255

    def to_u8(tf):  # lround(f * 255.0f): the float32 product, then halves up (f >= 0) in float64, where y + 0.5 is exact
        return torch.floor((tf * 255.0).to(torch.float64) + 0.5).to(torch.uint8)

    codes = torch.arange(256, dtype=torch.int32, device="cuda").to(torch.uint8)
    exact = np.arange(256, dtype=np.float32) / np.float32(255.0)
    assert np.array_equal(to_f32(codes).cpu().numpy(), exact), "torch's to_f32 is not v / 255.0f"

    def profile(fn):
        return {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(fn).items())}

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "window_ms": args.window_ms, "rounds": args.rounds, "cases": []}
    gen = torch.Generator(device="cuda")
    for name in args.cases.split(","):
        filt, (c, h, w), params = CASES[name]
        gen.manual_seed(h * 100003 + w)
        shape = (c, h, w) if c else (h, w)
        x8 = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)
        xf = to_f32(x8)
        y8, yf, y8t = torch.zeros_like(x8), torch.zeros_like(xf), torch.zeros_like(x8)
        b8i, b8o = HalideBuffer.from_torch(x8), HalideBuffer.from_torch(y8)
        bfi, bfo = HalideBuffer.from_torch(xf), HalideBuffer.from_torch(yf)
        f8 = filters.bilateral_grid_u8 if filt == "bg" else filters.nl_means_u8
        ff = filters.bilateral_grid if filt == "bg" else filters.nl_means

        def arm_u8():
            f8(b8i, *params, b8o)

        def arm_f32():
            ff(bfi, *params, bfo)

        def arm_torch():
            tf = to_f32(x8)
            of = torch.empty_like(tf)
            ff(HalideBuffer.from_torch(tf), *params, HalideBuffer.from_torch(of))
            y8t.copy_(to_u8(of))

        arms = {"u8": arm_u8, "f32": arm_f32, "torch": arm_torch}
        timing.warm_up(arms)
        assert torch.equal(y8, y8t), f"u8 and torch arms differ at {name}"
        iters, ms = timing.measure(arms, args.window_ms, args.rounds)
        assert torch.equal(y8, y8t), f"u8 and torch arms differ at {name} after timing"
        med = {k: statistics.median(v) for k, v in ms.items()}
        entry = {"case": name, "filter": filt, "shape": list(shape), "params": list(params), "iters": iters,
                 "ms_per_call": ms, "median_ms": med, "u8_equals_torch": True,
                 "profile_ms": {k: profile(fn) for k, fn in arms.items()}}
        result["cases"].append(entry)
        print(f"{name}: u8 {med['u8']:.3f} ms, f32 {med['f32']:.3f} ms, torch {med['torch']:.3f} ms "
              f"(u8/f32 {med['u8'] / med['f32']:.3f}, u8/torch {med['u8'] / med['torch']:.3f}); outputs u8 == torch; "
              "u8 profile " + ", ".join(f"{k} {v['ms']:.3f}" for k, v in entry["profile_ms"]["u8"].items()) +
              "; f32 profile " + ", ".join(f"{k} {v['ms']:.3f}" for k, v in entry["profile_ms"]["f32"].items()),
              flush=True)
        del x8, xf, y8, yf, y8t, b8i, b8o, bfi, bfo
        torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "bg_nl_u8_bench.json", result)


if __name__ == "__main__":
    main()
