"""8-bit local_laplacian on one GPU: what the fused 8-bit entry points cost next to the uint16 filter and next to what an
8-bit torch caller does without them.  Three arms on the same device-resident content (levels 8, alpha 1/7, beta 1):

  u8     halide_b200_local_laplacian_u8 (or _u8_batch) on the uint8 frames
  u16    local_laplacian (or halide_b200_local_laplacian_batch) on the uint16 frames to_u16(in8)
  torch  a torch conversion to uint16 (through int32), the uint16 call, and a torch conversion back to uint8

for 1080p, 4K and 16K single frames and batches of 8 x 1080p and 8 x 4K.

    python tools/ll_u8_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--sizes 1080p,4k,16k,8x1080p,8x4k]

Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window, the arms
alternating, `rounds` times each; the median round is reported.  The outputs of the u8 and torch arms are compared bit
for bit at every size.  Writes OUT_DIR/ll_u8_bench.json (ms per call of every round, and the per-kernel profile of one u8
and one u16 call) and prints one line per size.  The GPU's name, power limit and top SM clock are read in the same run."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters

SIZES = {"1080p": (1, 1920, 1080), "4k": (1, 3840, 2160), "16k": (1, 16384, 16384), "8x1080p": (8, 1920, 1080),
         "8x4k": (8, 3840, 2160)}
LEVELS, ALPHA, BETA = 8, 1.0 / 7.0, 1.0


def main():
    ap = timing.common_args()
    ap.add_argument("--sizes", default=",".join(SIZES))
    args = ap.parse_args()
    timing.setup("ll_u8_bench")

    def to_u16(t8):  # convert<uint16_t, uint8_t>: v * 257
        return (t8.to(torch.int32) * 257).to(torch.int16).view(torch.uint16)

    def to_u8(t16):  # convert<uint8_t, uint16_t>: ((w + 128) * 255 + 255) >> 16
        w = t16.view(torch.int16).to(torch.int32) & 0xFFFF
        return (((w + 128) * 255 + 255) >> 16).to(torch.uint8)

    def profile(fn):
        return {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(fn).items())}

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "levels": LEVELS, "alpha": ALPHA, "beta": BETA, "window_ms": args.window_ms,
              "rounds": args.rounds, "sizes": []}
    gen = torch.Generator(device="cuda")
    for name in args.sizes.split(","):
        n, w, h = SIZES[name]
        gen.manual_seed(n * 100003 + w)
        shape = (n, 3, h, w) if n > 1 else (3, h, w)
        x8 = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)
        x16 = to_u16(x8)
        y8, y16 = torch.zeros_like(x8), torch.zeros_like(x16)
        y8t = torch.zeros_like(x8)
        b8i, b8o = HalideBuffer.from_torch(x8), HalideBuffer.from_torch(y8)
        b16i, b16o = HalideBuffer.from_torch(x16), HalideBuffer.from_torch(y16)
        f8 = filters.local_laplacian_u8_batch if n > 1 else filters.local_laplacian_u8
        f16 = filters.local_laplacian_batch if n > 1 else filters.local_laplacian

        def arm_u8():
            f8(b8i, LEVELS, ALPHA, BETA, b8o)

        def arm_u16():
            f16(b16i, LEVELS, ALPHA, BETA, b16o)

        def arm_torch():
            t16 = to_u16(x8)
            o16 = torch.empty_like(t16)
            f16(HalideBuffer.from_torch(t16), LEVELS, ALPHA, BETA, HalideBuffer.from_torch(o16))
            y8t.copy_(to_u8(o16))

        arms = {"u8": arm_u8, "u16": arm_u16, "torch": arm_torch}
        timing.warm_up(arms)
        assert torch.equal(y8, y8t), f"u8 and torch arms differ at {name}"
        iters, ms = timing.measure(arms, args.window_ms, args.rounds)
        assert torch.equal(y8, y8t), f"u8 and torch arms differ at {name} after timing"
        med = {k: statistics.median(v) for k, v in ms.items()}
        entry = {"size": name, "n": n, "w": w, "h": h, "iters": iters, "ms_per_call": ms, "median_ms": med,
                 "u8_equals_torch": True, "profile_u8_ms": profile(arm_u8), "profile_u16_ms": profile(arm_u16)}
        result["sizes"].append(entry)
        print(f"{name}: u8 {med['u8']:.3f} ms, u16 {med['u16']:.3f} ms, torch {med['torch']:.3f} ms "
              f"(u8/u16 {med['u8'] / med['u16']:.3f}, u8/torch {med['u8'] / med['torch']:.3f}); outputs u8 == torch; "
              "u8 profile " + ", ".join(f"{k} {v['ms']:.3f}" for k, v in entry["profile_u8_ms"].items()) +
              "; u16 profile " + ", ".join(f"{k} {v['ms']:.3f}" for k, v in entry["profile_u16_ms"].items()), flush=True)
        del x8, x16, y8, y16, y8t, b8i, b8o, b16i, b16o
        torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "ll_u8_bench.json", result)


if __name__ == "__main__":
    main()
