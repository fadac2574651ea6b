"""Interleaved local_laplacian on one GPU: what the interleaved entry points cost next to the planar filter and next to
what a caller holding pixel-interleaved frames does without them.  Three arms on the same device-resident content (levels
8, alpha 1/7, beta 1), all on torch's current stream:

  il      halide_b200_local_laplacian[_u8]_interleaved[_batch] on the interleaved frames ([N,] H, W, P tensors)
  planar  the planar entry point on planar frames of the same size and type (a planar copy of the same content)
  torch   permute().contiguous() into a planar frame, the planar call, and the planar output permuted back into the
          interleaved output

for 1080p, 4K and 16K single frames and batches of 8 x 1080p and 8 x 4K, uint8 and uint16, RGB (pitch 3 in and out) and
RGBA -> RGB (pitch 4 in, 3 out).

    python tools/ll_interleaved_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--sizes 1080p,4k,16k,8x1080p,8x4k]
                                                 [--types u8,u16] [--layouts rgb,rgba]

Every arm is warmed up, then timed with CUDA events over enough calls to fill the window, the arms alternating, `rounds`
times each; the median round is reported.  The outputs of the three arms are compared bit for bit at every size.  Writes
OUT_DIR/ll_interleaved_bench.json (ms per call of every round, and the per-kernel profile of one il and one planar call)
and prints one line per case.  The GPU's name, power limit and top SM clock are read in the same run."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters

SIZES = {"1080p": (1, 1920, 1080), "4k": (1, 3840, 2160), "16k": (1, 16384, 16384), "8x1080p": (8, 1920, 1080),
         "8x4k": (8, 3840, 2160)}
LAYOUTS = {"rgb": 3, "rgba": 4}  # input pixel pitch; the output is RGB (pitch 3) either way
LEVELS, ALPHA, BETA = 8, 1.0 / 7.0, 1.0


def main():
    ap = timing.common_args()
    ap.add_argument("--sizes", default=",".join(SIZES))
    ap.add_argument("--types", default="u8,u16")
    ap.add_argument("--layouts", default=",".join(LAYOUTS))
    args = ap.parse_args()
    timing.setup("ll_interleaved_bench")

    def profile(fn):
        return {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(fn).items())}

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "levels": LEVELS, "alpha": ALPHA, "beta": BETA, "window_ms": args.window_ms,
              "rounds": args.rounds, "cases": []}
    gen = torch.Generator(device="cuda")
    for name in args.sizes.split(","):
        n, w, h = SIZES[name]
        for tname in args.types.split(","):
            for lname in args.layouts.split(","):
                pitch = LAYOUTS[lname]
                gen.manual_seed(n * 100003 + w + pitch)
                shape = (n, h, w, pitch) if n > 1 else (h, w, pitch)
                if tname == "u8":
                    x = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)
                else:
                    x = torch.randint(-32768, 32768, shape, dtype=torch.int16, device="cuda", generator=gen).view(torch.uint16)
                y = torch.empty(shape[:-1] + (3,), dtype=x.dtype, device="cuda")
                y_t = torch.empty_like(y)
                to_planar = (0, 3, 1, 2) if n > 1 else (2, 0, 1)
                to_il = (0, 2, 3, 1) if n > 1 else (1, 2, 0)
                xp = x.permute(*to_planar).contiguous()
                yp = torch.empty(xp.shape[:-3] + (3,) + xp.shape[-2:], dtype=x.dtype, device="cuda")
                b_il_in, b_il_out = HalideBuffer.from_torch(x.permute(*to_planar)), HalideBuffer.from_torch(y.permute(*to_planar))
                b_pl_in, b_pl_out = HalideBuffer.from_torch(xp), HalideBuffer.from_torch(yp)
                u8, batch = tname == "u8", n > 1
                f_il = {(False, False): filters.local_laplacian_interleaved, (False, True): filters.local_laplacian_interleaved_batch,
                        (True, False): filters.local_laplacian_u8_interleaved,
                        (True, True): filters.local_laplacian_u8_interleaved_batch}[u8, batch]
                f_pl = {(False, False): filters.local_laplacian, (False, True): filters.local_laplacian_batch,
                        (True, False): filters.local_laplacian_u8, (True, True): filters.local_laplacian_u8_batch}[u8, batch]

                def arm_il():
                    f_il(b_il_in, LEVELS, ALPHA, BETA, b_il_out)

                def arm_planar():
                    f_pl(b_pl_in, LEVELS, ALPHA, BETA, b_pl_out)

                def arm_torch():
                    t_in = x.permute(*to_planar).contiguous()
                    t_out = torch.empty(t_in.shape[:-3] + (3,) + t_in.shape[-2:], dtype=x.dtype, device="cuda")
                    f_pl(HalideBuffer.from_torch(t_in), LEVELS, ALPHA, BETA, HalideBuffer.from_torch(t_out))
                    y_t.copy_(t_out.permute(*to_il))

                arms = {"il": arm_il, "planar": arm_planar, "torch": arm_torch}
                timing.warm_up(arms)

                def check_outputs(when):
                    assert timing.same(y, y_t), f"il and torch arms differ at {name} {tname} {lname} {when}"
                    assert timing.same(y, yp.permute(*to_il)), f"il and planar arms differ at {name} {tname} {lname} {when}"

                check_outputs("after warm-up")
                iters, ms = timing.measure(arms, args.window_ms, args.rounds)
                check_outputs("after timing")
                med = {k: statistics.median(v) for k, v in ms.items()}
                entry = {"size": name, "type": tname, "layout": lname, "n": n, "w": w, "h": h, "iters": iters,
                         "ms_per_call": ms, "median_ms": med, "outputs_identical": True,
                         "profile_il_ms": profile(arm_il), "profile_planar_ms": profile(arm_planar)}
                result["cases"].append(entry)
                print(f"{name} {tname} {lname}: il {med['il']:.3f} ms, planar {med['planar']:.3f} ms, torch {med['torch']:.3f} ms "
                      f"(il/planar {med['il'] / med['planar']:.3f}, il/torch {med['il'] / med['torch']:.3f}); outputs identical; "
                      "il profile " + ", ".join(f"{k} {v['ms']:.3f}" for k, v in entry["profile_il_ms"].items()) +
                      "; planar profile " + ", ".join(f"{k} {v['ms']:.3f}" for k, v in entry["profile_planar_ms"].items()),
                      flush=True)
                del x, y, y_t, xp, yp, b_il_in, b_il_out, b_pl_in, b_pl_out
                torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "ll_interleaved_bench.json", result)


if __name__ == "__main__":
    main()
