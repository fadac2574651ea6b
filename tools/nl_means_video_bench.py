"""nl_means on video clips and pixel-interleaved frames on one GPU: what the batch and interleaved entry points cost next
to what a caller does without them.  For float32 and uint8, patch / search 3/7 and 7/7, and frames of 640 x 480,
1280 x 720, 1920 x 1080 and 3840 x 2160, three comparisons on the same device-resident content:

  interleaved vs planar     the interleaved entry point on an (H, W, 3) frame / the planar one on a (3, H, W) frame
  interleaved vs permutes   the interleaved entry point / torch's permute to a planar copy, the planar call and torch's
                            permute back to (H, W, 3)
  batch vs singles          the planar batch entry point on an (8, 3, H, W) clip / 8 planar one-frame calls

    python tools/nl_means_video_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--sizes 480p,720p,1080p,4k]

Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window, the arms of a
comparison alternating, `rounds` times each; the median round is reported.  The outputs of the arms of each comparison
are checked bit for bit in the same run.  Writes OUT_DIR/nl_means_video_bench.json and prints one line per comparison,
with the GPU's name, power limit and top SM clock read in the same run."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters, nl_means_video

SIZES = {"480p": (480, 640), "720p": (720, 1280), "1080p": (1080, 1920), "4k": (2160, 3840)}
SIGMA = 0.12
BATCH = 8


def main():
    ap = timing.common_args()
    ap.add_argument("--sizes", default=",".join(SIZES))
    args = ap.parse_args()
    timing.setup("nl_means_video_bench")
    info = timing.gpu_info()
    print(f"GPU: {info}")
    g = torch.Generator(device="cuda")
    g.manual_seed(2024)
    results = {"gpu": info, "window_ms": args.window_ms, "rounds": args.rounds, "cases": []}
    for dtype in (torch.float32, torch.uint8):
        u8 = dtype == torch.uint8
        one = filters.nl_means_u8 if u8 else filters.nl_means
        inter = nl_means_video.nl_means_u8_interleaved if u8 else nl_means_video.nl_means_interleaved
        batch = nl_means_video.nl_means_u8_batch if u8 else nl_means_video.nl_means_batch
        for size in args.sizes.split(","):
            h, w = SIZES[size]
            if u8:
                clip = torch.randint(0, 256, (BATCH, 3, h, w), dtype=torch.uint8, device="cuda", generator=g)
            else:
                clip = torch.rand((BATCH, 3, h, w), dtype=torch.float32, device="cuda", generator=g)
            planar = clip[0].contiguous()                       # (3, H, W)
            hwc = planar.permute(1, 2, 0).contiguous()          # (H, W, 3)
            out_p, out_hwc, out_b = torch.empty_like(planar), torch.empty_like(hwc), torch.empty_like(clip)
            outs_1 = [torch.empty_like(planar) for _ in range(BATCH)]
            frames = [clip[k] for k in range(BATCH)]
            # (the buffers are described once: a caller keeps its HalideBuffers across calls)
            b_planar, b_out_p = HalideBuffer.from_torch(planar), HalideBuffer.from_torch(out_p)
            b_hwc, b_out_hwc = HalideBuffer.from_torch(hwc.permute(2, 0, 1)), HalideBuffer.from_torch(out_hwc.permute(2, 0, 1))
            b_clip, b_out_b = HalideBuffer.from_torch(clip), HalideBuffer.from_torch(out_b)
            b_frames = [HalideBuffer.from_torch(f) for f in frames]
            b_outs_1 = [HalideBuffer.from_torch(o) for o in outs_1]
            for patch, search in ((3, 7), (7, 7)):
                p = (patch, search, SIGMA)
                out_perm = {}

                def permuted():
                    x = hwc.permute(2, 0, 1).contiguous()
                    y = torch.empty_like(x)
                    one(HalideBuffer.from_torch(x), *p, HalideBuffer.from_torch(y))
                    out_perm["y"] = y.permute(1, 2, 0).contiguous()

                def singles():
                    for bf, bo in zip(b_frames, b_outs_1):
                        one(bf, *p, bo)

                comparisons = {
                    "interleaved_vs_planar": {"interleaved": lambda: inter(b_hwc, *p, b_out_hwc),
                                              "planar": lambda: one(b_planar, *p, b_out_p)},
                    "interleaved_vs_permutes": {"interleaved": lambda: inter(b_hwc, *p, b_out_hwc),
                                                "permutes": permuted},
                    "batch_vs_singles": {"batch": lambda: batch(b_clip, *p, b_out_b), "singles": singles},
                }
                for cname, arms in comparisons.items():
                    timing.warm_up(arms)
                    if cname == "interleaved_vs_planar":
                        ok = timing.same(out_hwc.permute(2, 0, 1), out_p)
                    elif cname == "interleaved_vs_permutes":
                        ok = timing.same(out_hwc, out_perm["y"])
                    else:
                        ok = all(timing.same(out_b[k], outs_1[k]) for k in range(BATCH))
                    assert ok, f"{cname} {dtype} {size} {patch}/{search}: the arms' outputs differ"
                    iters, ms = timing.measure(arms, args.window_ms, args.rounds)
                    med = {k: statistics.median(v) for k, v in ms.items()}
                    names = list(arms)
                    ratio = med[names[0]] / med[names[1]]
                    tag = "u8" if u8 else "f32"
                    print(f"{tag:3s} {size:5s} {patch}/{search} {cname:24s} " +
                          "  ".join(f"{k} {med[k]:8.3f} ms" for k in names) + f"  ratio {ratio:.3f}  (outputs identical)")
                    results["cases"].append({"dtype": tag, "size": size, "patch": patch, "search": search,
                                             "comparison": cname, "calls_per_round": iters, "ms": ms, "median_ms": med,
                                             "ratio": ratio, "identical": ok})
            del clip, planar, hwc, out_p, out_hwc, out_b, outs_1, frames
            torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "nl_means_video_bench.json", results)


if __name__ == "__main__":
    main()
