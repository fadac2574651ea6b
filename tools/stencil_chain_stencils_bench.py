"""stencil_chain at every depth: what halide_b200_stencil_chain_stencils costs per call as the number of stencils moves,
on device-resident uint16 noise frames of 1536 x 2560 (the generator's estimate), 3840 x 2160 and 7680 x 4320 (whose
intermediate planes no longer fit in L2).

    python tools/stencil_chain_stencils_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--s 1,2,3,...]
                                                         [--frames 1536x2560,3840x2160,7680x4320]

Arms per frame: one per number of stencils S, plus `stencil_chain` itself (the fixed-32 entry point) on the same frame.
Every arm is warmed up, then timed with CUDA events on one stream over enough calls to fill the window, the arms
alternating, `rounds` times each; the median round is reported with the spread of the rounds.  For each S the script
reports the time per call, ns per stage per Mpx, the launch count and the work ratio: the stage work of the launch plan
(floor(S / 4) launches of 4 stages and one of S mod 4, each over its output region grown by twice the stages still to
run after it), sum(region area x stages) / (S x W x H), computed from the shapes.  The S = 32 output must equal
stencil_chain's byte for byte.  The GPU's name, power limit and top SM clock are read in the same run.  Writes
OUT_DIR/stencil_chain_stencils_bench.json and prints one line per S."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters

S_VALUES = "1,2,3,4,5,8,16,31,32,33,64,100"
FRAMES = "1536x2560,3840x2160,7680x4320"
FUSE = 4  # stages per launch in stencil_chain.cu


def launch_plan(s):
    """Stages per launch, in launch order: floor(S / 4) launches of 4, then the remainder."""
    full, rest = divmod(s, FUSE)
    return [FUSE] * full + ([rest] if rest else [])


def work_ratio(s, w, h):
    """sum over launches of (output region grown by 2 x stages still to run after it) x (its stages), over S x W x H."""
    done, work = 0, 0
    for f in launch_plan(s):
        r_out = 2 * (s - done - f)
        work += (w + 2 * r_out) * (h + 2 * r_out) * f
        done += f
    return work / (s * w * h)


def main():
    ap = timing.common_args()
    ap.add_argument("--s", default=S_VALUES)
    ap.add_argument("--frames", default=FRAMES)
    args = ap.parse_args()
    s_values = [int(v) for v in args.s.split(",")]
    frames = [tuple(int(v) for v in f.split("x")) for f in args.frames.split(",")]
    timing.setup("stencil_chain_stencils_bench")

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "window_ms": args.window_ms, "rounds": args.rounds, "frames": []}
    for w, h in frames:
        gen = torch.Generator(device="cuda")
        gen.manual_seed(w * h)
        x = torch.randint(-32768, 32768, (h, w), dtype=torch.int32, device="cuda", generator=gen)
        x = x.to(torch.int16).view(torch.uint16)
        bx = HalideBuffer.from_torch(x)
        outs = {s: torch.zeros((h, w), dtype=torch.int16, device="cuda").view(torch.uint16) for s in s_values}
        bouts = {s: HalideBuffer.from_torch(o) for s, o in outs.items()}
        y_ref = torch.zeros((h, w), dtype=torch.int16, device="cuda").view(torch.uint16)
        b_ref = HalideBuffer.from_torch(y_ref)

        arms = {}
        for s in s_values:
            arms[f"s{s}"] = (lambda s=s: filters.stencil_chain_stencils(bx, s, bouts[s]))
        arms["stencil_chain"] = lambda: filters.stencil_chain(bx, b_ref)
        timing.warm_up(arms)
        same32 = None
        if 32 in outs:
            same32 = timing.same(outs[32], y_ref)
            assert same32, f"{w}x{h}: stencils = 32 differs from stencil_chain"
        iters, ms = timing.measure(arms, args.window_ms, args.rounds)
        med = {k: statistics.median(v) for k, v in ms.items()}
        if 32 in outs:
            assert timing.same(outs[32], y_ref), f"{w}x{h}: stencils = 32 differs from stencil_chain after timing"

        mpx = w * h / 1e6
        entry = {"w": w, "h": h, "s32_equals_stencil_chain": same32,
                 "stencil_chain": {"iters": iters["stencil_chain"], "ms_per_call": ms["stencil_chain"],
                                   "median_ms": med["stencil_chain"],
                                   "ns_per_stage_per_mpx": med["stencil_chain"] * 1e6 / (32 * mpx),
                                   "work_ratio": work_ratio(32, w, h)},
                 "stencils": []}
        sc = ms["stencil_chain"]
        print(f"{w}x{h} stencil_chain: {med['stencil_chain']:.3f} ms (rounds {min(sc):.3f}..{max(sc):.3f})", flush=True)
        for s in s_values:
            k = f"s{s}"
            e = {"stencils": s, "launches": len(launch_plan(s)), "iters": iters[k], "ms_per_call": ms[k],
                 "median_ms": med[k], "ns_per_stage_per_mpx": med[k] * 1e6 / (s * mpx), "work_ratio": work_ratio(s, w, h)}
            entry["stencils"].append(e)
            print(f"{w}x{h} S {s}: {med[k]:.3f} ms (rounds {min(ms[k]):.3f}..{max(ms[k]):.3f}), "
                  f"{e['ns_per_stage_per_mpx']:.1f} ns/stage/Mpx, {e['launches']} launches, work x{e['work_ratio']:.3f}",
                  flush=True)
        result["frames"].append(entry)
    timing.write_json(args.out_dir, "stencil_chain_stencils_bench.json", result)


if __name__ == "__main__":
    main()
