"""camera_pipe bursts and interleaved output on one GPU: what the burst and interleaved entry points cost next to the
planar filter and next to what a caller who wants (H, W, 3) RGB does without them.  Arms on the same device-resident
raw content (10-bit, the harness's parameters), all on torch's current stream:

  il      halide_b200_camera_pipe_interleaved[_batch] into an ([N,] H, W, 3) uint8 tensor
  planar  camera_pipe (one frame) or halide_b200_camera_pipe_batch (a burst) into ([N,] 3, H, W)
  torch   the planar call into a planar frame, then permuted by torch into the interleaved output
  calls   bursts only: N single camera_pipe calls, one per frame, into the planar burst (against the planar arm's one
          batch call)

for outputs of 1920 x 1080, 2560 x 1920 (the harness frame), 3840 x 2160 and 7680 x 4320, each from the raw frame the
bounds query asks for, and bursts of 8 x 1080p and 8 x 2560 x 1920.

    python tools/camera_pipe_burst_bench.py OUT_DIR [--window-ms 300] [--rounds 3] [--sizes 1080p,2560x1920,4k,8k,8x1080p,8x2560x1920]

Every arm is warmed up, then timed with CUDA events over enough calls to fill the window, the arms alternating, `rounds`
times each; the median round is reported, with the achieved rate at the pipeline's 5 algorithmic bytes per output pixel
(2 raw + 3 RGB).  The outputs of all arms are compared bit for bit at every size.  Writes
OUT_DIR/camera_pipe_burst_bench.json (ms per call of every round, and the per-kernel profile of one call of each arm)
and prints one line per case.  The GPU's name, power limit and top SM clock are read in the same run."""
import statistics

import numpy as np
import torch

import timing
from halide_b200 import HalideBuffer, filters

SIZES = {"1080p": (1, 1920, 1080), "2560x1920": (1, 2560, 1920), "4k": (1, 3840, 2160), "8k": (1, 7680, 4320),
         "8x1080p": (8, 1920, 1080), "8x2560x1920": (8, 2560, 1920)}
M3200 = np.array([[1.6697, -0.2693, -0.4004, -42.4346], [-0.3576, 1.0615, 1.5949, -37.1158],
                  [-0.2175, -1.8751, 6.9640, -26.6970]], np.float32)
M7000 = np.array([[2.2997, -0.4478, 0.1706, -39.0923], [-0.3826, 1.5906, -0.2080, -25.4311],
                  [-0.0888, -0.7344, 2.2832, -20.0826]], np.float32)
PARAMS = (3700.0, 2.0, 50.0, 1.0, 25, 1023)  # color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel
BYTES_PER_PIXEL = 5


def raw_region(n, w, h, b32, b70):
    """(x0, y0, raw width, raw height) the bounds query asks for n frames of a w x h output."""
    q = HalideBuffer.bounds_query(np.uint16, 3)
    filters.camera_pipe_batch(q, b32, b70, *PARAMS, HalideBuffer(np.uint8, (w, h, 3, n)))
    (x0, rw, _), (y0, rh, _), _ = q.shape()
    return x0, y0, rw, rh


def main():
    ap = timing.common_args()
    ap.add_argument("--sizes", default=",".join(SIZES))
    args = ap.parse_args()
    timing.setup("camera_pipe_burst_bench")

    def profile(fn):
        return {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(fn).items())}

    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "params": PARAMS, "bytes_per_pixel": BYTES_PER_PIXEL, "window_ms": args.window_ms,
              "rounds": args.rounds, "cases": []}
    b32, b70 = HalideBuffer.from_torch(torch.from_numpy(M3200).cuda()), HalideBuffer.from_torch(torch.from_numpy(M7000).cuda())
    gen = torch.Generator(device="cuda")
    for name in args.sizes.split(","):
        n, w, h = SIZES[name]
        batch = n > 1
        x0, y0, rw, rh = raw_region(n, w, h, b32, b70)
        gen.manual_seed(n * 100003 + w)
        raw = torch.randint(0, 1024, (n, rh, rw), dtype=torch.int16, device="cuda", generator=gen).view(torch.uint16)
        il = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
        planar = torch.empty((n, 3, h, w), dtype=torch.uint8, device="cuda")
        il_t = torch.empty_like(il)
        planar_t = torch.empty_like(planar)
        planar_c = torch.empty_like(planar)
        if batch:
            b_in = HalideBuffer.from_torch(raw, (x0, y0, 0))
            b_il, b_pl, b_pl_t = (HalideBuffer.from_torch(il.permute(0, 3, 1, 2)), HalideBuffer.from_torch(planar),
                                  HalideBuffer.from_torch(planar_t))
            f_il, f_pl = filters.camera_pipe_interleaved_batch, filters.camera_pipe_batch
        else:
            b_in = HalideBuffer.from_torch(raw[0], (x0, y0))
            b_il, b_pl, b_pl_t = (HalideBuffer.from_torch(il[0].permute(2, 0, 1)), HalideBuffer.from_torch(planar[0]),
                                  HalideBuffer.from_torch(planar_t[0]))
            f_il, f_pl = filters.camera_pipe_interleaved, filters.camera_pipe
        frames_in = [HalideBuffer.from_torch(raw[k], (x0, y0)) for k in range(n)]
        frames_out = [HalideBuffer.from_torch(planar_c[k]) for k in range(n)]

        def arm_il():
            f_il(b_in, b32, b70, *PARAMS, b_il)

        def arm_planar():
            f_pl(b_in, b32, b70, *PARAMS, b_pl)

        def arm_torch():
            f_pl(b_in, b32, b70, *PARAMS, b_pl_t)
            il_t.copy_(planar_t.permute(0, 2, 3, 1))

        def arm_calls():
            for k in range(n):
                filters.camera_pipe(frames_in[k], b32, b70, *PARAMS, frames_out[k])

        arms = {"il": arm_il, "planar": arm_planar, "torch": arm_torch}
        if batch:
            arms["calls"] = arm_calls
        timing.warm_up(arms)
        arm_calls()  # (the calls arm's output is compared at every size)
        torch.cuda.synchronize()

        def check_outputs(when):
            assert torch.equal(il, planar.permute(0, 2, 3, 1)), f"il and planar arms differ at {name} {when}"
            assert torch.equal(il, il_t), f"il and torch arms differ at {name} {when}"
            assert torch.equal(planar, planar_c), f"planar arm and single calls differ at {name} {when}"

        check_outputs("after warm-up")
        iters, ms = timing.measure(arms, args.window_ms, args.rounds)
        check_outputs("after timing")
        med = {k: statistics.median(v) for k, v in ms.items()}
        gbs = {k: BYTES_PER_PIXEL * n * w * h / (v * 1e6) for k, v in med.items()}
        entry = {"size": name, "n": n, "w": w, "h": h, "raw": [rw, rh], "iters": iters, "ms_per_call": ms,
                 "median_ms": med, "gb_per_s": gbs, "outputs_identical": True,
                 "profile_ms": {k: profile(fn) for k, fn in arms.items()}}
        result["cases"].append(entry)
        line = ", ".join(f"{k} {med[k]:.4f} ms ({gbs[k]:.0f} GB/s)" for k in arms)
        line += f"; il/planar {med['il'] / med['planar']:.3f}, il/torch {med['il'] / med['torch']:.3f}"
        if batch:
            line += f", batch/calls {med['planar'] / med['calls']:.3f}"
        prof = entry["profile_ms"]
        line += "; profile " + "; ".join(f"{a}: " + ", ".join(f"{k} {v['ms']:.4f}" for k, v in prof[a].items()) for a in arms)
        print(f"{name} ({n} x {w} x {h}, raw {rw} x {rh}): {line}; outputs identical", flush=True)
        del raw, il, planar, il_t, planar_t, planar_c, b_in, b_il, b_pl, b_pl_t, frames_in, frames_out
        torch.cuda.empty_cache()
    timing.write_json(args.out_dir, "camera_pipe_burst_bench.json", result)


if __name__ == "__main__":
    main()
