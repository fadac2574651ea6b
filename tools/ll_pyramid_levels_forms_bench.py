"""The pyramid_levels forms of local_laplacian (batch, 8-bit, interleaved): what each costs per call as J moves, against
the uint16 planar halide_b200_local_laplacian_pyramid_levels with the torch conversions or permutes a caller would
otherwise put around it, against N single-frame calls for a batch, and against the fixed-depth form at J = 8.  Device-
resident RGB frames (smooth content + noise, seeded), levels 8, alpha 1/7, beta 1.

    python tools/ll_pyramid_levels_forms_bench.py OUT_DIR [--window-ms 100] [--rounds 3] [--J 1,3,8,11,14]
        [--configs 1080p,4k,16k,1080p_x8,4k_x8] [--kinds u8,u16,u8_il,u16_il]

Arms per (config, kind, J): `form` (the new entry point), `torch` (the uint16 planar call, frame by frame, with the
conversions / permutes in torch), `singles` (batches: the one-frame form of the same kind, frame by frame) and `fixed`
(J = 8: the fixed-depth entry point, whose output `form` must equal byte for byte).  Every arm is warmed up, then timed
with CUDA events over enough calls to fill the window, `rounds` times, the arms alternating; the median round is
reported.  At J = 1 the tone kernel's bandwidth is given at its algorithmic bytes (6 B/px for uint8 RGB, 12 for uint16).
The GPU's name, power limit and top SM clock are read in the same run.  Writes OUT_DIR/ll_pyramid_levels_forms_bench.json
and prints one line per (config, kind, J)."""
import statistics

import torch

import timing
from halide_b200 import HalideBuffer, filters, local_laplacian_depth

CONFIGS = {"1080p": (1920, 1080, 1), "4k": (3840, 2160, 1), "16k": (16384, 16384, 1), "1080p_x8": (1920, 1080, 8),
           "4k_x8": (3840, 2160, 8)}
LEVELS, ALPHA, BETA = 8, 1.0 / 7.0, 1.0


def u16(t):
    """int32 values in [0, 65535] as a uint16 tensor (int32 -> int16 wraps)."""
    return t.to(torch.int16).view(torch.uint16)


def widen(x8):
    return u16(x8.to(torch.int32) * 257)


def narrow(y16):
    return ((((y16.view(torch.int16).to(torch.int32) & 0xFFFF) + 128) * 255 + 255) >> 16).to(torch.uint8)


def frames(W, H, N, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    yy = torch.linspace(0, 1, H, device="cuda").view(H, 1)
    xx = torch.linspace(0, 1, W, device="cuda").view(1, W)
    out = []
    for n in range(N):
        base = torch.stack([0.5 + 0.4 * torch.sin(6.0 * xx + c + n) * torch.cos(5.0 * yy - c) for c in range(3)])
        out.append(((base + 0.03 * torch.rand((3, H, W), device="cuda", generator=gen)).clamp(0, 1) * 65535).to(torch.int32))
    return torch.stack(out)  # [N, 3, H, W] int32 in [0, 65535]


def il_view(t):
    """[.., 3, H, W] samples as a pixel-interleaved tensor of the same shape (channels_last storage)."""
    if t.dim() == 4:
        return t.view(torch.int16).contiguous(memory_format=torch.channels_last).view(t.dtype) if t.dtype == torch.uint16 \
            else t.contiguous(memory_format=torch.channels_last)
    hwc = (t.view(torch.int16) if t.dtype == torch.uint16 else t).permute(1, 2, 0).contiguous()
    hwc = hwc.view(t.dtype) if t.dtype == torch.uint16 else hwc
    return hwc.permute(2, 0, 1)


def planar(t):
    v = t.view(torch.int16) if t.dtype == torch.uint16 else t
    v = v.contiguous()
    return v.view(t.dtype) if t.dtype == torch.uint16 else v


def main():
    ap = timing.common_args(window_ms=100.0)
    ap.add_argument("--J", default="1,3,8,11,14")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--kinds", default="u8,u16,u8_il,u16_il")
    args = ap.parse_args()
    js = [int(v) for v in args.J.split(",")]
    timing.setup("ll_pyramid_levels_forms_bench")
    info = timing.gpu_info()
    print(f"gpu: {info}", flush=True)
    result = {"gpu": info, "levels": LEVELS, "alpha": ALPHA, "beta": BETA, "window_ms": args.window_ms, "rounds": args.rounds,
              "runs": []}
    for cname in args.configs.split(","):
        W, H, N = CONFIGS[cname]
        raw = frames(W, H, N, W + N)
        for kind in args.kinds.split(","):
            is8, il = kind.startswith("u8"), kind.endswith("_il")
            x = (((raw + 128) * 255 + 255) >> 16).to(torch.uint8) if is8 else u16(raw)
            batch = N > 1
            xs = x if batch else x[0]
            if il:
                xs = il_view(xs)
            y = torch.empty_like(xs)
            bx, by = HalideBuffer.from_torch(xs), HalideBuffer.from_torch(y)
            suffix = ("_u8" if is8 else "") + ("_interleaved" if il else "") + ("_batch" if batch else "")
            # (the uint16 planar frame: the one-frame entry point itself, whose arms are the same call)
            form_fn = getattr(local_laplacian_depth, "local_laplacian_pyramid_levels" + suffix) if suffix \
                else filters.local_laplacian_pyramid_levels
            fixed_fn = getattr(filters, "local_laplacian" + suffix)
            one_suffix = suffix.replace("_batch", "")
            one_fn = getattr(local_laplacian_depth, "local_laplacian_pyramid_levels" + one_suffix) if one_suffix \
                else filters.local_laplacian_pyramid_levels
            frames_in = [xs[n] for n in range(N)] if batch else [xs]
            frames_out = [y[n] for n in range(N)] if batch else [y]
            one_bufs = [(HalideBuffer.from_torch(a), HalideBuffer.from_torch(b)) for a, b in zip(frames_in, frames_out)]
            # the torch route: a planar uint16 copy of each frame, the uint16 planar call, the result converted back
            t_in = torch.empty((3, H, W), dtype=torch.uint16, device="cuda")
            t_out = torch.empty_like(t_in)
            b_tin, b_tout = HalideBuffer.from_torch(t_in), HalideBuffer.from_torch(t_out)
            y_ref = torch.empty_like(xs)

            def torch_route(J):
                for n in range(N):
                    f = frames_in[n]
                    src = widen(f) if is8 else f
                    t_in.view(torch.int16).copy_(planar(src).view(torch.int16))
                    filters.local_laplacian_pyramid_levels(b_tin, J, LEVELS, ALPHA, BETA, b_tout)
                    res = narrow(t_out) if is8 else t_out
                    dst = y_ref[n] if batch else y_ref
                    (dst.view(torch.int16) if not is8 else dst).copy_(res.view(torch.int16) if not is8 else res)

            for J in js:
                arms = {"form": lambda J=J: form_fn(bx, J, LEVELS, ALPHA, BETA, by), "torch": lambda J=J: torch_route(J)}
                if batch:
                    arms["singles"] = lambda J=J: [one_fn(a, J, LEVELS, ALPHA, BETA, b) for a, b in one_bufs]
                if J == 8:
                    y8 = torch.empty_like(xs)
                    b8 = HalideBuffer.from_torch(y8)
                    arms["fixed"] = lambda: fixed_fn(bx, LEVELS, ALPHA, BETA, b8)
                timing.warm_up(arms)
                eq = bool(timing.same(y, y_ref))
                assert eq, f"{cname} {kind} J {J}: the form differs from the uint16 planar call"
                if J == 8:
                    assert timing.same(y, y8), f"{cname} {kind}: J = 8 differs from the fixed-depth form"
                iters, ms = timing.measure(arms, args.window_ms, args.rounds)
                prof = {k: {"launches": c, "ms": t} for k, (c, t) in sorted(timing.profile(arms["form"]).items())}
                entry = {"config": cname, "kind": kind, "J": J, "iters": iters,
                         "median_ms": {k: statistics.median(v) for k, v in ms.items()}, "ms": ms, "profile_ms": prof}
                if "ll_tone" in prof:
                    bpp = 6 if is8 else 12
                    t = prof["ll_tone"]["ms"] * 1e-3
                    entry["tone_tb_per_s"] = bpp * W * H * N / t / 1e12
                result["runs"].append(entry)
                med = entry["median_ms"]
                extra = f", tone {entry['tone_tb_per_s']:.2f} TB/s" if "tone_tb_per_s" in entry else ""
                print(f"{cname} {kind} J {J}: " + ", ".join(f"{k} {v:.3f} ms" for k, v in med.items()) + extra, flush=True)
            del bx, by, x, xs, y, y_ref, one_bufs, b_tin, b_tout, t_in, t_out
            torch.cuda.empty_cache()
        del raw
    timing.write_json(args.out_dir, "ll_pyramid_levels_forms_bench.json", result)


if __name__ == "__main__":
    main()
