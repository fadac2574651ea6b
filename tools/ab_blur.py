"""A/B timing of halide_blur under its test hook (halide_b200_blur_force_general): python tools/ab_blur.py W H hook [hook ...]"""
import itertools, sys
import torch
import timing
import halide_b200
from halide_b200 import HalideBuffer, filters
W, H = int(sys.argv[1]), int(sys.argv[2])
hooks = [int(m) for m in sys.argv[3:]] or [0]
NS = 4
g = torch.Generator(device="cuda"); g.manual_seed(1)
ins = [torch.randint(-32768, 32768, (H + 2, W + 2), dtype=torch.int16, device="cuda", generator=g).view(torch.uint16) for _ in range(NS)]
outs = [torch.zeros((H, W), dtype=torch.uint16, device="cuda") for _ in range(NS)]
bi = [HalideBuffer.from_torch(t) for t in ins]; bo = [HalideBuffer.from_torch(t) for t in outs]
step = itertools.count()
def fn():  # each call takes the next frame pair
    i = next(step) % NS
    filters.halide_blur(bi[i], bo[i])
l = halide_b200.load_library()
ref = None
for m in hooks:
    l.halide_b200_blur_force_general(m)
    for _ in range(10): fn()
    torch.cuda.synchronize()
    us = timing.timed(fn, 100) * 1e3
    chk = int(outs[0].view(torch.int16).to(torch.int64).sum().item())
    if ref is None: ref = chk
    print(f"blur {W}x{H} hook {m}: {us:.2f} us/call  same_output={chk == ref}", flush=True)
l.halide_b200_blur_force_general(0)
