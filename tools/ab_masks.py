"""A/B timing of local_laplacian under test-hook masks (halide_b200_ll_force_generic) on one GPU:
    python tools/ab_masks.py W H mask [mask ...]
Prints us/step (CUDA events over 20 calls, frame pairs rotating through > L2) and the per-kernel split for each mask."""
import itertools, sys
import torch
import timing
import halide_b200
from halide_b200 import HalideBuffer, filters
W, H = int(sys.argv[1]), int(sys.argv[2])
masks = [int(m) for m in sys.argv[3:]] or [0]
NS = 4 if W * H < 2e7 else 1
g = torch.Generator(device="cuda"); g.manual_seed(1)
ins = [torch.randint(-32768, 32768, (3, H, W), dtype=torch.int16, device="cuda", generator=g).view(torch.uint16) for _ in range(NS)]
outs = [torch.zeros((3, H, W), dtype=torch.uint16, device="cuda") for _ in range(NS)]
bi = [HalideBuffer.from_torch(t) for t in ins]; bo = [HalideBuffer.from_torch(t) for t in outs]
step = itertools.count()
def fn():  # each call takes the next frame pair
    i = next(step) % NS
    filters.local_laplacian(bi[i], 8, 1 / 7, 1.0, bo[i])
l = halide_b200.load_library()
ref = None
for m in masks:
    l.halide_b200_ll_force_generic(m)
    for _ in range(5): fn()
    torch.cuda.synchronize()
    us = timing.timed(fn, 20) * 1e3
    chk = int(outs[0].view(torch.int16).to(torch.int64).sum().item())
    if ref is None: ref = chk
    rep = timing.profile(fn, 5)
    print(f"{W}x{H} mask {m}: {us:.1f} us/step  same_output={chk == ref}",
          {k: (c // 5, round(ms / 5 * 1e3, 1)) for k, (c, ms) in rep.items()}, flush=True)
l.halide_b200_ll_force_generic(0)
