"""Times the row-sharded code path with a single rank (no neighbours): isolates the compute-side cost of sharding
(per-level launches, halo-aware input path) from the communication cost.  torchrun --nproc-per-node 1 tools/shard1_time.py"""
import itertools, sys
import torch, torch.distributed as td
import timing
torch.cuda.set_device(0)
td.init_process_group("nccl", device_id=torch.device("cuda", 0))
from halide_b200 import HalideBuffer, dist, filters
W, H = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (3840, 2160)
NS = 4 if W * H < 2e7 else 1
g = torch.Generator(device="cuda"); g.manual_seed(1)
ins = [torch.randint(-32768, 32768, (3, H, W), dtype=torch.int16, device="cuda", generator=g).view(torch.uint16) for _ in range(NS)]
outs = [torch.zeros((3, H, W), dtype=torch.uint16, device="cuda") for _ in range(NS)]
bi = [HalideBuffer.from_torch(t) for t in ins]; bo = [HalideBuffer.from_torch(t) for t in outs]
sh = dist.RowSharder(0, 1, W, H)
step = itertools.count()
def rotating(f):  # each call takes the next frame pair
    def call():
        i = next(step) % NS
        f(bi[i], 8, 1 / 7, 1.0, bo[i])
    return call
for name, fn in (("sharded(1 rank)", rotating(sh.local_laplacian)), ("single", rotating(filters.local_laplacian))):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    us = timing.timed(fn, 20) * 1e3
    rep = timing.profile(fn, 5)
    print(name, f"{us:.1f} us/step", {k: (c // 5, round(ms / 5 * 1e3, 1)) for k, (c, ms) in rep.items()})
td.destroy_process_group()
