"""local_laplacian's level-1 kernel walks the strips of one uint16 frame with warp pairs (8 pairs per block), and those
of 8-bit frames (and batches) with single warps (16 per block).  These frames end the grid's runs part-way through a
block's walkers, so walkers of the last block have no run while their block neighbours work (and, for pairs, both warps
of an idle pair skip the pair's barriers together).  Each element type must still give the oracle's bits: uint16 directly, 8-bit through the
uint16 filter composed with the element conversions, which also runs the other walker shape."""
import numpy as np
import pytest
import torch

from halide_b200.image_io import convert
from test_ll_level12_gpu import _chunks, _strips
from util import run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
LEVELS, ALPHA = 8, 1.0 / 7.0
WALKERS = {"u16": 8, "u8": 16}  # strip walkers per block (ll_kernels.cuh kL1Walkers)


def _runs(w, h, walkers, pairs):
    """Runs of a one-frame launch (local_laplacian.cu launch_level12_kernel), one block per SM."""
    s, xbase = _strips(w)
    ns = max((s[1][1] - xbase) // 28 + 1, (s[2][1] - xbase // 2) // 14 + 1)
    t, ybase = _chunks(h)
    nc = (max(t[1][1], 2 * t[2][1] + 2) - ybase) // 8 + 1
    npairs = torch.cuda.get_device_properties(0).multi_processor_count * walkers
    cost = {r: (ns * r + npairs - 1) // npairs * (4 * ((nc + r - 1) // r) + 1) for r in range(1, nc + 1)}
    nr = min(cost, key=lambda r: (cost[r], r))
    if pairs:
        nr = max(r for r in cost if cost[r] * 100 <= cost[nr] * 101)
    return ns * nr


@pytest.mark.parametrize("w,h", [(300, 150), (1500, 900)])
def test_partly_idle_last_block(hb, oracle, w, h):
    for kind, walkers in WALKERS.items():
        assert _runs(w, h, walkers, kind == "u16") % walkers != 0, kind
    img = u16_frame((3, h, w), w + h)
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, 1.0)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, 1.0))
    img8 = np.random.default_rng(w * h).integers(0, 256, (3, h, w), dtype=np.uint8)
    out8 = np.zeros_like(img8)
    bi, bo = hb.HalideBuffer.from_numpy(img8), hb.HalideBuffer.from_numpy(out8, host_dirty=False)
    hb.filters.local_laplacian_u8(bi, LEVELS, ALPHA, 1.0, bo)
    bo.copy_to_host()
    want = convert(run_local_laplacian(hb, convert(img8, np.uint16), LEVELS, ALPHA, 1.0), np.uint8)
    assert np.array_equal(out8, want)
