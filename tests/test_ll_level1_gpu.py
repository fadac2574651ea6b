"""local_laplacian's level-1 kernel (levels == 8) at the boundaries of its work decomposition: units of 30 level-1
columns x 8 level-1 rows, dealt round-robin to the warps of one persistent block per SM, each warp copying its next
unit's frame rows into shared memory while it computes the current one.  Units whose column pairs are not 4-byte
aligned (odd x min, odd row strides) load their rows when they start instead; every layout must give the same bits."""
import numpy as np
import pytest

from util import run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
LEVELS, ALPHA, BETA = 8, 1.0 / 7.0, 1.0
STRIP, CHUNK = 30, 8  # level-1 columns / rows of one unit


def _level1_extent(out_lo, out_hi, in_lo, in_hi, levels=LEVELS):
    """Stored level-1 span of one axis (ll_geom.h compute_axis): the level-1 columns / rows the kernel computes."""
    o = [(out_lo, out_hi)]
    for _ in range(1, levels):
        o.append(((o[-1][0] - 1) >> 1, (o[-1][1] + 1) >> 1))
    g = o[-1]
    for j in range(levels - 2, 0, -1):
        g = (min(o[j][0], 2 * g[0] - 1), max(o[j][1], 2 * g[1] + 2))
    lo, hi = max(g[0], (in_lo - 2) >> 1), min(g[1], (in_hi + 2) >> 1)
    lo = min(lo, g[1])
    return hi - lo + 1 if hi >= lo else 1


def _units(w, h):
    nx, ny = _level1_extent(0, w - 1, 0, w - 1), _level1_extent(0, h - 1, 0, h - 1)
    return -(-nx // STRIP) * -(-ny // CHUNK), nx, ny


def _size_with_tail(rem, unit, start):
    """Smallest frame size >= start whose level-1 extent leaves a last unit of `rem` columns / rows."""
    n = start
    while _level1_extent(0, n - 1, 0, n - 1) % unit != rem % unit:
        n += 1
    return n


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("last_cols,last_rows", [(1, 1), (29, 7), (1, 7), (29, 1)])
def test_last_strip_and_chunk_widths(hb, oracle, last_cols, last_rows):
    """Last strip 1 or 29 columns wide, last chunk 1 or 7 rows tall; the frame has fewer units than the GPU has SMs."""
    w = _size_with_tail(last_cols, STRIP, 100)
    h = _size_with_tail(last_rows, CHUNK, 40)
    units, nx, ny = _units(w, h)
    assert nx % STRIP == last_cols % STRIP and ny % CHUNK == last_rows % CHUNK
    assert units < _sm_count()
    img = u16_frame((3, h, w), w * 100 + h)
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, BETA)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, BETA))


def _with_generic_level1(hb, fn):
    """fn() with level 1 (and the down-sweep) on the generic per-pixel kernels, which equal the oracle
    (test_local_laplacian_gpu.py); everything else stays on the default kernels."""
    l = hb.load_library()
    try:
        l.halide_b200_ll_force_generic(1)
        return fn()
    finally:
        l.halide_b200_ll_force_generic(0)


# Frames with several units per warp (more units than 64 warps per SM could hold), so a warp's sequence mixes
# prefetched units, units with edge lanes that load their own clamped columns, and the last short strip / chunk.
BIG_H, BIG_W = 2400, 4000


def test_many_units_per_warp(hb):
    units, _, _ = _units(BIG_W, BIG_H)
    assert units > 64 * _sm_count()
    img = u16_frame((3, BIG_H, BIG_W), 3)
    run = lambda: run_local_laplacian(hb, img, LEVELS, ALPHA, BETA)
    assert np.array_equal(run(), _with_generic_level1(hb, run))


@pytest.mark.parametrize("case", ["odd_x_min", "odd_row_stride", "y_offset_crop"])
def test_unaligned_layouts_and_crops(hb, case):
    """Odd x min and odd row strides turn the aligned pair loads (and the prefetch) off; a crop with a y offset moves
    the units' source rows inside the input.  Each must give the bits of the generic level-1 kernel."""
    kw = {}
    if case == "odd_x_min":
        img = u16_frame((3, BIG_H, BIG_W), 4)
        kw = dict(in_mins=(1, 0, 0), out_mins=(1, 0, 0))
    elif case == "odd_row_stride":
        img = u16_frame((3, BIG_H, BIG_W + 1), 5)[:, :, :BIG_W]
        assert img.strides[1] // img.itemsize % 2 == 1
    else:
        img = u16_frame((3, BIG_H, BIG_W), 6)
        kw = dict(out_shape=(3, BIG_H - 53, BIG_W - 40), in_mins=(0, 0, 0), out_mins=(16, 37, 0))
    run = lambda: run_local_laplacian(hb, img, LEVELS, ALPHA, BETA, **kw)
    assert np.array_equal(run(), _with_generic_level1(hb, run))


@pytest.mark.parametrize("beta", [1.0, 0.6])
def test_small_crop_with_offsets_matches_oracle(hb, oracle, beta):
    """Both kernel variants (beta == 1 and not) against the oracle on a crop with odd x and y offsets."""
    img = u16_frame((3, 150, 221), 11)
    kw = dict(out_shape=(3, 111, 160), in_mins=(0, 0, 0), out_mins=(13, 21, 0))
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, beta, **kw)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, beta, **kw))
