"""local_laplacian's fast final kernel (levels == 8, up to 3 channels) computes outGPyramid[1] for its own 60 x 32 tile
from inGPyramid[1], the gPyramid[1] tile it stages anyway and an 11 x 18 tile of level 2, instead of reading an array
that a level-1 up-sweep launch wrote.  These tests check that no such launch runs any more, and that the tile positions
at frame edges, crops and tile seams — where a position is clamped into level 1's outGPyramid region — give the
oracle's bits on every final-kernel path (TMA frame tile, aligned loads, general layout) and in batches."""
import numpy as np
import pytest

from util import run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
LEVELS, ALPHA = 8, 1.0 / 7.0
TILE_W, TILE_H = 60, 32  # fine pixels of a final-kernel tile
# final-kernel paths: TMA frame tile (when the layout allows it), aligned loads without TMA, general layout
FINAL_MASKS = [0, 64, 16 | 64]


def _span(out_lo, out_hi, in_lo, in_hi, j):
    """Stored span of level j on one axis (ll_geom.h compute_axis)."""
    o = [(out_lo, out_hi)]
    for _ in range(1, LEVELS):
        o.append(((o[-1][0] - 1) >> 1, (o[-1][1] + 1) >> 1))
    g = [None] * LEVELS
    g[-1] = o[-1]
    for k in range(LEVELS - 2, -1, -1):
        g[k] = (min(o[k][0], 2 * g[k + 1][0] - 1), max(o[k][1], 2 * g[k + 1][1] + 2))
    lo_b, hi_b = in_lo, in_hi
    for k in range(1, j + 1):
        lo_b, hi_b = (lo_b - 2) >> 1, (hi_b + 2) >> 1
    lo = min(max(g[j][0], lo_b), g[j][1])
    return lo, max(min(g[j][1], hi_b), lo)


def _up_sweep_levels(w, h):
    """Levels whose up-sweep has a launch of its own on one GPU: j0 .. 1, j0 = the last level above the cooperative
    tail (levels of at most 40 K stored pixels, local_laplacian.cu run_coarse_sweep)."""
    j0 = LEVELS - 1
    while j0 > 1:
        sx, sy = _span(0, w - 1, 0, w - 1, j0), _span(0, h - 1, 0, h - 1, j0)
        if (sx[1] - sx[0] + 1) * (sy[1] - sy[0] + 1) > 40 * 1024:
            break
        j0 -= 1
    return j0


def _with_mask(hb, mask, fn):
    l = hb.load_library()
    try:
        l.halide_b200_ll_force_generic(mask)
        return fn()
    finally:
        l.halide_b200_ll_force_generic(0)


def _profiled(hb, img):
    """{kernel: launches} of one call (after a warm-up call: the remap table is built once)."""
    lib = hb.lib
    run_local_laplacian(hb, img, LEVELS, ALPHA, 1.0)
    lib.profile(True)
    lib.profile_reset()
    try:
        run_local_laplacian(hb, img, LEVELS, ALPHA, 1.0)
        return {k: v[0] for k, v in lib.profile_report().items()}
    finally:
        lib.profile(False)
        lib.profile_reset()


@pytest.mark.parametrize("w,h", [(3840, 2160), (1920, 1080)])
def test_no_level1_up_sweep_launch(hb, w, h):
    """The fast final kernel leaves level 1's up-sweep out of the launch sequence; with the generic final kernel
    (hook bit 4) level 1 still has its own up-sweep launch, and a call has one launch more."""
    img = u16_frame((3, h, w), w + h)
    j0 = _up_sweep_levels(w, h)
    assert j0 >= 2
    fused = _profiled(hb, img)
    generic = _with_mask(hb, 4, lambda: _profiled(hb, img))
    assert fused.get("ll_up2", 0) == j0 - 1, fused
    assert generic.get("ll_up2", 0) == j0, generic
    assert fused.get("ll_final2") == 1 and "ll_final2" not in generic
    assert sum(generic.values()) - sum(fused.values()) == 1, (fused, generic)


def _oracle_and_paths(hb, oracle, img, beta, **kw):
    want = oracle.local_laplacian(img, LEVELS, ALPHA, beta, **kw)
    for mask in FINAL_MASKS:
        got = _with_mask(hb, mask, lambda: run_local_laplacian(hb, img, LEVELS, ALPHA, beta, **kw))
        bad = np.argwhere(got != want)
        assert bad.size == 0, f"mask {mask}: {len(bad)} mismatches, first at (c,y,x)={bad[0]}"


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("wide_input", [False, True])
@pytest.mark.parametrize("last_rows", [2, 30])
@pytest.mark.parametrize("last_cols", [2, 30, 58])
def test_last_tile_widths_and_heights(hb, oracle, last_cols, last_rows, wide_input, beta):
    """Frames whose last tile holds 2, 30 or 58 columns and 2 or 30 rows.  With wide_input the input has rows of a
    multiple of 8 columns and one row more than the output (so the TMA frame tile can be used and the frame's edge is
    not the output's); otherwise input and output are the same frame."""
    w, h = 2 * TILE_W + last_cols, 2 * TILE_H + last_rows
    if wide_input:
        img = u16_frame((3, h + 1, (w + 7) & ~7), w * 7 + h)
        _oracle_and_paths(hb, oracle, img, beta, out_shape=(3, h, w))
    else:
        img = u16_frame((3, h, w), w * 7 + h)
        _oracle_and_paths(hb, oracle, img, beta)


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("in_mins,out_mins", [
    ((-20, -11, 0), (-13, -3, 0)),   # negative mins, odd output mins
    ((3, 5, 0), (21, 17, 0)),        # odd input and output mins
    ((-7, -9, 0), (-7, -9, 0)),      # output at the input's odd negative corner
    ((0, 0, 0), (16, 37, 0)),        # even x / odd y offset (the TMA box start stays 16-byte aligned)
    ((-20, -11, 0), (-12, -3, 0)),   # negative mins, even x offset of 8 columns: TMA with an odd negative y min
])
def test_crops_with_odd_and_negative_mins(hb, oracle, in_mins, out_mins, beta):
    """Crops whose level-1 outGPyramid region starts at another column / row than the stored level-1 planes, so a tile
    position clamped into the former is not the column the staged planes hold there."""
    h, w = 170, 256
    img = u16_frame((3, h, w), 100 + in_mins[0] + 3 * out_mins[1])
    out_shape = (3, h - 40 - max(0, out_mins[1] - in_mins[1]), w - 50 - max(0, out_mins[0] - in_mins[0]))
    _oracle_and_paths(hb, oracle, img, beta, out_shape=out_shape, in_mins=in_mins, out_mins=out_mins)


def _strided(a, row_pad, frame_pad):
    n, c, h, w = a.shape
    pitch = w + row_pad
    fs = c * h * pitch + frame_pad
    flat = np.zeros(n * fs, np.uint16)
    v = np.lib.stride_tricks.as_strided(flat, shape=a.shape, strides=(2 * fs, 2 * h * pitch, 2 * pitch, 2))
    v[...] = a
    return v


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("row_pad,frame_pad", [(0, 0), (0, 2), (3, 5)])
def test_batches_match_single_calls(hb, row_pad, frame_pad, beta):
    """N = 3 frames with frame strides that meet TMA's 16-byte rules (4-D frame tile), that are even but not 16-byte
    multiples (aligned loads) and that are odd (general layout), against one call per frame."""
    n, h, w = 3, 130, 3 * TILE_W + 4
    a = np.stack([u16_frame((3, h, w), 500 + k) for k in range(n)])
    want = np.stack([run_local_laplacian(hb, np.ascontiguousarray(a[k]), LEVELS, ALPHA, beta) for k in range(n)])
    inp = _strided(a, row_pad, frame_pad)
    out = _strided(np.zeros_like(a), row_pad, frame_pad)
    bi = hb.HalideBuffer.from_numpy(inp)
    bo = hb.HalideBuffer.from_numpy(out, host_dirty=False)
    hb.filters.local_laplacian_batch(bi, LEVELS, ALPHA, beta, bo)
    bo.copy_to_host()
    for k in range(n):
        assert np.array_equal(out[k], want[k]), f"frame {k}"
