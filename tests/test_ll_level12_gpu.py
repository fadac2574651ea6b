"""local_laplacian's level-1 kernel (levels == 8) also builds level 2: each warp walks a strip of 28 level-1 columns
(14 level-2 columns) down a run of 8-row chunks, carrying the last two level-1 rows of a chunk to the next, and a run
starts with a lead-in that recomputes the two level-1 rows above it.  These frames put the boundaries of that walk —
the last strip and chunk of either level, run starts, the level-2 columns left of level 1's array origin — where every
layout must still give the bits of the generic kernels (or of the oracle)."""
import numpy as np
import pytest

from util import run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
LEVELS, ALPHA = 8, 1.0 / 7.0
STRIP1, STRIP2, CHUNK = 28, 14, 8  # level-1 / level-2 columns of a strip, level-1 rows of a chunk


def _stored(out_lo, out_hi, in_lo, in_hi, levels=LEVELS):
    """Stored span of each level on one axis (ll_geom.h compute_axis)."""
    o = [(out_lo, out_hi)]
    for _ in range(1, levels):
        o.append(((o[-1][0] - 1) >> 1, (o[-1][1] + 1) >> 1))
    g = [None] * levels
    g[-1] = o[-1]
    for j in range(levels - 2, -1, -1):
        g[j] = (min(o[j][0], 2 * g[j + 1][0] - 1), max(o[j][1], 2 * g[j + 1][1] + 2))
    s, lo_b, hi_b = [], in_lo, in_hi
    for j in range(levels):
        if j:
            lo_b, hi_b = (lo_b - 2) >> 1, (hi_b + 2) >> 1
        lo = min(max(g[j][0], lo_b), g[j][1])
        s.append((lo, max(min(g[j][1], hi_b), lo)))
    return s


def _strips(n):
    """Stored spans of an n-wide frame and the first level-1 column of its first strip (xbase, local_laplacian.cu)."""
    s = _stored(0, n - 1, 0, n - 1)
    xo = s[1][0] & ~1
    d = xo - 2 * s[2][0]
    return s, xo - ((d + 3) & ~3 if d > 0 else 0)


def _chunks(n):
    """Stored spans of an n-tall frame and the first level-1 row of its first chunk (ybase, odd): the chunks cover the
    level-1 rows stored and the taps 2y-1 .. 2y+2 of the level-2 rows stored."""
    s = _stored(0, n - 1, 0, n - 1)
    lo = min(s[1][0], 2 * s[2][0] - 1)
    return s, lo if lo & 1 else lo - 1


def _last_strip_cols1(n):
    """Level-1 columns stored by the last strip that stores any (the kernel's level-1 store lanes, `writer`)."""
    s, xbase = _strips(n)
    return (s[1][1] - xbase) % STRIP1 + 1


def _last_strip_cols2(n):
    """Level-2 columns in the last strip of an n-wide frame."""
    s, xbase = _strips(n)
    return (s[2][1] - xbase // 2) % STRIP2 + 1


def _last_chunk_rows1(n):
    """Level-1 rows stored by the last chunk that stores any."""
    s, ybase = _chunks(n)
    return (s[1][1] - ybase) % CHUNK + 1


def _last_chunk_rows2(n):
    """Level-2 rows emitted by the last chunk of an n-tall frame (level-2 row y is emitted on level-1 row 2y+2)."""
    s, ybase = _chunks(n)
    hi = max(s[1][1], 2 * s[2][1] + 2)
    last = ybase + CHUNK * ((hi - ybase) // CHUNK)
    return sum(1 for y in range(s[2][0], s[2][1] + 1) if last <= 2 * y + 2 <= last + CHUNK - 1)


def _find(pred, start):
    n = start
    while not pred(n):
        n += 1
    return n


def _with_generic_down(hb, fn):
    """fn() with level 1 and the whole down-sweep on the generic per-pixel kernels (the reference the fast ones match)."""
    l = hb.load_library()
    try:
        l.halide_b200_ll_force_generic(1)
        return fn()
    finally:
        l.halide_b200_ll_force_generic(0)


@pytest.mark.parametrize("cols1,rows1", [(1, 1), (27, 7), (1, 7), (27, 1)])
def test_last_level1_strip_and_chunk(hb, oracle, cols1, rows1):
    """Last strip storing 1 or 27 level-1 columns, last chunk storing 1 or 7 level-1 rows."""
    w = _find(lambda n: _last_strip_cols1(n) == cols1, 100)
    h = _find(lambda n: _last_chunk_rows1(n) == rows1, 40)
    assert _last_strip_cols1(w) == cols1 and _last_chunk_rows1(h) == rows1
    img = u16_frame((3, h, w), w * 100 + h)
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, 1.0)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, 1.0))


@pytest.mark.parametrize("cols2,rows2", [(1, 1), (13, 2), (1, 3), (13, 1)])
def test_last_strip_and_chunk(hb, oracle, cols2, rows2):
    """Last strip with 1 or 13 level-2 columns, last chunk emitting 1, 2 or 3 level-2 rows; fewer runs than warps."""
    w = _find(lambda n: _last_strip_cols2(n) == cols2, 300)
    h = _find(lambda n: _last_chunk_rows2(n) == rows2, 150)
    img = u16_frame((3, h, w), w * 1000 + h)
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, 1.0)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, 1.0))


@pytest.mark.parametrize("shape", [(3, 4000, 6000), (3, 6000, 600)])
def test_many_chunks_per_run(hb, shape):
    """Frames with runs of many chunks (and a lead-in at every run start), against the generic kernels."""
    img = u16_frame(shape, shape[1] + shape[2])
    run = lambda: run_local_laplacian(hb, img, LEVELS, ALPHA, 1.0)
    assert np.array_equal(run(), _with_generic_down(hb, run))


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("case", ["odd_x_min", "odd_row_stride", "negative_mins", "odd_mins", "y_offset_crop"])
def test_layouts_and_crops(hb, case, beta):
    """Odd x min and odd row strides take the unaligned load path; crops move the level-2 columns and rows against the
    level-1 array origin, and a crop at an even x and odd y offset moves the strips' source rows inside the input.  Each
    must give the bits of the generic kernels, for both kernel variants."""
    h, w = 900, 1300
    kw = {}
    if case == "odd_x_min":
        img = u16_frame((3, h, w), 21)
        kw = dict(in_mins=(1, 0, 0), out_mins=(1, 0, 0))
    elif case == "odd_row_stride":
        img = u16_frame((3, h, w + 1), 22)[:, :, :w]
        assert img.strides[1] // img.itemsize % 2 == 1
    elif case == "negative_mins":
        img = u16_frame((3, h, w), 23)
        kw = dict(out_shape=(3, h - 31, w - 45), in_mins=(-20, -11, 0), out_mins=(-13, -3, 0))
    elif case == "odd_mins":
        img = u16_frame((3, h, w), 24)
        kw = dict(out_shape=(3, h - 40, w - 50), in_mins=(3, 5, 0), out_mins=(20, 17, 0))
    else:
        img = u16_frame((3, h, w), 25)
        kw = dict(out_shape=(3, h - 53, w - 40), in_mins=(0, 0, 0), out_mins=(16, 37, 0))
    run = lambda: run_local_laplacian(hb, img, LEVELS, ALPHA, beta, **kw)
    assert np.array_equal(run(), _with_generic_down(hb, run))


@pytest.mark.parametrize("beta", [1.0, 0.6])
def test_small_crop_with_offsets_matches_oracle(hb, oracle, beta):
    """Both kernel variants (beta == 1 and not) against the oracle on a crop with odd x and y offsets."""
    img = u16_frame((3, 150, 221), 11)
    kw = dict(out_shape=(3, 111, 160), in_mins=(0, 0, 0), out_mins=(13, 21, 0))
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, beta, **kw)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, beta, **kw))


@pytest.mark.parametrize("beta", [1.0, 0.6])
def test_level2_in_cooperative_tail(hb, oracle, beta):
    """A frame whose level 2 is small enough for the fused coarse launch: its down-sweep starts at level 3, and its
    up-sweep still produces level 2's outGPyramid."""
    img = u16_frame((3, 130, 210), 31)
    s = _stored(0, 209, 0, 209)
    t = _stored(0, 129, 0, 129)
    assert (s[2][1] - s[2][0] + 1) * (t[2][1] - t[2][0] + 1) <= 40 * 1024
    got = run_local_laplacian(hb, img, LEVELS, ALPHA, beta)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, beta))
