"""bilateral_grid at cell sizes other than 8, without a GPU: the two restatements of the generator agree at every s_sigma,
halide_b200_bilateral_grid_s_sigma's argument checks (all of which return before any CUDA call), and the input halo a
row band needs (halide_b200.dist.halo_rows)."""
import ctypes

import numpy as np
import pytest

from util import f32_frame

ENTRY = "halide_b200_bilateral_grid_s_sigma"


@pytest.mark.parametrize("s", [1, 2, 3, 5, 8, 12, 16, 33])
def test_restatements_agree(oracle, s):
    from oracle import np_restatement as npr
    img = f32_frame((53, 77), s)
    a, b = oracle.bilateral_grid(img, 0.1, s_sigma=s), npr.bilateral_grid(img, 0.1, s_sigma=s)
    assert np.array_equal(a, b), float(np.abs(a - b).max())
    for r_sigma, kw in [(0.25, dict(out_shape=(30, 41), in_mins=(-13, -7), out_mins=(-9, -5))),
                        (0.1, dict(out_shape=(37, 50), in_mins=(-29, -31), out_mins=(-23, -17)))]:
        a = oracle.bilateral_grid(img, r_sigma, s_sigma=s, **kw)
        b = npr.bilateral_grid(img, r_sigma, s_sigma=s, **kw)
        assert np.array_equal(a, b), (kw, float(np.abs(a - b).max()))


# ---- argument checks ------------------------------------------------------------------------------------------------

def _call(hb, bi, bo, s_sigma=5, r_sigma=0.1):
    l = hb.load_library()
    return getattr(l, ENTRY)(None if bi is None else bi.ptr, ctypes.c_int32(s_sigma), ctypes.c_float(r_sigma),
                             None if bo is None else bo.ptr)


def _buf(hb, shape, dtype=np.float32, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def _fails(hb, code, message, *args, **kw):
    from halide_b200.lib import capture_errors, last_error_message
    with capture_errors():
        assert _call(hb, *args, **kw) == code
        assert message in last_error_message(), last_error_message()


def test_null_buffers(hb):
    assert _call(hb, None, _buf(hb, (8, 10), host_dirty=False)) == -12
    assert _call(hb, _buf(hb, (8, 10)), None) == -12


def test_wrong_type(hb):
    assert _call(hb, _buf(hb, (8, 10), np.uint16), _buf(hb, (8, 10), host_dirty=False)) == -3
    assert _call(hb, _buf(hb, (8, 10)), _buf(hb, (8, 10), np.int32, host_dirty=False)) == -3


def test_wrong_dimensions(hb):
    assert _call(hb, _buf(hb, (3, 8, 10)), _buf(hb, (8, 10), host_dirty=False)) == -43
    assert _call(hb, _buf(hb, (8, 10)), _buf(hb, (10,), host_dirty=False)) == -43


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((8, 10), None, (9, 10), None),            # rows
    ((8, 10), None, (8, 11), None),            # columns
    ((8, 10), (1, 0), (8, 10), (0, 0)),        # shifted by one column
    ((8, 10), (0, -2), (8, 10), (0, -3)),      # shifted by one row
])
def test_output_not_covered_by_the_input(hb, in_shape, in_mins, out_shape, out_mins):
    for s in (1, 8, 33):
        assert _call(hb, _buf(hb, in_shape, mins=in_mins), _buf(hb, out_shape, mins=out_mins, host_dirty=False), s) == -4


@pytest.mark.parametrize("s,code", [(0, -9), (-1, -9), (129, -10)])
def test_s_sigma_out_of_range(hb, s, code):
    _fails(hb, code, f"Parameter s_sigma is {s} but must be in [1, 128]", _buf(hb, (8, 10)),
           _buf(hb, (8, 10), host_dirty=False), s)
    # checked before r_sigma
    _fails(hb, code, "s_sigma", _buf(hb, (8, 10)), _buf(hb, (8, 10), host_dirty=False), s, -1.0)


@pytest.mark.parametrize("s", [1, 3, 8, 128])
@pytest.mark.parametrize("r_sigma", [0.0, -0.5])
def test_r_sigma_not_positive(hb, s, r_sigma):
    _fails(hb, -9, f"Parameter r_sigma is {r_sigma:g} but must be positive", _buf(hb, (8, 10)),
           _buf(hb, (8, 10), host_dirty=False), s, r_sigma)


@pytest.mark.parametrize("s", [1, 3, 8, 128])
def test_201_bins_are_refused(hb, s):
    """r_sigma = 1/200 gives bins 0..200: one more than the largest grid bilateral_grid accepts."""
    r = float(np.float32(1.0) / np.float32(200))
    assert int(np.float32(np.float32(1.0) / np.float32(r)) + np.float32(0.5)) == 200
    _fails(hb, -9, "more than 200 intensity bins", _buf(hb, (8, 10)), _buf(hb, (8, 10), host_dirty=False), s, r)


def test_bounds_query_fills_the_input_region(hb):
    bi = hb.HalideBuffer.bounds_query(np.float32, 2)
    bo = _buf(hb, (20, 30), mins=(5, -3), host_dirty=False)
    assert _call(hb, bi, bo, 13) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30)]
    assert bo.shape() == [(5, 30, 1), (-3, 20, 30)]


def test_bounds_query_comes_before_the_parameter_checks(hb):
    bi = hb.HalideBuffer.bounds_query(np.float32, 2)
    assert _call(hb, bi, _buf(hb, (4, 6), host_dirty=False), 0, -1.0) == 0
    assert bi.shape() == [(0, 6, 1), (0, 4, 6)]


# ---- slice index arithmetic ---------------------------------------------------------------------------------------

def test_magic_division_is_exact_over_the_tile_offsets():
    """bilateral_grid.cu: the slice computes floor(n / S) as (n * ceil(2^20 / S)) >> 20 for tile offsets
    n < S + 1024; exact for every S in [1, 128], and the product fits in 32 bits."""
    n = np.arange(0, 128 + 1024, dtype=np.uint64)
    for s in range(1, 129):
        mag = ((1 << 20) + s - 1) // s
        assert int((n * mag).max()) < 1 << 32
        assert np.array_equal((n * mag) >> 20, n // s), s


# ---- halo of a row band -------------------------------------------------------------------------------------------

def test_halo_rows_default_is_unchanged():
    from halide_b200 import dist
    assert dist.halo_rows("bilateral_grid") == (32, 32)
    assert dist.halo_rows("bilateral_grid", s_sigma=8) == (32, 32)


@pytest.mark.parametrize("s", [1, 3, 8, 16, 33])
def test_halo_rows_cover_a_band(oracle, s):
    """The oracle on a band's rows extended by halo_rows (clipped to the frame) equals the whole-frame oracle there."""
    from halide_b200 import dist
    up, down = dist.halo_rows("bilateral_grid", s_sigma=s)
    assert (up, down) == (4 * s, 4 * s)
    h, w = 10 * s + 37, 45
    img = f32_frame((h, w), 300 + s)
    whole = oracle.bilateral_grid(img, 0.1, s_sigma=s)
    for lo, hi in [(0, h // 3), (h // 3 + 1, 2 * h // 3), (2 * h // 3 + 1, h - 1), (s + 1, s + 1)]:
        a, b = max(0, lo - up), min(h - 1, hi + down)
        ext = np.ascontiguousarray(img[a:b + 1])
        band = oracle.bilateral_grid(ext, 0.1, out_shape=(hi - lo + 1, w), in_mins=(0, a), out_mins=(0, lo), s_sigma=s)
        assert np.array_equal(band, whole[lo:hi + 1]), (lo, hi)
