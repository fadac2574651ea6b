"""Argument checks of the 8-bit float-pipeline entry points, halide_b200_bilateral_grid_u8 (2-D (x, y) uint8 buffers) and
halide_b200_nl_means_u8 (3-D (x, y, c)).  They follow bilateral_grid and nl_means exactly, so most cases run the float
entry point on float32 buffers of the same shapes next to the 8-bit one and expect the same code from both.  Every case
returns before the library makes a CUDA call, so none needs a GPU."""
import ctypes

import numpy as np
import pytest

BG, NL = "bilateral_grid", "nl_means"
U8 = {BG: "halide_b200_bilateral_grid_u8", NL: "halide_b200_nl_means_u8"}
SHAPES = {BG: (8, 10), NL: (3, 8, 10)}  # numpy shapes: (y, x) and (c, y, x)


def _call(hb, filt, bi, bo, u8=True, r_sigma=0.1, patch=3, search=7, sigma=0.12):
    l = hb.load_library()
    bi = None if bi is None else bi.ptr
    bo = None if bo is None else bo.ptr
    if filt == BG:
        return getattr(l, U8[BG] if u8 else BG)(bi, ctypes.c_float(r_sigma), bo)
    return getattr(l, U8[NL] if u8 else NL)(bi, ctypes.c_int32(patch), ctypes.c_int32(search), ctypes.c_float(sigma), bo)


def _buf(hb, shape, dtype=np.uint8, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def _both(hb, filt, code, in_shape, out_shape, in_mins=None, out_mins=None, **kw):
    """The 8-bit entry point on uint8 buffers and the float one on float32 buffers of the same shapes both return code."""
    for u8, dt in ((True, np.uint8), (False, np.float32)):
        bi, bo = _buf(hb, in_shape, dt, in_mins), _buf(hb, out_shape, dt, out_mins, host_dirty=False)
        assert _call(hb, filt, bi, bo, u8, **kw) == code, ("8-bit" if u8 else "float", in_shape, out_shape, kw)


def _fails(hb, filt, code, message, **kw):
    """Both entry points fail with code and the same message."""
    from halide_b200.lib import capture_errors, last_error_message
    s = SHAPES[filt]
    for u8, dt in ((True, np.uint8), (False, np.float32)):
        with capture_errors():
            assert _call(hb, filt, _buf(hb, s, dt), _buf(hb, s, dt, host_dirty=False), u8, **kw) == code
            assert message in last_error_message(), last_error_message()


@pytest.fixture(params=[BG, NL])
def filt(request):
    return request.param


def test_null_buffers(hb, filt):
    s = SHAPES[filt]
    assert _call(hb, filt, None, _buf(hb, s, host_dirty=False)) == -12
    assert _call(hb, filt, _buf(hb, s), None) == -12


@pytest.mark.parametrize("tin,tout", [
    (np.float32, np.float32), (np.uint16, np.uint16), (np.int8, np.int8),   # other element types
    (np.uint8, np.float32), (np.float32, np.uint8),                          # mixed pairs
    (np.uint8, np.uint16), (np.uint16, np.uint8),
])
def test_wrong_type(hb, filt, tin, tout):
    s = SHAPES[filt]
    assert _call(hb, filt, _buf(hb, s, tin), _buf(hb, s, tout, host_dirty=False)) == -3


def test_float_entry_points_refuse_uint8(hb, filt):
    s = SHAPES[filt]
    assert _call(hb, filt, _buf(hb, s), _buf(hb, s, host_dirty=False), u8=False) == -3
    assert _call(hb, filt, _buf(hb, s), _buf(hb, s, np.float32, host_dirty=False), u8=False) == -3


def test_dimension_mixups(hb):
    _both(hb, BG, -43, (3, 8, 10), (8, 10))
    _both(hb, BG, -43, (8, 10), (3, 8, 10))
    _both(hb, BG, -43, (8, 10), (10,))
    _both(hb, NL, -43, (8, 10), (3, 8, 10))
    _both(hb, NL, -43, (3, 8, 10), (8, 10))
    _both(hb, NL, -43, (1, 3, 8, 10), (3, 8, 10))


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((8, 10), None, (9, 10), None),            # rows
    ((8, 10), None, (8, 11), None),            # columns
    ((8, 10), (1, 0), (8, 10), (0, 0)),        # shifted by one column
    ((8, 10), (0, -2), (8, 10), (0, -3)),      # shifted by one row
])
def test_bilateral_grid_output_not_covered_by_the_input(hb, in_shape, in_mins, out_shape, out_mins):
    _both(hb, BG, -4, in_shape, out_shape, in_mins, out_mins)


def test_bilateral_grid_larger_input_passes_the_checks(hb):
    """An input covering more than the output is accepted up to the r_sigma check, so coverage did not refuse it."""
    _both(hb, BG, -9, (12, 14), (8, 10), (-1, -2), (0, 0), r_sigma=0.0)


def test_nl_means_input_is_clamped_not_required(hb):
    """nl_means clamps every input access: an input smaller than, or away from, the output passes the checks (up to a
    parameter check, which returns before any CUDA call)."""
    _both(hb, NL, -9, (1, 2, 3), (3, 8, 10), patch=0)
    _both(hb, NL, -9, (4, 8, 10), (3, 8, 10), (100, -50, 0), None, patch=0)


@pytest.mark.parametrize("out_shape,out_mins", [((4, 8, 10), None), ((2, 8, 10), None), ((3, 8, 10), (0, 0, 1))])
def test_nl_means_output_channels_must_be_0_to_3(hb, out_shape, out_mins):
    _both(hb, NL, -8, (3, 8, 10), out_shape, None, out_mins)


def test_nl_means_channel_constraint_comes_before_the_parameter_checks(hb):
    _both(hb, NL, -8, (3, 8, 10), (4, 8, 10), patch=0, search=64)


def test_nl_means_empty_input(hb):
    for u8, dt in ((True, np.uint8), (False, np.float32)):
        backing = np.zeros(16, dt)
        for shape in [(10, 8, 0), (10, 0, 3), (0, 8, 3)]:  # (x, y, c), dense strides
            bi = hb.HalideBuffer(dt, shape)
            bi.buf.host = backing.ctypes.data
            bi.buf.flags = 1
            assert _call(hb, NL, bi, _buf(hb, (3, 8, 10), dt, host_dirty=False), u8) == -4


@pytest.mark.parametrize("r_sigma", [0.0, -0.5, float("nan")])
def test_bilateral_grid_r_sigma_not_positive(hb, r_sigma):
    _fails(hb, BG, -9, f"Parameter r_sigma is {r_sigma:g} but must be positive", r_sigma=r_sigma)


def test_bilateral_grid_201_bins_are_refused(hb):
    """r_sigma = 1/200 gives bins 0..200, one more than the largest grid; 1/199 is accepted up to the first CUDA call,
    which is not tested here."""
    r = float(np.float32(1.0) / np.float32(200))
    _fails(hb, BG, -9, "more than 200 intensity bins", r_sigma=r)


@pytest.mark.parametrize("patch,search,code", [
    (0, 7, -9), (3, 0, -9), (-1, 7, -9), (32, 7, -10), (3, 64, -10),
    (0, 64, -9), (32, 0, -9),     # a size below range is reported before one above it
])
def test_nl_means_sizes_out_of_range(hb, patch, search, code):
    _fails(hb, NL, code, f"patch_size {patch} / search_area {search} outside", patch=patch, search=search)


def test_empty_output_returns_zero(hb):
    """An empty output returns 0 before the parameter checks, as in the float entry points."""
    backing = {np.uint8: np.zeros(16, np.uint8), np.float32: np.zeros(16, np.float32)}
    for u8, dt in ((True, np.uint8), (False, np.float32)):
        for shape in [(10, 0), (0, 8)]:  # (x, y), dense strides
            bo = hb.HalideBuffer(dt, shape)
            bo.buf.host = backing[dt].ctypes.data
            assert _call(hb, BG, _buf(hb, (8, 10), dt), bo, u8) == 0
            assert _call(hb, BG, _buf(hb, (8, 10), dt), bo, u8, r_sigma=0.0) == 0
        for shape in [(10, 0, 3), (0, 8, 3)]:  # (x, y, c)
            bo = hb.HalideBuffer(dt, shape)
            bo.buf.host = backing[dt].ctypes.data
            assert _call(hb, NL, _buf(hb, (3, 8, 10), dt), bo, u8) == 0
            assert _call(hb, NL, _buf(hb, (3, 8, 10), dt), bo, u8, patch=0) == 0


def test_size_limits(hb):
    """The -5 / -6 limits of the other filters: per-dimension span and product of extents."""
    backing = np.zeros(16, np.uint8)  # (never read: the checks return before any copy)

    def raw(shape, strides):
        b = hb.HalideBuffer(np.uint8, shape, strides=strides)
        b.buf.host = backing.ctypes.data
        b.buf.flags = 1
        return b

    assert _call(hb, BG, raw((4, 4), (1, 1 << 30)), _buf(hb, (4, 4), host_dirty=False)) == -5
    assert _call(hb, BG, raw((1 << 16, 1 << 16), (1, 0)), _buf(hb, (4, 4), host_dirty=False)) == -6
    assert _call(hb, NL, raw((4, 4, 3), (1, 4, 1 << 30)), _buf(hb, (3, 4, 4), host_dirty=False)) == -5
    assert _call(hb, NL, raw((1 << 16, 1 << 16, 1), (1, 0, 0)), _buf(hb, (3, 4, 4), host_dirty=False)) == -6


def test_bounds_query_fills_the_input_region(hb):
    """A bounds query on the input proposes the float path's region with dense uint8 strides; the output is left as it
    was."""
    bi = hb.HalideBuffer.bounds_query(np.uint8, 2)
    bo = _buf(hb, (20, 30), mins=(5, -3), host_dirty=False)
    assert _call(hb, BG, bi, bo) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30)]
    assert bo.shape() == [(5, 30, 1), (-3, 20, 30)]
    bi = hb.HalideBuffer.bounds_query(np.uint8, 3)
    bo = _buf(hb, (3, 20, 30), mins=(5, -3, 0), host_dirty=False)
    assert _call(hb, NL, bi, bo) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600)]
    assert bo.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600)]


def test_bounds_query_matches_the_float_path(hb, filt):
    """Same output, same proposed region from the float and the 8-bit entry points (strides in elements)."""
    s = SHAPES[filt]
    mins = (7, -11) if filt == BG else (7, -11, 0)
    got = []
    for u8, dt in ((True, np.uint8), (False, np.float32)):
        bi = hb.HalideBuffer.bounds_query(dt, len(s))
        assert _call(hb, filt, bi, _buf(hb, s, dt, mins=mins, host_dirty=False), u8) == 0
        got.append(bi.shape())
    assert got[0] == got[1]


def test_bounds_query_comes_before_the_parameter_checks(hb):
    bi = hb.HalideBuffer.bounds_query(np.uint8, 2)
    assert _call(hb, BG, bi, _buf(hb, (4, 6), host_dirty=False), r_sigma=-1.0) == 0
    assert bi.shape() == [(0, 6, 1), (0, 4, 6)]
    bi = hb.HalideBuffer.bounds_query(np.uint8, 3)
    assert _call(hb, NL, bi, _buf(hb, (3, 4, 6), host_dirty=False), patch=0) == 0
    assert bi.shape() == [(0, 6, 1), (0, 4, 6), (0, 3, 24)]


def test_python_wrappers_raise(hb):
    from halide_b200 import HalideError, filters
    with pytest.raises(HalideError) as e:
        filters.bilateral_grid_u8(_buf(hb, (8, 10), np.float32), 0.1, _buf(hb, (8, 10), host_dirty=False))
    assert e.value.code == -3
    with pytest.raises(HalideError) as e:
        filters.nl_means_u8(_buf(hb, (3, 8, 10)), 0, 7, 0.12, _buf(hb, (3, 8, 10), host_dirty=False))
    assert e.value.code == -9
