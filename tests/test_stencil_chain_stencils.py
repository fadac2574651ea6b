"""stencil_chain at depths other than 32, without a GPU: the two restatements of the generator agree at every number of
stencils, halide_b200_stencil_chain_stencils's argument checks (all of which return before any CUDA call), and the
input halo a row band needs (halide_b200.dist.halo_rows)."""
import ctypes

import numpy as np
import pytest

from util import u16_frame

ENTRY = "halide_b200_stencil_chain_stencils"


@pytest.mark.parametrize("s", [1, 2, 3, 4, 5, 7, 33, 100])
def test_restatements_agree(oracle, s):
    from oracle import np_restatement as npr
    img = u16_frame((29, 37), s)
    assert np.array_equal(oracle.stencil_chain(img, stencils=s), npr.stencil_chain(img, stencils=s))
    for kw in [dict(out_shape=(45, 52), in_mins=(3, -2), out_mins=(-10, -9)),     # output larger than the input
               dict(out_shape=(17, 21), in_mins=(-13, 7), out_mins=(-5, 11))]:    # odd mins, a crop
        a = oracle.stencil_chain(img, stencils=s, **kw)
        b = npr.stencil_chain(img, stencils=s, **kw)
        assert np.array_equal(a, b), kw


# ---- argument checks ------------------------------------------------------------------------------------------------

def _call(hb, bi, bo, stencils=5):
    l = hb.load_library()
    return getattr(l, ENTRY)(None if bi is None else bi.ptr, ctypes.c_int32(stencils), None if bo is None else bo.ptr)


def _buf(hb, shape, dtype=np.uint16, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def _empty(hb, dim, host_dirty=True):
    """An 8 x 10 buffer with dimension `dim`'s extent set to 0 (numpy gives empty arrays zero strides, which the
    inner-stride check would refuse first)."""
    b = _buf(hb, (8, 10), host_dirty=host_dirty)
    b.dims[dim].extent = 0
    return b


def _fails(hb, code, message, *args, **kw):
    from halide_b200.lib import capture_errors, last_error_message
    with capture_errors():
        assert _call(hb, *args, **kw) == code
        assert message in last_error_message(), last_error_message()


def test_null_buffers(hb):
    assert _call(hb, None, _buf(hb, (8, 10), host_dirty=False)) == -12
    assert _call(hb, _buf(hb, (8, 10)), None) == -12


def test_wrong_type(hb):
    assert _call(hb, _buf(hb, (8, 10), np.float32), _buf(hb, (8, 10), host_dirty=False)) == -3
    assert _call(hb, _buf(hb, (8, 10)), _buf(hb, (8, 10), np.uint8, host_dirty=False)) == -3


def test_wrong_dimensions(hb):
    assert _call(hb, _buf(hb, (3, 8, 10)), _buf(hb, (8, 10), host_dirty=False)) == -43
    assert _call(hb, _buf(hb, (8, 10)), _buf(hb, (10,), host_dirty=False)) == -43


def test_inner_stride_must_be_one(hb):
    bad = _buf(hb, (8, 10))
    bad.dims[0].stride = 2
    assert _call(hb, bad, _buf(hb, (8, 10), host_dirty=False)) == -8


@pytest.mark.parametrize("dim", [0, 1])
def test_empty_input(hb, dim):
    for s in (1, 32, 100):
        _fails(hb, -4, "Input buffer input is empty", _empty(hb, dim), _buf(hb, (8, 10), host_dirty=False), s)


@pytest.mark.parametrize("s,code", [(0, -9), (-1, -9), (101, -10)])
def test_stencils_out_of_range(hb, s, code):
    _fails(hb, code, f"Parameter stencils is {s} but must be in [1, 100]", _buf(hb, (8, 10)),
           _buf(hb, (8, 10), host_dirty=False), s)


def test_buffer_checks_come_before_the_range_check(hb):
    assert _call(hb, _buf(hb, (8, 10), np.float32), _buf(hb, (8, 10), host_dirty=False), 0) == -3
    _fails(hb, -4, "empty", _empty(hb, 1), _buf(hb, (8, 10), host_dirty=False), 101)


def test_bounds_query_fills_the_output_region(hb):
    """Every input access is clamped, so a query is answered with the output's region, whatever the depth."""
    for s in (0, 1, 33, 101):
        bi = hb.HalideBuffer.bounds_query(np.uint16, 2)
        bo = _buf(hb, (20, 30), mins=(5, -3), host_dirty=False)
        assert _call(hb, bi, bo, s) == 0
        assert bi.shape() == [(5, 30, 1), (-3, 20, 30)]
        assert bo.shape() == [(5, 30, 1), (-3, 20, 30)]


@pytest.mark.parametrize("dim", [0, 1])
def test_empty_output_does_nothing(hb, dim):
    for s in (0, 1, 32, 101):
        assert _call(hb, _buf(hb, (8, 10)), _empty(hb, dim, host_dirty=False), s) == 0
        assert _call(hb, _empty(hb, 1 - dim), _empty(hb, dim, host_dirty=False), s) == 0


def test_python_call_site_raises(hb):
    with pytest.raises(hb.HalideError) as e:
        hb.filters.stencil_chain_stencils(_buf(hb, (8, 10)), 101, _buf(hb, (8, 10), host_dirty=False))
    assert e.value.code == -10 and "Parameter stencils is 101" in e.value.message


# ---- halo of a row band -------------------------------------------------------------------------------------------

def test_halo_rows_default_is_unchanged():
    from halide_b200 import dist
    assert dist.halo_rows("stencil_chain") == (64, 64)
    assert dist.halo_rows("stencil_chain", stencils=32) == (64, 64)


@pytest.mark.parametrize("s", [1, 3, 33, 100])
def test_halo_rows_cover_a_band(oracle, s):
    """The oracle on a band's rows extended by halo_rows (clipped to the frame) equals the whole-frame oracle there."""
    from halide_b200 import dist
    up, down = dist.halo_rows("stencil_chain", stencils=s)
    assert (up, down) == (2 * s, 2 * s)
    h, w = 6 * s + 37, 23
    img = u16_frame((h, w), 500 + s)
    whole = oracle.stencil_chain(img, stencils=s)
    for lo, hi in [(0, h // 3), (h // 3 + 1, 2 * h // 3), (2 * h // 3 + 1, h - 1), (2 * s + 1, 2 * s + 1)]:
        a, b = max(0, lo - up), min(h - 1, hi + down)
        ext = np.ascontiguousarray(img[a:b + 1])
        band = oracle.stencil_chain(ext, out_shape=(hi - lo + 1, w), in_mins=(0, a), out_mins=(0, lo), stencils=s)
        assert np.array_equal(band, whole[lo:hi + 1]), (lo, hi)
