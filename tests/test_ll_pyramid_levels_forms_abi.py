"""Argument checks of the seven pyramid_levels forms of local_laplacian (batch, 8-bit and interleaved, in every
combination).  Every case returns before the library makes a CUDA call, so none needs a GPU.  Planar buffers are numpy
arrays indexed [(n,) c, y, x], interleaved ones [(n,) y, x, c]."""
import ctypes

import numpy as np
import pytest

P = "halide_b200_local_laplacian_pyramid_levels"
# suffix -> (element type, batch, interleaved)
FORMS = {
    "_batch": (np.uint16, True, False),
    "_u8": (np.uint8, False, False),
    "_u8_batch": (np.uint8, True, False),
    "_interleaved": (np.uint16, False, True),
    "_interleaved_batch": (np.uint16, True, True),
    "_u8_interleaved": (np.uint8, False, True),
    "_u8_interleaved_batch": (np.uint8, True, True),
}


def _call(hb, suffix, bi, bo, J=5, levels=8):
    l = hb.load_library()
    return getattr(l, P + suffix)(None if bi is None else bi.ptr, ctypes.c_int32(J), ctypes.c_int32(levels),
                                  ctypes.c_float(1 / 7), ctypes.c_float(1.0), None if bo is None else bo.ptr)


def _buf(hb, suffix, h=8, w=10, c=3, n=2, dtype=None, mins=None, host_dirty=True, interleaved=None):
    """A zero buffer of the form's type and layout (or those given): (x, y, c[, n])."""
    t, batch, il = FORMS[suffix]
    t = t if dtype is None else dtype
    il = il if interleaved is None else interleaved
    if il:
        arr = np.zeros(((n,) if batch else ()) + (h, w, c), t).transpose((0, 3, 1, 2) if batch else (2, 0, 1))
    else:
        arr = np.zeros(((n,) if batch else ()) + (c, h, w), t)
    return hb.HalideBuffer.from_numpy(arr, mins, host_dirty=host_dirty)


@pytest.fixture(params=list(FORMS))
def suffix(request):
    return request.param


def test_every_form_is_exported_and_wrapped(hb):
    """The library exports the seven forms, and halide_b200.local_laplacian_depth wraps exactly those."""
    import inspect
    l = hb.load_library()
    for s in FORMS:
        assert hasattr(l, P + s)
    m = hb.local_laplacian_depth
    public = {n for n, f in inspect.getmembers(m, inspect.isfunction) if f.__module__ == m.__name__ and not n.startswith("_")}
    assert public == {"local_laplacian_pyramid_levels" + s for s in FORMS}


def test_null_buffers(hb, suffix):
    assert _call(hb, suffix, None, _buf(hb, suffix, host_dirty=False)) == -12
    assert _call(hb, suffix, _buf(hb, suffix), None) == -12


def test_wrong_type(hb, suffix):
    t = FORMS[suffix][0]
    other = np.uint8 if t == np.uint16 else np.uint16
    for ti, to in [(other, other), (t, other), (other, t), (np.float32, np.float32)]:
        assert _call(hb, suffix, _buf(hb, suffix, dtype=ti), _buf(hb, suffix, dtype=to, host_dirty=False)) == -3, (ti, to)


def test_wrong_dimensions(hb, suffix):
    """A batch form given 3-D buffers, a one-frame form 4-D ones."""
    t, batch, il = FORMS[suffix]
    wrong = np.zeros((3, 8, 10) if batch else (2, 3, 8, 10), t)
    if il:
        wrong = np.ascontiguousarray(np.moveaxis(wrong, -3, -1))
        wrong = wrong.transpose((2, 0, 1) if batch else (0, 3, 1, 2))
    assert _call(hb, suffix, hb.HalideBuffer.from_numpy(wrong), _buf(hb, suffix, host_dirty=False)) == -43
    assert _call(hb, suffix, _buf(hb, suffix), hb.HalideBuffer.from_numpy(wrong, host_dirty=False)) == -43


def test_planar_buffer_refused_by_the_interleaved_forms(hb):
    for s, (t, batch, il) in FORMS.items():
        if not il:
            continue
        for which in ("input", "output"):
            bi = _buf(hb, s, interleaved=which != "input")
            bo = _buf(hb, s, interleaved=which != "output", host_dirty=False)
            with hb.lib.capture_errors() as err:
                assert _call(hb, s, bi, bo) == -8, (s, which)
            assert f"{which}.stride.2" in err.msg


def test_interleaved_buffer_refused_by_the_planar_forms(hb):
    for s, (t, batch, il) in FORMS.items():
        if il:
            continue
        with hb.lib.capture_errors() as err:
            assert _call(hb, s, _buf(hb, s, interleaved=True), _buf(hb, s, interleaved=True, host_dirty=False)) == -8, s
        assert "stride.0" in err.msg


@pytest.mark.parametrize("J,code", [(0, -9), (21, -10)])
def test_pyramid_levels_out_of_range(hb, suffix, J, code):
    with hb.lib.capture_errors() as err:
        assert _call(hb, suffix, _buf(hb, suffix), _buf(hb, suffix, host_dirty=False), J) == code
    assert f"Parameter pyramid_levels is {J} but must be in [1, 20]" in err.msg


def test_pyramid_levels_checked_after_the_buffers(hb, suffix):
    """A bad J behind a bad buffer reports the buffer; behind levels out of range, levels."""
    t = FORMS[suffix][0]
    other = np.uint8 if t == np.uint16 else np.uint16
    assert _call(hb, suffix, _buf(hb, suffix, dtype=other), _buf(hb, suffix, host_dirty=False), 0) == -3
    assert _call(hb, suffix, _buf(hb, suffix), _buf(hb, suffix, w=11, host_dirty=False), 21) == -4
    with hb.lib.capture_errors() as err:
        assert _call(hb, suffix, _buf(hb, suffix), _buf(hb, suffix, host_dirty=False), 0, levels=1) == -9
    assert "Parameter levels is 1" in err.msg


def test_bounds_query_matches_the_fixed_depth_form(hb, suffix):
    """The bounds query proposes what the fixed-depth counterpart proposes (dense interleaved strides for the interleaved
    forms), at any J, even one out of range."""
    t, batch, il = FORMS[suffix]
    l = hb.load_library()
    fixed = getattr(l, "halide_b200_local_laplacian" + suffix)
    dims = 4 if batch else 3
    mins = (5, -3, 0, -2)[:dims]
    want = hb.HalideBuffer.bounds_query(t, dims)
    bo = _buf(hb, suffix, h=20, w=30, n=4, mins=mins, host_dirty=False)
    assert fixed(want.ptr, ctypes.c_int32(8), ctypes.c_float(1 / 7), ctypes.c_float(1.0), bo.ptr) == 0
    for J in (1, 2, 8, 14, 20, 0):
        bi = hb.HalideBuffer.bounds_query(t, dims)
        assert _call(hb, suffix, bi, bo, J) == 0
        assert bi.shape() == want.shape(), J
    if il:
        assert want.shape()[:3] == [(5, 30, 3), (-3, 20, 90), (0, 3, 1)]
    else:
        assert want.shape()[:3] == [(5, 30, 1), (-3, 20, 30), (0, 3, 600)]
