"""Argument checks of the interleaved local_laplacian entry points (uint16 / uint8, one frame / batch).  Every case returns
before the library makes a CUDA call, so none needs a GPU.  Buffers are numpy arrays indexed [(n,) y, x, c] described as
(x, y, c[, n]) with strides (C, W*C, 1[, H*W*C])."""
import ctypes

import numpy as np
import pytest

IL16, IL16B = "halide_b200_local_laplacian_interleaved", "halide_b200_local_laplacian_interleaved_batch"
IL8, IL8B = "halide_b200_local_laplacian_u8_interleaved", "halide_b200_local_laplacian_u8_interleaved_batch"
DTYPE = {IL16: np.uint16, IL16B: np.uint16, IL8: np.uint8, IL8B: np.uint8}
BATCH = {IL16B, IL8B}


def _call(hb, fn, bi, bo, levels=8):
    l = hb.load_library()
    return getattr(l, fn)(None if bi is None else bi.ptr, ctypes.c_int32(levels), ctypes.c_float(1 / 7),
                          ctypes.c_float(1.0), None if bo is None else bo.ptr)


def _il(hb, hwc, dtype, mins=None, host_dirty=True, channels=None):
    """An interleaved host buffer over a zero array of numpy shape [(n,) h, w, pitch]; `channels` < pitch describes the
    first channels only."""
    arr = np.zeros(hwc, dtype)
    if channels is not None:
        arr = arr[..., :channels]
    perm = (2, 0, 1) if arr.ndim == 3 else (0, 3, 1, 2)
    return hb.HalideBuffer.from_numpy(arr.transpose(perm), mins, host_dirty=host_dirty)


def _shape(fn, h=8, w=10, c=3):
    return (2, h, w, c) if fn in BATCH else (h, w, c)


@pytest.fixture(params=[IL16, IL16B, IL8, IL8B])
def fn(request):
    return request.param


def test_valid_layout_passes_the_checks(hb, fn):
    """A valid interleaved pair reaches the levels check (levels = 1 fails there, before any CUDA call)."""
    s, t = _shape(fn), DTYPE[fn]
    assert _call(hb, fn, _il(hb, s, t), _il(hb, s, t, host_dirty=False), levels=1) == -9
    # RGBA input, RGB output, and channels [0, 3) of an RGBA output
    s4 = _shape(fn, c=4)
    assert _call(hb, fn, _il(hb, s4, t), _il(hb, s, t, host_dirty=False), levels=1) == -9
    assert _call(hb, fn, _il(hb, s4, t), _il(hb, s4, t, host_dirty=False, channels=3), levels=1) == -9


def test_null_buffers(hb, fn):
    s, t = _shape(fn), DTYPE[fn]
    assert _call(hb, fn, None, _il(hb, s, t, host_dirty=False)) == -12
    assert _call(hb, fn, _il(hb, s, t), None) == -12


@pytest.mark.parametrize("other", [np.float32, np.int16, np.int8, "swap"])
@pytest.mark.parametrize("which", ["input", "output", "both"])
def test_wrong_or_mixed_type(hb, fn, other, which):
    s, t = _shape(fn), DTYPE[fn]
    if other == "swap":  # the other frame element type of the two accepted ones: a mixed uint8 / uint16 pair
        other = np.uint8 if t == np.uint16 else np.uint16
    ti = other if which in ("input", "both") else t
    to = other if which in ("output", "both") else t
    assert _call(hb, fn, _il(hb, s, ti), _il(hb, s, to, host_dirty=False)) == -3


def test_wrong_dimensions(hb):
    for fn in (IL16, IL8):
        t = DTYPE[fn]
        assert _call(hb, fn, _il(hb, (2, 8, 10, 3), t), _il(hb, (2, 8, 10, 3), t, host_dirty=False)) == -43
        assert _call(hb, fn, _il(hb, (8, 10, 3), t), _il(hb, (2, 8, 10, 3), t, host_dirty=False)) == -43
    for fn in (IL16B, IL8B):
        t = DTYPE[fn]
        assert _call(hb, fn, _il(hb, (8, 10, 3), t), _il(hb, (8, 10, 3), t, host_dirty=False)) == -43
        assert _call(hb, fn, _il(hb, (2, 8, 10, 3), t), _il(hb, (8, 10, 3), t, host_dirty=False)) == -43


def _planar(hb, fn, host_dirty=True):
    s = _shape(fn)
    planar = (s[0], s[3], s[1], s[2]) if fn in BATCH else (s[2], s[0], s[1])
    return hb.HalideBuffer.from_numpy(np.zeros(planar, DTYPE[fn]), host_dirty=host_dirty)


@pytest.mark.parametrize("which", ["input", "output"])
def test_planar_buffer_refused(hb, fn, which):
    s, t = _shape(fn), DTYPE[fn]
    bi = _planar(hb, fn) if which == "input" else _il(hb, s, t)
    bo = _planar(hb, fn, False) if which == "output" else _il(hb, s, t, host_dirty=False)
    with hb.lib.capture_errors() as err:
        assert _call(hb, fn, bi, bo) == -8
    assert f"{which}.stride.2" in err.msg


def _strided(hb, fn, strides, host_dirty=True, c=3):
    """(x, y, c[, n]) buffer of 8 x 10 pixels with the given strides over a zero backing array large enough for them."""
    shape = (10, 8, c, 2) if fn in BATCH else (10, 8, c)
    backing = np.zeros(4096, DTYPE[fn])
    b = hb.HalideBuffer(DTYPE[fn], shape, strides=strides)
    b.buf.host = backing.ctypes.data
    b._keep = backing
    if host_dirty:
        b.buf.flags = 1
    return b


@pytest.mark.parametrize("case,rule", [
    ("c_stride_2", "stride.2"),      # channels not adjacent (dim[2].stride != 1)
    ("pitch_below_c", "stride.0"),   # pixel pitch 2 below 3 channels
    ("pitch_below_c4", "stride.0"),  # pixel pitch 3 below 4 channels
    ("y_stride_0", "stride.1"),      # rows must advance
    ("y_stride_neg", "stride.1"),
])
@pytest.mark.parametrize("which", ["input", "output"])
def test_layout_rules(hb, fn, case, rule, which):
    batch = fn in BATCH
    ok = (3, 30, 1, 240) if batch else (3, 30, 1)
    c = 4 if case == "pitch_below_c4" else 3
    bad = {"c_stride_2": (6, 60, 2), "pitch_below_c": (2, 20, 1), "pitch_below_c4": (3, 30, 1),
           "y_stride_0": (3, 0, 1), "y_stride_neg": (3, -30, 1)}[case]
    if batch:
        bad = bad + (480,)
    if which == "input":
        bi, bo = _strided(hb, fn, bad, c=c), _strided(hb, fn, ok, host_dirty=False)
    else:  # (an RGBA input covers an output of 3 or 4 channels)
        bi, bo = _strided(hb, fn, (4, 40, 1, 320) if batch else (4, 40, 1), c=4), _strided(hb, fn, bad, host_dirty=False, c=c)
    with hb.lib.capture_errors() as err:
        assert _call(hb, fn, bi, bo) == -8
    assert f"{which}.{rule}" in err.msg


def test_batch_frame_stride_must_be_positive(hb):
    for fn in (IL16B, IL8B):
        bi, bo = _strided(hb, fn, (3, 30, 1, 0)), _strided(hb, fn, (3, 30, 1, 240), host_dirty=False)
        with hb.lib.capture_errors() as err:
            assert _call(hb, fn, bi, bo) == -8
        assert "input.stride.3" in err.msg


@pytest.mark.parametrize("in_hwc,in_mins,out_hwc,out_mins", [
    ((8, 10, 3), None, (9, 10, 3), None),          # rows
    ((8, 10, 3), None, (8, 11, 3), None),          # columns
    ((8, 10, 2), None, (8, 10, 3), None),          # channels
    ((8, 10, 3), (1, 0, 0), (8, 10, 3), None),     # columns shifted
    ((8, 10, 3), (0, -1, 0), (8, 10, 3), None),    # rows shifted
])
def test_output_not_covered_by_the_input(hb, in_hwc, in_mins, out_hwc, out_mins):
    for fn in (IL16, IL8):
        t = DTYPE[fn]
        assert _call(hb, fn, _il(hb, in_hwc, t, mins=in_mins), _il(hb, out_hwc, t, mins=out_mins, host_dirty=False)) == -4
    for fn in (IL16B, IL8B):
        t = DTYPE[fn]
        bm = None if in_mins is None else in_mins + (0,)
        assert _call(hb, fn, _il(hb, (2,) + in_hwc, t, mins=bm), _il(hb, (2,) + out_hwc, t, host_dirty=False)) == -4
        # one frame too few
        assert _call(hb, fn, _il(hb, (2, 8, 10, 3), t), _il(hb, (3, 8, 10, 3), t, host_dirty=False)) == -4


def test_planar_entry_points_refuse_interleaved_buffers(hb):
    """The planar entry points keep their rule: an interleaved buffer (stride.0 != 1) gets -8."""
    l = hb.load_library()
    args = (ctypes.c_int32(8), ctypes.c_float(1 / 7), ctypes.c_float(1.0))
    for name, t, batch in [("local_laplacian", np.uint16, False), ("halide_b200_local_laplacian_batch", np.uint16, True),
                           ("halide_b200_local_laplacian_u8", np.uint8, False),
                           ("halide_b200_local_laplacian_u8_batch", np.uint8, True)]:
        s = (2, 8, 10, 3) if batch else (8, 10, 3)
        bi, bo = _il(hb, s, t), _il(hb, s, t, host_dirty=False)
        with hb.lib.capture_errors() as err:
            assert getattr(l, name)(bi.ptr, *args, bo.ptr) == -8, name
        assert "stride.0" in err.msg


def test_bounds_query_proposes_interleaved_strides(hb):
    for fn in (IL16, IL8):
        bi = hb.HalideBuffer.bounds_query(DTYPE[fn], 3)
        bo = _il(hb, (20, 30, 3), DTYPE[fn], mins=(5, -3, 0), host_dirty=False)
        assert _call(hb, fn, bi, bo) == 0
        assert bi.shape() == [(5, 30, 3), (-3, 20, 90), (0, 3, 1)]
        assert bo.shape() == [(5, 30, 3), (-3, 20, 90), (0, 3, 1)]
        # RGBA-pitched output, channels [0, 3): the input is proposed dense over the 3 channels it must cover
        bi = hb.HalideBuffer.bounds_query(DTYPE[fn], 3)
        bo = _il(hb, (20, 30, 4), DTYPE[fn], host_dirty=False, channels=3)
        assert _call(hb, fn, bi, bo) == 0
        assert bi.shape() == [(0, 30, 3), (0, 20, 90), (0, 3, 1)]
    for fn in (IL16B, IL8B):
        bi = hb.HalideBuffer.bounds_query(DTYPE[fn], 4)
        bo = _il(hb, (4, 20, 30, 3), DTYPE[fn], mins=(5, -3, 0, -2), host_dirty=False)
        assert _call(hb, fn, bi, bo) == 0
        assert bi.shape() == [(5, 30, 3), (-3, 20, 90), (0, 3, 1), (-2, 4, 1800)]


def test_planar_bounds_query_unchanged(hb):
    bi = hb.HalideBuffer.bounds_query(np.uint16, 3)
    bo = hb.HalideBuffer.from_numpy(np.zeros((3, 20, 30), np.uint16), host_dirty=False)
    assert _call(hb, "local_laplacian", bi, bo) == 0
    assert bi.shape() == [(0, 30, 1), (0, 20, 30), (0, 3, 600)]
