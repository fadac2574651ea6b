"""Argument checks of the camera_pipe burst and interleaved entry points (halide_b200_camera_pipe_batch, _interleaved and
_interleaved_batch).  Every case returns before the library makes a CUDA call, so none needs a GPU.  Raw buffers are numpy
arrays indexed [(n,) y, x]; planar outputs [(n,) c, y, x]; interleaved outputs [(n,) y, x, pitch] described as
(x, y, c[, n]) with strides (pitch, W*pitch, 1[, H*W*pitch])."""
import ctypes

import numpy as np
import pytest

BATCH, IL, ILB = ("halide_b200_camera_pipe_batch", "halide_b200_camera_pipe_interleaved",
                  "halide_b200_camera_pipe_interleaved_batch")
BURST = {BATCH, ILB}        # input (x, y, n), output (x, y, c, n)
INTERLEAVED = {IL, ILB}
H, W, N = 8, 10, 2          # output frame size and frames
# camera_pipe's raw region for that output at mins (0, 0): x [10, 32), y [6, 26)
RAW_X0, RAW_W, RAW_Y0, RAW_H = 10, 22, 6, 20
SCALARS = (ctypes.c_float(3700), ctypes.c_float(2.0), ctypes.c_float(50), ctypes.c_float(1.0), ctypes.c_int32(25),
           ctypes.c_int32(1023))
OUT_OF_BOUNDS, CONSTRAINT = -4, -8


def _ptr(b):
    return None if b is None else b.ptr


def _call(hb, fn, bi, bo, m32="dense", m70="dense"):
    l = hb.load_library()
    m = {"dense": lambda: hb.HalideBuffer.from_numpy(np.zeros((3, 4), np.float32)), None: lambda: None}
    b32 = m[m32]() if m32 in m else m32
    b70 = m[m70]() if m70 in m else m70
    return getattr(l, fn)(_ptr(bi), _ptr(b32), _ptr(b70), *SCALARS, _ptr(bo))


def raw(hb, fn, n=N, x0=RAW_X0, w=RAW_W, y0=RAW_Y0, h=RAW_H, n0=0, dtype=np.uint16):
    """A raw buffer (a burst of n frames for the burst entry points) over [x0, x0 + w) x [y0, y0 + h)."""
    if fn in BURST:
        return hb.HalideBuffer.from_numpy(np.zeros((n, h, w), dtype), (x0, y0, n0))
    return hb.HalideBuffer.from_numpy(np.zeros((h, w), dtype), (x0, y0))


def out(hb, fn, n=N, h=H, w=W, c=3, pitch=None, mins=None, interleaved=None, dtype=np.uint8):
    """The output for `fn`: interleaved (pixel pitch `pitch`, default c) or planar, with n frames for a burst."""
    il = fn in INTERLEAVED if interleaved is None else interleaved
    burst = fn in BURST
    # (an extent of 0 is a slice of an allocation of extent 1: numpy gives a zero-size array all-zero strides)
    full = lambda dims: np.zeros(tuple(max(d, 1) for d in dims), dtype)[tuple(slice(0, d) for d in dims)]  # noqa: E731
    if il:
        arr = full(((n,) if burst else ()) + (h, w, pitch or max(c, 1)))[..., :c]
        arr = arr.transpose((0, 3, 1, 2) if burst else (2, 0, 1))
    else:
        arr = full(((n,) if burst else ()) + (c, h, w))
    return hb.HalideBuffer.from_numpy(arr, mins, host_dirty=False)


@pytest.fixture(params=[BATCH, IL, ILB])
def fn(request):
    return request.param


def test_valid_arguments_reach_the_channel_check(hb, fn):
    """Buffers that pass every check up to the output's channel range: with channels [1, 4) the call fails there, the last
    check before the library touches the device."""
    for pitch in (None, 4):
        if pitch and fn not in INTERLEAVED:
            continue
        bo = out(hb, fn, c=3, pitch=pitch, mins=(0, 0, 1, 0) if fn in BURST else (0, 0, 1))
        with hb.lib.capture_errors() as err:
            assert _call(hb, fn, raw(hb, fn), bo) == OUT_OF_BOUNDS
        assert "channel range [1,4)" in err.msg


def test_null_buffers(hb, fn):
    assert _call(hb, fn, None, out(hb, fn)) == -12
    assert _call(hb, fn, raw(hb, fn), out(hb, fn), m32=None) == -12
    assert _call(hb, fn, raw(hb, fn), out(hb, fn), m70=None) == -12
    assert _call(hb, fn, raw(hb, fn), None) == -12


@pytest.mark.parametrize("which,dtype", [("input", np.uint8), ("input", np.int16), ("input", np.float32),
                                         ("output", np.uint16), ("output", np.int8), ("matrix", np.float64),
                                         ("matrix", np.int32)])
def test_wrong_types(hb, fn, which, dtype):
    if which == "input":
        assert _call(hb, fn, raw(hb, fn, dtype=dtype), out(hb, fn)) == -3
    elif which == "output":
        assert _call(hb, fn, raw(hb, fn), out(hb, fn, dtype=dtype)) == -3
    else:
        m = hb.HalideBuffer.from_numpy(np.zeros((3, 4), dtype))
        assert _call(hb, fn, raw(hb, fn), out(hb, fn), m32=m) == -3


def test_wrong_dimensions(hb):
    one = lambda a: hb.HalideBuffer.from_numpy(a)  # noqa: E731
    for fn in BURST:
        # a single raw frame, a single output frame
        assert _call(hb, fn, one(np.zeros((RAW_H, RAW_W), np.uint16)), out(hb, fn)) == -43
        assert _call(hb, fn, raw(hb, fn), out(hb, IL if fn == ILB else "camera_pipe", n=1)) == -43
    # the single-frame interleaved entry point takes neither a burst nor a 4-D output
    assert _call(hb, IL, raw(hb, BATCH), out(hb, IL)) == -43
    assert _call(hb, IL, raw(hb, IL), out(hb, ILB)) == -43
    # matrices are 2-D everywhere
    for fn in (BATCH, IL, ILB):
        assert _call(hb, fn, raw(hb, fn), out(hb, fn), m32=one(np.zeros((1, 3, 4), np.float32))) == -43


def _strided_out(hb, fn, strides, c=3):
    """An (x, y, c[, n]) uint8 output of W x H pixels with the given strides over a zero backing array large enough."""
    shape = (W, H, c, N) if fn in BURST else (W, H, c)
    backing = np.zeros(4096, np.uint8)
    b = hb.HalideBuffer(np.uint8, shape, strides=strides)
    b.buf.host = backing.ctypes.data
    b._keep = backing
    return b


@pytest.mark.parametrize("case,rule", [
    ("planar", "stride.2"),          # a planar output: channels not adjacent
    ("c_stride_2", "stride.2"),
    ("pitch_below_c", "stride.0"),   # pixel pitch 2 below 3 channels
    ("pitch_below_c4", "stride.0"),  # pixel pitch 3 below 4 channels
    ("y_stride_0", "stride.1"),      # rows must advance
    ("y_stride_neg", "stride.1"),
    ("n_stride_0", "stride.3"),      # frames must advance
    ("n_stride_neg", "stride.3"),
])
def test_interleaved_output_rules(hb, case, rule):
    c = 4 if case == "pitch_below_c4" else 3
    bad = {"planar": (1, W, W * H, 3 * W * H), "c_stride_2": (6, 60, 2, 480), "pitch_below_c": (2, 20, 1, 160),
           "pitch_below_c4": (3, 30, 1, 240), "y_stride_0": (3, 0, 1, 240), "y_stride_neg": (3, -30, 1, 240),
           "n_stride_0": (3, 30, 1, 0), "n_stride_neg": (3, 30, 1, -240)}[case]
    for fn in (IL, ILB):
        if fn == IL and rule == "stride.3":
            continue
        strides = bad if fn == ILB else bad[:3]
        with hb.lib.capture_errors() as err:
            assert _call(hb, fn, raw(hb, fn), _strided_out(hb, fn, strides, c=c)) == CONSTRAINT, fn
        assert f"processed.{rule}" in err.msg


def test_planar_entry_points_refuse_an_interleaved_output(hb):
    """The planar batch keeps camera_pipe's rule, dim[0].stride == 1; so does camera_pipe itself."""
    for fn in (BATCH, "camera_pipe"):
        bi = raw(hb, BATCH) if fn == BATCH else raw(hb, IL)
        bo = out(hb, BATCH, interleaved=True) if fn == BATCH else out(hb, IL)
        with hb.lib.capture_errors() as err:
            assert _call(hb, fn, bi, bo) == CONSTRAINT, fn
        assert "processed.stride.0" in err.msg


def test_raw_input_is_never_interleaved(hb, fn):
    """A raw buffer whose columns are not adjacent (every other sample of a wider row) is refused by every entry point."""
    rows = np.zeros(((N,) if fn in BURST else ()) + (RAW_H, 2 * RAW_W), np.uint16)
    bi = hb.HalideBuffer.from_numpy(rows[..., ::2], (RAW_X0, RAW_Y0, 0) if fn in BURST else (RAW_X0, RAW_Y0))
    with hb.lib.capture_errors() as err:
        assert _call(hb, fn, bi, out(hb, fn)) == CONSTRAINT
    assert "input.stride.0" in err.msg


@pytest.mark.parametrize("side", ["left", "right", "top", "bottom"])
def test_raw_region_one_short(hb, fn, side):
    x0, w, y0, h = RAW_X0, RAW_W, RAW_Y0, RAW_H
    if side == "left":
        x0, w = x0 + 1, w - 1
    elif side == "right":
        w -= 1
    elif side == "top":
        y0, h = y0 + 1, h - 1
    else:
        h -= 1
    with hb.lib.capture_errors() as err:
        assert _call(hb, fn, raw(hb, fn, x0=x0, w=w, y0=y0, h=h), out(hb, fn)) == OUT_OF_BOUNDS
    assert "Input buffer input" in err.msg and ("dimension 0" if side in ("left", "right") else "dimension 1") in err.msg


@pytest.mark.parametrize("in_n0,in_n,out_n0,out_n", [
    (0, 2, 0, 3),     # one frame too few
    (1, 3, 0, 3),     # the input starts a frame late
    (0, 3, 1, 3),     # the output's last frame past the input's
    (-5, 4, -6, 1),   # negative mins
])
def test_input_frames_must_cover_the_output_frames(hb, in_n0, in_n, out_n0, out_n):
    for fn in BURST:
        bo = out(hb, fn, n=out_n, mins=(0, 0, 0, out_n0))
        with hb.lib.capture_errors() as err:
            assert _call(hb, fn, raw(hb, fn, n=in_n, n0=in_n0), bo) == OUT_OF_BOUNDS
        assert "dimension 2" in err.msg


@pytest.mark.parametrize("c0,c", [(-1, 3), (-1, 1), (1, 3), (3, 1), (0, 4), (2, 2)])
def test_channels_outside_0_3(hb, fn, c0, c):
    pitch = max(c, 3) if fn in INTERLEAVED else None
    mins = (0, 0, c0, 0) if fn in BURST else (0, 0, c0)
    with hb.lib.capture_errors() as err:
        assert _call(hb, fn, raw(hb, fn), out(hb, fn, c=c, pitch=pitch, mins=mins)) == OUT_OF_BOUNDS
    assert f"channel range [{c0},{c0 + c})" in err.msg


def _camera_pipe_query(hb, ox, oy, w, h):
    """camera_pipe's own answer for the raw region of a (w, h) output at (ox, oy): [(min, extent, stride)] of x and y."""
    q = hb.HalideBuffer.bounds_query(np.uint16, 2)
    assert _call(hb, "camera_pipe", q, hb.HalideBuffer.from_numpy(np.zeros((3, h, w), np.uint8), (ox, oy, 0), host_dirty=False)) == 0
    return q.shape()


def test_bounds_query_of_the_raw_burst(hb):
    assert _camera_pipe_query(hb, 0, 0, W, H) == [(RAW_X0, RAW_W, 1), (RAW_Y0, RAW_H, RAW_W)]
    for ox, oy in [(0, 0), (5, -3), (-7, 4), (1001, -37)]:
        (x0, w, _), (y0, h, _) = _camera_pipe_query(hb, ox, oy, 30, 20)
        for fn in BURST:
            bi = hb.HalideBuffer.bounds_query(np.uint16, 3)
            assert _call(hb, fn, bi, out(hb, fn, n=4, h=20, w=30, mins=(ox, oy, 0, -2))) == 0
            assert bi.shape() == [(x0, w, 1), (y0, h, w), (-2, 4, w * h)], fn
        bi = hb.HalideBuffer.bounds_query(np.uint16, 2)
        assert _call(hb, IL, bi, out(hb, IL, h=20, w=30, mins=(ox, oy, 0))) == 0
        assert bi.shape() == [(x0, w, 1), (y0, h, w)]


def test_bounds_query_of_the_output(hb):
    """An output with mins and extents but no memory gets dense strides: interleaved (C, W*C, 1[, W*H*C]) for the
    interleaved entry points, planar for the batch; the raw input is left as it is."""
    cases = [(IL, (30, 20, 3), (5, -3, 0), [(5, 30, 3), (-3, 20, 90), (0, 3, 1)]),
             (IL, (30, 20, 2), (5, -3, 1), [(5, 30, 2), (-3, 20, 60), (1, 2, 1)]),
             (ILB, (30, 20, 3, 4), (5, -3, 0, -2), [(5, 30, 3), (-3, 20, 90), (0, 3, 1), (-2, 4, 1800)]),
             (BATCH, (30, 20, 3, 4), (5, -3, 0, -2), [(5, 30, 1), (-3, 20, 30), (0, 3, 600), (-2, 4, 1800)])]
    for fn, shape, mins, want in cases:
        bo = hb.HalideBuffer(np.uint8, shape, mins=mins)
        bi = raw(hb, fn)
        before = bi.shape()
        assert _call(hb, fn, bi, bo) == 0
        assert bo.shape() == want, fn
        assert bi.shape() == before


@pytest.mark.parametrize("empty", ["W", "H", "C", "N"])
def test_empty_output_returns_0_before_any_launch(hb, fn, empty):
    """An empty output returns 0, even over an input that covers nothing, and launches nothing."""
    if empty == "N" and fn not in BURST:
        return
    dims = dict(n=N, h=H, w=W, c=3)
    dims[empty.lower()] = 0
    bo = out(hb, fn, pitch=3, **dims)
    bi = raw(hb, fn, n=1, n0=7, x0=500, w=2, h=2)
    l = hb.load_library()
    n0 = l.halide_b200_kernel_launch_count()
    assert _call(hb, fn, bi, bo) == 0
    assert l.halide_b200_kernel_launch_count() == n0
    assert not bo.device_dirty
