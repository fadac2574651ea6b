"""Argument checks of the batch bilateral_grid entry points (float32, uint8, and float32 at any cell size): each returns
the code its one-frame counterpart returns on one-frame buffers of the same x/y shape, checks that the input's frames
cover the output's, answers bounds queries with the output's (x, y, n) region, and returns 0 on an empty clip.  Every
case returns before the library makes a CUDA call, so none needs a GPU.

Buffers are numpy arrays: a frame is (y, x), a clip (n, y, x), described as (x, y[, n])."""
import ctypes

import numpy as np
import pytest

# (batch symbol, one-frame symbol, element type, takes s_sigma)
ENTRIES = [
    ("halide_b200_bilateral_grid_batch", "bilateral_grid", np.float32, False),
    ("halide_b200_bilateral_grid_u8_batch", "halide_b200_bilateral_grid_u8", np.uint8, False),
    ("halide_b200_bilateral_grid_s_sigma_batch", "halide_b200_bilateral_grid_s_sigma", np.float32, True),
]
IDS = [e[0][len("halide_b200_"):] for e in ENTRIES]
H, W, N = 8, 10, 3
INT32_MIN = -(1 << 31)


@pytest.fixture(params=ENTRIES, ids=IDS)
def entry(request):
    return request.param


def call(hb, sym, takes_s, bi, bo, s_sigma=5, r_sigma=0.1):
    fn = getattr(hb.load_library(), sym)
    args = [None if bi is None else bi.ptr]
    if takes_s:
        args.append(ctypes.c_int32(s_sigma))
    args += [ctypes.c_float(r_sigma), None if bo is None else bo.ptr]
    return fn(*args)


def buf(hb, shape, dtype, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def pair(hb, dtype, batch, in_shape=(H, W), out_shape=(H, W), in_mins=None, out_mins=None, out_dtype=None):
    """Input and output buffers of x/y shapes (h, w): one frame, or N frames (frame mins 0) for a batch."""
    n = (N,) if batch else ()
    nm = (0,) if batch else ()
    return (buf(hb, n + in_shape, dtype, None if in_mins is None else tuple(in_mins) + nm),
            buf(hb, n + out_shape, dtype if out_dtype is None else out_dtype,
                None if out_mins is None else tuple(out_mins) + nm, host_dirty=False))


def same_code(hb, entry, want, make, **kw):
    """make(batch) -> (input, output): the batch entry point on the clip and its one-frame counterpart on the frame both
    return `want`."""
    sym, one, dt, takes_s = entry
    got_batch = call(hb, sym, takes_s, *make(True), **kw)
    got_one = call(hb, one, takes_s, *make(False), **kw)
    assert (got_batch, got_one) == (want, want), (sym, kw)


def raw(hb, dt, shape, strides, mins=None, host_dirty=True):
    """A buffer of (x, y[, n]) extents and strides over a zeroed backing store large enough for any of them."""
    b = hb.HalideBuffer(dt, shape, strides=strides, mins=mins)
    b._keep = np.zeros(1 << 16, dt)  # (never read: the checks return before any copy)
    b.buf.host = b._keep.ctypes.data
    b.set_host_dirty(host_dirty)
    return b


def test_null_buffers(hb, entry):
    dt = entry[2]
    same_code(hb, entry, -12, lambda b: (None, pair(hb, dt, b)[1]))
    same_code(hb, entry, -12, lambda b: (pair(hb, dt, b)[0], None))


@pytest.mark.parametrize("other", [np.uint16, np.int8, np.float64])
def test_wrong_and_mixed_types(hb, entry, other):
    dt = entry[2]
    wrong = np.uint8 if dt == np.float32 else np.float32  # the float entry points refuse uint8 and the reverse
    for t in (wrong, other):
        same_code(hb, entry, -3, lambda b: pair(hb, t, b))
        same_code(hb, entry, -3, lambda b: pair(hb, dt, b, out_dtype=t))
        same_code(hb, entry, -3, lambda b: (pair(hb, t, b)[0], pair(hb, dt, b)[1]))


def test_wrong_dimensions(hb, entry):
    sym, one, dt, takes_s = entry
    clip_i, clip_o = pair(hb, dt, True)
    frame_i, frame_o = pair(hb, dt, False)
    four_i, four_o = buf(hb, (2, N, H, W), dt), buf(hb, (2, N, H, W), dt, host_dirty=False)
    for bi, bo in [(frame_i, clip_o), (clip_i, frame_o), (frame_i, frame_o), (four_i, clip_o), (clip_i, four_o)]:
        assert call(hb, sym, takes_s, bi, bo) == -43
    # and the one-frame entry points keep refusing clips
    assert call(hb, one, takes_s, clip_i, frame_o) == -43
    assert call(hb, one, takes_s, frame_i, clip_o) == -43


def test_x_stride_not_one(hb, entry):
    dt = entry[2]

    def make(batch, which):
        shape = (W, H) + ((N,) if batch else ())
        dense = (1, W) + ((W * H,) if batch else ())
        bad = (2, 2 * W) + ((2 * W * H,) if batch else ())
        return (raw(hb, dt, shape, bad if which == 0 else dense),
                raw(hb, dt, shape, bad if which == 1 else dense, host_dirty=False))

    same_code(hb, entry, -8, lambda b: make(b, 0))
    same_code(hb, entry, -8, lambda b: make(b, 1))


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((8, 10), None, (9, 10), None),            # rows
    ((8, 10), None, (8, 11), None),            # columns
    ((8, 10), (1, 0), (8, 10), (0, 0)),        # shifted by one column
    ((8, 10), (0, -2), (8, 10), (0, -3)),      # shifted by one row
])
def test_output_x_y_not_covered_by_the_input(hb, entry, in_shape, in_mins, out_shape, out_mins):
    dt = entry[2]
    for s in (1, 8, 33):
        same_code(hb, entry, -4, lambda b: pair(hb, dt, b, in_shape, out_shape, in_mins, out_mins), s_sigma=s)


@pytest.mark.parametrize("s,code", [(0, -9), (129, -10), (INT32_MIN, -9)])
def test_s_sigma_out_of_range(hb, entry, s, code):
    from halide_b200.lib import capture_errors, last_error_message
    if not entry[3]:
        pytest.skip("entry point runs s_sigma = 8")
    with capture_errors():
        same_code(hb, entry, code, lambda b: pair(hb, entry[2], b), s_sigma=s)
        assert f"Parameter s_sigma is {s} but must be in [1, 128]" in last_error_message()
        same_code(hb, entry, code, lambda b: pair(hb, entry[2], b), s_sigma=s, r_sigma=-1.0)  # checked before r_sigma
        assert "s_sigma" in last_error_message()


@pytest.mark.parametrize("r_sigma", [0.0, -0.5, float("nan")])
def test_r_sigma_not_positive(hb, entry, r_sigma):
    from halide_b200.lib import capture_errors, last_error_message
    with capture_errors():
        for s in (1, 3, 8, 128):
            same_code(hb, entry, -9, lambda b: pair(hb, entry[2], b), s_sigma=s, r_sigma=r_sigma)
            assert "must be positive" in last_error_message()


def test_201_bins_are_refused(hb, entry):
    """r_sigma = 1/200 gives bins 0..200: one more than the largest grid bilateral_grid accepts."""
    from halide_b200.lib import capture_errors, last_error_message
    r = float(np.float32(1.0) / np.float32(200))
    with capture_errors():
        same_code(hb, entry, -9, lambda b: pair(hb, entry[2], b), r_sigma=r)
        assert "more than 200 intensity bins" in last_error_message()


@pytest.mark.parametrize("in_n,in_min,out_n,out_min,ok", [
    (3, 0, 3, 0, True),
    (5, -1, 3, 0, True),     # more input frames than output frames
    (3, 4, 2, 5, True),      # output frames a sub-range of the input's, away from 0
    (2, 0, 3, 0, False),     # one frame short at the end
    (3, 1, 3, 0, False),     # one frame short at the start
    (2, 5, 2, 0, False),     # disjoint
])
def test_input_frames_must_cover_the_output_frames(hb, entry, in_n, in_min, out_n, out_min, ok):
    from halide_b200.lib import capture_errors, last_error_message
    sym, _, dt, takes_s = entry
    bi = buf(hb, (in_n, H, W), dt, (0, 0, in_min))
    bo = buf(hb, (out_n, H, W), dt, (0, 0, out_min), host_dirty=False)
    with capture_errors():
        # (r_sigma 0: a clip that passes the frame check stops at the parameter check, before any CUDA call)
        assert call(hb, sym, takes_s, bi, bo, r_sigma=0.0) == (-9 if ok else -4)
        if not ok:
            msg = last_error_message()
            assert "Input buffer input is accessed at" in msg and "in dimension 2" in msg, msg


def test_bounds_query_of_the_input(hb, entry):
    """The output's (x, y, n) region with dense strides; the output is left as it was.  Before the parameter checks."""
    sym, _, dt, takes_s = entry
    bo = buf(hb, (3, 20, 30), dt, (5, -3, -2), host_dirty=False)
    before = bo.shape()
    bi = hb.HalideBuffer.bounds_query(dt, 3)
    assert call(hb, sym, takes_s, bi, bo, s_sigma=0, r_sigma=-1.0) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30), (-2, 3, 600)]
    assert bo.shape() == before


def test_bounds_query_of_both_buffers(hb, entry):
    """An output with no memory keeps its region and gets dense strides; the input is given that region."""
    sym, _, dt, takes_s = entry
    bi, bo = hb.HalideBuffer.bounds_query(dt, 3), hb.HalideBuffer.bounds_query(dt, 3)
    for d, (m, e) in enumerate([(4, 6), (-1, 5), (7, 2)]):
        bo.buf.dim[d].min, bo.buf.dim[d].extent = m, e
    assert call(hb, sym, takes_s, bi, bo) == 0
    want = [(4, 6, 1), (-1, 5, 6), (7, 2, 30)]
    assert bo.shape() == want
    assert bi.shape() == want


def test_empty_clip_returns_zero(hb, entry):
    """N = 0 (and W or H = 0) returns 0, before the parameter checks, as an empty frame does in the one-frame entry
    point."""
    sym, _, dt, takes_s = entry
    bi = buf(hb, (N, H, W), dt, (0, 0, 0))
    for shape in [(0, H, W), (N, 0, W), (N, H, 0)]:
        n, h, w = shape
        bo = raw(hb, dt, (w, h, n), (1, max(w, 1), max(w * h, 1)), host_dirty=False)
        assert call(hb, sym, takes_s, bi, bo) == 0, shape
        assert call(hb, sym, takes_s, bi, bo, s_sigma=0, r_sigma=0.0) == 0, shape
    # no output frames: the input's frames need not be anywhere near
    far = buf(hb, (N, H, W), dt, (0, 0, 100))
    assert call(hb, sym, takes_s, far, raw(hb, dt, (W, H, 0), (1, W, W * H), host_dirty=False)) == 0


def test_python_wrappers(hb, entry):
    from halide_b200 import HalideError, bilateral_grid_video
    sym, _, dt, takes_s = entry
    fn = getattr(bilateral_grid_video, sym[len("halide_b200_"):])
    assert fn.__doc__ and "frame" in fn.__doc__
    args = (0, 0.1) if takes_s else (0.0,)  # s_sigma 0 (-9), or r_sigma 0 (-9)
    with pytest.raises(HalideError) as e:
        fn(*pair(hb, dt, True)[:1], *args, pair(hb, dt, True)[1])
    assert e.value.code == -9


def test_module_holds_the_three_entry_points():
    import inspect

    from halide_b200 import bilateral_grid_video
    public = {n for n, f in inspect.getmembers(bilateral_grid_video, inspect.isfunction)
              if f.__module__ == bilateral_grid_video.__name__ and not n.startswith("_")}
    assert public == {e[0][len("halide_b200_"):] for e in ENTRIES}
