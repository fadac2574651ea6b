"""Argument checks of the batch halide_blur and stencil_chain entry points: each returns the code its one-frame
counterpart returns on one-frame buffers of the same x/y shape, checks that the input's frames cover the output's,
answers bounds queries with its x/y region extended by the output's frames, and returns 0 on an empty clip.  Every case
returns before the library makes a CUDA call, so none needs a GPU.

Buffers are numpy arrays: a frame is (y, x), a clip (n, y, x), described as (x, y[, n])."""
import ctypes

import numpy as np
import pytest

# (batch symbol, one-frame symbol, takes stencils, apron: how much larger than the output the input must be in x and y)
ENTRIES = [
    ("halide_b200_blur_batch", "halide_blur", False, 2),
    ("halide_b200_stencil_chain_batch", "stencil_chain", False, 0),
    ("halide_b200_stencil_chain_stencils_batch", "halide_b200_stencil_chain_stencils", True, 0),
]
IDS = [e[0][len("halide_b200_"):] for e in ENTRIES]
H, W, N = 8, 10, 3
INT32_MIN = -(1 << 31)
INT32_MAX = (1 << 31) - 1


@pytest.fixture(params=ENTRIES, ids=IDS)
def entry(request):
    return request.param


def call(hb, sym, takes_s, bi, bo, stencils=5):
    fn = getattr(hb.load_library(), sym)
    args = [None if bi is None else bi.ptr]
    if takes_s:
        args.append(ctypes.c_int32(stencils))
    args.append(None if bo is None else bo.ptr)
    return fn(*args)


def buf(hb, shape, dtype=np.uint16, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def pair(hb, entry, batch, dtype=np.uint16, out_dtype=None):
    """Input and output buffers that pass every x/y check: one frame, or N frames (frame mins 0) for a batch."""
    n = (N,) if batch else ()
    a = entry[3]
    return (buf(hb, n + (H + a, W + a), dtype),
            buf(hb, n + (H, W), dtype if out_dtype is None else out_dtype, host_dirty=False))


def same_code(hb, entry, want, make, **kw):
    """make(batch) -> (input, output): the batch entry point on the clip and its one-frame counterpart on the frame both
    return `want`."""
    sym, one, takes_s, _ = entry
    got_batch = call(hb, sym, takes_s, *make(True), **kw)
    got_one = call(hb, one, takes_s, *make(False), **kw)
    assert (got_batch, got_one) == (want, want), (sym, kw)


def raw(hb, shape, strides, mins=None, host_dirty=True):
    """A uint16 buffer of (x, y[, n]) extents and strides over a zeroed backing store large enough for any of them."""
    b = hb.HalideBuffer(np.uint16, shape, strides=strides, mins=mins)
    b._keep = np.zeros(1 << 16, np.uint16)  # (never read: the checks return before any copy)
    b.buf.host = b._keep.ctypes.data
    b.set_host_dirty(host_dirty)
    return b


def test_null_buffers(hb, entry):
    same_code(hb, entry, -12, lambda b: (None, pair(hb, entry, b)[1]))
    same_code(hb, entry, -12, lambda b: (pair(hb, entry, b)[0], None))


@pytest.mark.parametrize("other", [np.uint8, np.int16, np.float32])
def test_wrong_and_mixed_types(hb, entry, other):
    same_code(hb, entry, -3, lambda b: pair(hb, entry, b, dtype=other))
    same_code(hb, entry, -3, lambda b: pair(hb, entry, b, out_dtype=other))
    same_code(hb, entry, -3, lambda b: (pair(hb, entry, b, dtype=other)[0], pair(hb, entry, b)[1]))


def test_wrong_dimensions(hb, entry):
    sym, one, takes_s, a = entry
    clip_i, clip_o = pair(hb, entry, True)
    frame_i, frame_o = pair(hb, entry, False)
    four_i, four_o = buf(hb, (2, N, H + a, W + a)), buf(hb, (2, N, H, W), host_dirty=False)
    for bi, bo in [(frame_i, clip_o), (clip_i, frame_o), (frame_i, frame_o), (four_i, clip_o), (clip_i, four_o)]:
        assert call(hb, sym, takes_s, bi, bo) == -43
    # and the one-frame entry points keep refusing clips
    assert call(hb, one, takes_s, clip_i, frame_o) == -43
    assert call(hb, one, takes_s, frame_i, clip_o) == -43


def test_x_stride_not_one(hb, entry):
    a = entry[3]

    def make(batch, which):
        ish, osh = (W + a, H + a), (W, H)
        n = (N,) if batch else ()
        idense = (1, W + a) + (((W + a) * (H + a),) if batch else ())
        odense = (1, W) + ((W * H,) if batch else ())
        ibad = (2, 2 * (W + a)) + ((2 * (W + a) * (H + a),) if batch else ())
        obad = (2, 2 * W) + ((2 * W * H,) if batch else ())
        return (raw(hb, ish + n, ibad if which == 0 else idense),
                raw(hb, osh + n, obad if which == 1 else odense, host_dirty=False))

    same_code(hb, entry, -8, lambda b: make(b, 0))
    same_code(hb, entry, -8, lambda b: make(b, 1))


@pytest.mark.parametrize("in_shape,in_mins,out_mins", [
    ((9, 12), None, None),            # one row short
    ((10, 11), None, None),           # one column short
    ((10, 12), (1, 0), (0, 0)),       # shifted by one column
    ((10, 12), (0, -2), (0, -3)),     # shifted by one row
])
def test_blur_x_y_not_covered_by_the_input(hb, in_shape, in_mins, out_mins):
    """halide_blur needs [ox, ox + W + 1] x [oy, oy + H + 1]: -4, from the clip as from the frame."""
    entry = ENTRIES[0]

    def make(batch):
        n, nm = ((N,), (0,)) if batch else ((), ())
        return (buf(hb, n + in_shape, mins=None if in_mins is None else tuple(in_mins) + nm),
                buf(hb, n + (H, W), mins=None if out_mins is None else tuple(out_mins) + nm, host_dirty=False))

    same_code(hb, entry, -4, make)


@pytest.mark.parametrize("shape", [(0, W), (H, 0), (0, 0)])
def test_stencil_chain_empty_input(hb, entry, shape):
    """stencil_chain needs nothing of the input in x and y but that it is not empty: -4 with the same message."""
    from halide_b200.lib import capture_errors, last_error_message
    if entry[3]:
        pytest.skip("halide_blur requires a region of the input")
    with capture_errors():
        def make(batch):
            n = (N,) if batch else ()
            h, w = shape
            bi = raw(hb, (w, h) + n, (1, max(w, 1)) + ((max(w * h, 1),) if batch else ()))
            return bi, buf(hb, n + (H, W), host_dirty=False)

        same_code(hb, entry, -4, make)
        assert "Input buffer input is empty" in last_error_message()


@pytest.mark.parametrize("s,code", [(0, -9), (101, -10), (-1, -9), (INT32_MIN, -9), (INT32_MAX, -10)])
def test_stencils_out_of_range(hb, entry, s, code):
    from halide_b200.lib import capture_errors, last_error_message
    if not entry[2]:
        pytest.skip("entry point takes no stencils")
    with capture_errors():
        same_code(hb, entry, code, lambda b: pair(hb, entry, b), stencils=s)
        assert f"Parameter stencils is {s} but must be in [1, 100]" in last_error_message()


def test_stencils_checked_after_the_empty_input(hb):
    """An empty input is -4 even with stencils out of range, in the clip as in the frame."""
    entry = ENTRIES[2]
    same_code(hb, entry, -4, lambda b: (raw(hb, (0, H) + ((N,) if b else ()), (1, 1) + ((1,) if b else ())),
                                        pair(hb, entry, b)[1]), stencils=0)


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
    sym, _, takes_s, a = entry
    if ok and not takes_s:
        pytest.skip("a clip that passes the frame check would run (this entry point has no parameter to stop it)")
    bi = buf(hb, (in_n, H + a, W + a), mins=(0, 0, in_min))
    bo = buf(hb, (out_n, H, W), mins=(0, 0, out_min), host_dirty=False)
    with capture_errors():
        # (stencils 0: a clip that passes the frame check stops at the parameter check, before any CUDA call)
        assert call(hb, sym, takes_s, bi, bo, stencils=0) == (-9 if ok else -4)
        msg = last_error_message()
        if not ok:
            assert "Input buffer input is accessed at" in msg and "in dimension 2" in msg, msg


def test_bounds_query_of_the_input(hb, entry):
    """The entry point's x/y region of the input (blur: the output's grown by 2; stencil_chain: the output's) and the
    output's frames, with dense strides; the output is left as it was.  Before the parameter checks."""
    sym, _, takes_s, a = entry
    bo = buf(hb, (3, 20, 30), mins=(5, -3, -2), host_dirty=False)
    before = bo.shape()
    bi = hb.HalideBuffer.bounds_query(np.uint16, 3)
    assert call(hb, sym, takes_s, bi, bo, stencils=0) == 0
    w, h = 30 + a, 20 + a
    assert bi.shape() == [(5, w, 1), (-3, h, w), (-2, 3, w * h)]
    assert bo.shape() == before


def test_bounds_query_of_both_buffers(hb, entry):
    """An output with no memory keeps its region and gets dense strides; the input is given its region from it."""
    sym, _, takes_s, a = entry
    bi, bo = hb.HalideBuffer.bounds_query(np.uint16, 3), hb.HalideBuffer.bounds_query(np.uint16, 3)
    for d, (m, e) in enumerate([(4, 6), (-1, 5), (7, 2)]):
        bo.buf.dim[d].min, bo.buf.dim[d].extent = m, e
    assert call(hb, sym, takes_s, bi, bo) == 0
    assert bo.shape() == [(4, 6, 1), (-1, 5, 6), (7, 2, 30)]
    assert bi.shape() == [(4, 6 + a, 1), (-1, 5 + a, 6 + a), (7, 2, (6 + a) * (5 + a))]


def test_empty_clip_returns_zero(hb, entry):
    """N = 0 (and W or H = 0) returns 0, before the parameter checks, as an empty frame does in the one-frame entry
    point."""
    sym, _, takes_s, a = entry
    bi = buf(hb, (N, H + a, W + a), mins=(0, 0, 0))
    for shape in [(0, H, W), (N, 0, W), (N, H, 0)]:
        n, h, w = shape
        bo = raw(hb, (w, h, n), (1, max(w, 1), max(w * h, 1)), host_dirty=False)
        assert call(hb, sym, takes_s, bi, bo) == 0, shape
        assert call(hb, sym, takes_s, bi, bo, stencils=0) == 0, shape
    # no output frames: the input's frames need not be anywhere near
    far = buf(hb, (N, H + a, W + a), mins=(0, 0, 100))
    assert call(hb, sym, takes_s, far, raw(hb, (W, H, 0), (1, W, W * H), host_dirty=False)) == 0


def test_python_wrappers(hb, entry):
    from halide_b200 import HalideError, blur_video, stencil_chain_video
    sym, _, takes_s, a = entry
    name = sym[len("halide_b200_"):]
    fn = getattr(blur_video if name.startswith("blur") else stencil_chain_video, name)
    assert fn.__doc__ and "frame" in fn.__doc__
    bi, bo = pair(hb, entry, True)
    with pytest.raises(HalideError) as e:
        if takes_s:
            fn(bi, 0, bo)  # stencils 0: -9
        else:
            fn(bi, buf(hb, (N, H, W), np.float32, host_dirty=False))  # a float output: -3
    assert e.value.code == (-9 if takes_s else -3)


@pytest.mark.parametrize("module,names", [("blur_video", {"blur_batch"}),
                                          ("stencil_chain_video", {"stencil_chain_batch", "stencil_chain_stencils_batch"})])
def test_each_module_holds_exactly_its_entry_points(module, names):
    import importlib
    import inspect

    m = importlib.import_module("halide_b200." + module)
    public = {n for n, f in inspect.getmembers(m, inspect.isfunction) if f.__module__ == m.__name__ and not n.startswith("_")}
    assert public == names
