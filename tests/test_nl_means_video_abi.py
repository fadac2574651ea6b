"""Argument checks of the batch and interleaved nl_means entry points (float32 and uint8): types, dimensions, the
interleaved layout rules, the output's channels, the patch / search ranges, the input's coverage of the output's frames,
bounds queries and empty outputs.  Every case returns before the library makes a CUDA call, so none needs a GPU.

Buffers are numpy arrays: a planar one-frame array is (c, y, x), a planar batch (n, c, y, x); an interleaved frame is
(y, x, c) and an interleaved batch (n, y, x, c), described as (x, y, c[, n]) by a transposed view."""
import ctypes

import numpy as np
import pytest

# (symbol, element type, batch, interleaved)
ENTRIES = [
    ("halide_b200_nl_means_batch", np.float32, True, False),
    ("halide_b200_nl_means_interleaved", np.float32, False, True),
    ("halide_b200_nl_means_interleaved_batch", np.float32, True, True),
    ("halide_b200_nl_means_u8_batch", np.uint8, True, False),
    ("halide_b200_nl_means_u8_interleaved", np.uint8, False, True),
    ("halide_b200_nl_means_u8_interleaved_batch", np.uint8, True, True),
]
IDS = [e[0][len("halide_b200_"):] for e in ENTRIES]
H, W = 8, 10


@pytest.fixture(params=ENTRIES, ids=IDS)
def entry(request):
    return request.param


def call(hb, sym, bi, bo, patch=3, search=7, sigma=0.12):
    fn = getattr(hb.load_library(), sym)
    return fn(None if bi is None else bi.ptr, ctypes.c_int32(patch), ctypes.c_int32(search), ctypes.c_float(sigma),
              None if bo is None else bo.ptr)


def array(dtype, batch, interleaved, c=3, n=2, h=H, w=W):
    shape = (h, w, c) if interleaved else (c, h, w)
    return np.zeros(((n,) if batch else ()) + shape, dtype)


def buf(hb, arr, interleaved, mins=None, host_dirty=True):
    """The (x, y, c[, n]) buffer over arr (see the module docstring)."""
    if interleaved:
        arr = arr.transpose((2, 0, 1) if arr.ndim == 3 else (0, 3, 1, 2))
    return hb.HalideBuffer.from_numpy(arr, mins, host_dirty=host_dirty)


def bufs(hb, dtype, batch, interleaved, in_mins=None, out_mins=None, **kw):
    return (buf(hb, array(dtype, batch, interleaved, **kw), interleaved, in_mins),
            buf(hb, array(dtype, batch, interleaved), interleaved, out_mins, host_dirty=False))


def test_null_buffers(hb, entry):
    sym, dt, batch, il = entry
    bi, bo = bufs(hb, dt, batch, il)
    assert call(hb, sym, None, bo) == -12
    assert call(hb, sym, bi, None) == -12


@pytest.mark.parametrize("other", [np.uint16, np.int8, np.float64])
def test_wrong_type(hb, entry, other):
    sym, dt, batch, il = entry
    wrong = np.uint8 if dt == np.float32 else np.float32  # the float entry points refuse uint8 and the reverse
    for t in (wrong, other):
        bi, bo = bufs(hb, t, batch, il)
        assert call(hb, sym, bi, bo) == -3, t
        bi, bo = bufs(hb, dt, batch, il)[0], bufs(hb, t, batch, il)[1]
        assert call(hb, sym, bi, bo) == -3, t


def test_wrong_dimensions(hb, entry):
    sym, dt, batch, il = entry
    good_i, good_o = bufs(hb, dt, batch, il)
    other_i, other_o = bufs(hb, dt, not batch, il)
    assert call(hb, sym, other_i, good_o) == -43
    assert call(hb, sym, good_i, other_o) == -43
    flat = hb.HalideBuffer.from_numpy(np.zeros((H, W), dt))
    assert call(hb, sym, flat, good_o) == -43


def raw(hb, dt, shape, strides, mins=None, host_dirty=True):
    """A buffer of (x, y, c[, n]) extents and strides over a zeroed backing store large enough for any of them."""
    b = hb.HalideBuffer(dt, shape, strides=strides, mins=mins)
    b._keep = np.zeros(1 << 16, dt)  # (never read: the checks return before any copy)
    b.buf.host = b._keep.ctypes.data
    b.set_host_dirty(host_dirty)
    return b


def good_shape(batch, c=3):
    return ((W, H, c, 2), (c, W * c, 1, W * H * c)) if batch else ((W, H, c), (c, W * c, 1))


def test_interleaved_layout_rules(hb, entry):
    """Each rule check_shapes applies to interleaved buffers, on the input and on the output: -8."""
    sym, dt, batch, il = entry
    if not il:
        pytest.skip("planar entry point")
    shape, strides = good_shape(batch)
    bad = [
        list(strides[:1]) + [strides[1], 2] + list(strides[3:]),  # channels not adjacent
        [2, W * 3, 1] + list(strides[3:]),                          # pitch below the channel extent
        [3, -W * 3, 1] + list(strides[3:]),                         # negative row stride
        [3, 0, 1] + list(strides[3:]),                              # zero row stride
    ]
    if batch:
        bad += [[3, W * 3, 1, 0], [3, W * 3, 1, -W * H * 3]]         # frame stride not positive
    for s in bad:
        assert call(hb, sym, raw(hb, dt, shape, s), raw(hb, dt, shape, strides, host_dirty=False)) == -8, s
        assert call(hb, sym, raw(hb, dt, shape, strides), raw(hb, dt, shape, s, host_dirty=False)) == -8, s
    # a good pair passes the layout checks (up to the patch check, before any CUDA call)
    assert call(hb, sym, raw(hb, dt, shape, strides), raw(hb, dt, shape, strides, host_dirty=False), patch=0) == -9


def test_planar_buffers_refused_by_interleaved_entry_points(hb, entry):
    sym, dt, batch, il = entry
    if not il:
        pytest.skip("planar entry point")
    pi, po = bufs(hb, dt, batch, False)
    ii, io = bufs(hb, dt, batch, True)
    assert call(hb, sym, pi, io) == -8
    assert call(hb, sym, ii, po) == -8


def test_interleaved_buffers_refused_by_planar_entry_points(hb, entry):
    """nl_means / nl_means_u8 (one frame) and the planar batch entry points keep dim[0].stride == 1."""
    sym, dt, batch, il = entry
    ii, io = bufs(hb, dt, batch, True)
    one = "nl_means" if dt == np.float32 else "halide_b200_nl_means_u8"
    if not batch:
        assert call(hb, one, ii, io) == -8
    else:
        assert call(hb, sym.replace("_interleaved", ""), ii, io) == -8
        pi, po = bufs(hb, dt, True, False)  # and the one-frame entry points refuse 4-D buffers
        assert call(hb, one, pi, po) == -43


def test_rgba_and_single_channel_inputs_pass_the_layout_checks(hb, entry):
    """An RGBA input (pitch 4) and a 1-channel input of pitch 1; an RGBA output covering channels [0, 3)."""
    sym, dt, batch, il = entry
    if not il:
        pytest.skip("planar entry point")
    n = (2,) if batch else ()
    for c in (4, 1):
        bi = buf(hb, np.zeros(n + (H, W, c), dt), True)
        bo = buf(hb, np.zeros(n + (H, W, 3), dt), True, host_dirty=False)
        assert call(hb, sym, bi, bo, patch=0) == -9, c
    rgba_out = np.zeros(n + (H, W, 4), dt)[..., :3]
    assert call(hb, sym, buf(hb, np.zeros(n + (H, W, 3), dt), True), buf(hb, rgba_out, True, host_dirty=False),
                patch=0) == -9


@pytest.mark.parametrize("c,cmin", [(4, 0), (2, 0), (3, 1)])
def test_output_channels_must_be_0_to_3(hb, entry, c, cmin):
    sym, dt, batch, il = entry
    bi = bufs(hb, dt, batch, il)[0]
    out = array(dtype=dt, batch=batch, interleaved=il, c=c)
    mins = (0, 0, cmin) + ((0,) if batch else ())
    assert call(hb, sym, bi, buf(hb, out, il, mins, host_dirty=False)) == -8
    # (before the parameter checks, as in nl_means)
    assert call(hb, sym, bi, buf(hb, out, il, mins, host_dirty=False), patch=0, search=64) == -8


@pytest.mark.parametrize("patch,search,code", [
    (0, 7, -9), (3, 0, -9), (-1, 7, -9), (32, 7, -10), (3, 64, -10), (0, 64, -9), (32, 0, -9),
])
def test_sizes_out_of_range(hb, entry, patch, search, code):
    from halide_b200.lib import capture_errors, last_error_message
    sym, dt, batch, il = entry
    with capture_errors():
        assert call(hb, sym, *bufs(hb, dt, batch, il), patch=patch, search=search) == code
        assert f"patch_size {patch} / search_area {search} outside" in last_error_message()


def test_input_is_clamped_in_x_y_and_c(hb, entry):
    """An input smaller than, and away from, the output in x, y and c passes the checks."""
    sym, dt, batch, il = entry
    bi = buf(hb, array(dt, batch, il, c=1, h=2, w=3), il, (100, -50, 0) + ((0,) if batch else ()))
    assert call(hb, sym, bi, bufs(hb, dt, batch, il)[1], patch=0) == -9


@pytest.mark.parametrize("in_n,in_min,out_n,out_min,ok", [
    (2, 0, 2, 0, True),
    (5, -1, 3, 0, True),     # more input frames than output frames
    (2, 0, 3, 0, False),     # one frame short at the end
    (3, 1, 3, 0, False),     # one frame short at the start
    (2, 5, 2, 0, False),     # disjoint
])
def test_input_frames_must_cover_the_output_frames(hb, entry, in_n, in_min, out_n, out_min, ok):
    from halide_b200.lib import capture_errors, last_error_message
    sym, dt, batch, il = entry
    if not batch:
        pytest.skip("one-frame entry point")
    bi = buf(hb, array(dt, True, il, n=in_n), il, (0, 0, 0, in_min))
    bo = buf(hb, array(dt, True, il, n=out_n), il, (0, 0, 0, out_min), host_dirty=False)
    with capture_errors():
        assert call(hb, sym, bi, bo, patch=0) == (-9 if ok else -4)
        if not ok:
            assert "dimension 3" in last_error_message()


def test_empty_input_frame(hb, entry):
    sym, dt, batch, il = entry
    for c, h, w in [(0, H, W), (3, 0, W), (3, H, 0)]:
        shape = (w, h, c) + ((2,) if batch else ())
        strides = (max(c, 1), max(w * c, 1), 1) if il else (1, max(w, 1), max(w * h, 1))
        if batch:
            strides += (max(w * h * c, 1),)
        assert call(hb, sym, raw(hb, dt, shape, strides), bufs(hb, dt, batch, il)[1]) == -4, (c, h, w)


def test_empty_output_returns_zero(hb, entry):
    """Before the parameter checks and the coverage of the output's frames, as in nl_means."""
    sym, dt, batch, il = entry
    shapes = [(0, H), (W, 0)] + ([(W, H, 0)] if batch else [])
    for s in shapes:
        w, h = s[0], s[1]
        n = s[2] if len(s) > 2 else 2
        shape = (w, h, 3) + ((n,) if batch else ())
        strides = (3, max(w * 3, 1), 1) if il else (1, max(w, 1), max(w * h, 1))
        if batch:
            strides += (max(w * h * 3, 1),)
        bo = raw(hb, dt, shape, strides, host_dirty=False)
        bi = bufs(hb, dt, batch, il)[0]
        assert call(hb, sym, bi, bo) == 0, s
        assert call(hb, sym, bi, bo, patch=0) == 0, s
        if batch:  # input frames far away from the output's
            far = buf(hb, array(dt, True, il), il, (0, 0, 0, 100))
            assert call(hb, sym, far, bo) == 0, s


def test_size_limits(hb, entry):
    sym, dt, batch, il = entry
    n = (1,) if batch else ()
    nst = (1,) if batch else ()
    if il:
        assert call(hb, sym, raw(hb, dt, (4, 4, 3) + n, (3, 1 << 30, 1) + nst), bufs(hb, dt, batch, il)[1]) == -5
        assert call(hb, sym, raw(hb, dt, (1 << 16, 1 << 16, 1) + n, (1, 1, 1) + nst), bufs(hb, dt, batch, il)[1]) == -6
    else:
        assert call(hb, sym, raw(hb, dt, (4, 4, 3) + n, (1, 4, 1 << 30) + nst), bufs(hb, dt, batch, il)[1]) == -5
        assert call(hb, sym, raw(hb, dt, (1 << 16, 1 << 16, 1) + n, (1, 0, 0) + nst), bufs(hb, dt, batch, il)[1]) == -6


def test_bounds_query_of_the_input(hb, entry):
    """The output's x/y region, channels [0, 3) and (a batch) the output's frames, with dense strides of the entry
    point's layout; the output is left as it was."""
    sym, dt, batch, il = entry
    n = (3,) if batch else ()
    out = np.zeros(n + ((20, 30, 3) if il else (3, 20, 30)), dt)
    mins = (5, -3, 0) + ((-2,) if batch else ())
    bo = buf(hb, out, il, mins, host_dirty=False)
    before = bo.shape()
    bi = hb.HalideBuffer.bounds_query(dt, 4 if batch else 3)
    assert call(hb, sym, bi, bo, patch=0) == 0  # (before the parameter checks)
    want = [(5, 30, 3 if il else 1), (-3, 20, 90 if il else 30), (0, 3, 1 if il else 600)]
    if batch:
        want.append((-2, 3, 1800))
    assert bi.shape() == want
    assert bo.shape() == before


def test_bounds_query_of_the_output(hb, entry):
    """An output with no memory is given its own x/y region, channels [0, 3) and frames, with the layout's dense
    strides."""
    sym, dt, batch, il = entry
    bi = bufs(hb, dt, batch, il)[0]
    bo = hb.HalideBuffer.bounds_query(dt, 4 if batch else 3)
    for d, (m, e) in enumerate([(4, 6), (-1, 5), (0, 3), (7, 2)][:4 if batch else 3]):
        bo.buf.dim[d].min, bo.buf.dim[d].extent = m, e
    assert call(hb, sym, bi, bo) == 0
    want = [(4, 6, 3 if il else 1), (-1, 5, 18 if il else 6), (0, 3, 1 if il else 30)]
    if batch:
        want.append((7, 2, 90))
    assert bo.shape() == want


def test_python_wrappers(hb, entry):
    from halide_b200 import HalideError, nl_means_video
    sym, dt, batch, il = entry
    fn = getattr(nl_means_video, sym[len("halide_b200_"):])
    assert fn.__doc__ and ("interleaved" in fn.__doc__) == il
    with pytest.raises(HalideError) as e:
        fn(*bufs(hb, dt, batch, il)[:1], 0, 7, 0.12, bufs(hb, dt, batch, il)[1])
    assert e.value.code == -9
