"""halide_b200_conv_layer_any_shape without a GPU: its argument checks and bounds query (all of which return before any
CUDA call), conv_layer's unchanged fixed-shape rule, and the two CPU restatements of the generator at shapes other than
the fixed one."""
import numpy as np
import pytest

from util import f32_frame

ENTRY = "halide_b200_conv_layer_any_shape"
N, CI, CO, W, H = 2, 5, 7, 6, 4  # the shape the checks are built around (Halide order below: innermost first)


def _buf(hb, shape_xyz, dtype=np.float32, mins=None, host_dirty=True):
    """A dense host buffer of zeros with Halide extents `shape_xyz` (innermost first)."""
    return hb.HalideBuffer.from_numpy(np.zeros(tuple(reversed(shape_xyz)), dtype), mins, host_dirty=host_dirty)


def _bufs(hb, inp=(CI, W + 2, H + 2, N), filt=(CO, 3, 3, CI), bias=(CO,), relu=(CO, W, H, N), in_mins=None, f_mins=None,
          b_mins=None, out_mins=None):
    return [_buf(hb, inp, mins=in_mins), _buf(hb, filt, mins=f_mins), _buf(hb, bias, mins=b_mins),
            _buf(hb, relu, mins=out_mins, host_dirty=False)]


def _call(hb, bufs, entry=ENTRY):
    return getattr(hb.load_library(), entry)(*[None if b is None else b.ptr for b in bufs])


def _fails(hb, code, message, bufs):
    from halide_b200.lib import capture_errors, last_error_message
    with capture_errors():
        assert _call(hb, bufs) == code
        assert message in last_error_message(), last_error_message()


def test_null_buffers(hb):
    for i in range(4):
        bufs = _bufs(hb)
        bufs[i] = None
        assert _call(hb, bufs) == -12


def test_wrong_type(hb):
    for i, shape in enumerate([(CI, W + 2, H + 2, N), (CO, 3, 3, CI), (CO,), (CO, W, H, N)]):
        bufs = _bufs(hb)
        bufs[i] = _buf(hb, shape, np.int32, host_dirty=i < 3)
        assert _call(hb, bufs) == -3


def test_wrong_dimensions(hb):
    for i, shape in enumerate([(CI, W + 2, H + 2), (CO, 3, 3), (CO, 1), (CO, W, H)]):
        bufs = _bufs(hb)
        bufs[i] = _buf(hb, shape, host_dirty=i < 3)
        assert _call(hb, bufs) == -43


@pytest.mark.parametrize("kw,message", [
    (dict(inp=(CI, W + 1, H + 2, N)), "Input buffer input is accessed at 7, which is beyond the max (6) in dimension 1"),
    (dict(inp=(CI, W + 2, H + 1, N)), "Input buffer input is accessed at 5, which is beyond the max (4) in dimension 2"),
    (dict(inp=(CI - 1, W + 2, H + 2, N)), "Input buffer input is accessed at 4, which is beyond the max (3) in dimension 0"),
    (dict(inp=(CI, W + 2, H + 2, N - 1)), "Input buffer input is accessed at 1, which is beyond the max (0) in dimension 3"),
    (dict(filt=(CO, 2, 3, CI)), "Input buffer filter is accessed at 2, which is beyond the max (1) in dimension 1"),
    (dict(filt=(CO, 3, 2, CI)), "Input buffer filter is accessed at 2, which is beyond the max (1) in dimension 2"),
    (dict(filt=(CO - 1, 3, 3, CI)), "Input buffer filter is accessed at 6, which is beyond the max (5) in dimension 0"),
    (dict(bias=(CO - 1,)), "Input buffer bias is accessed at 6, which is beyond the max (5) in dimension 0"),
    (dict(in_mins=(0, 1, 0, 0)), "Input buffer input is accessed at 0, which is before the min (1) in dimension 1"),
    (dict(in_mins=(1, 0, 0, 0)), "Input buffer input is accessed at 0, which is before the min (1) in dimension 0"),
    (dict(f_mins=(0, 0, 0, 1)), "Input buffer filter is accessed at 0, which is before the min (1) in dimension 3"),
    (dict(out_mins=(3, 0, 0, 0)), "Input buffer filter is accessed at 9, which is beyond the max (6) in dimension 0"),
])
def test_buffer_does_not_cover_its_region(hb, kw, message):
    _fails(hb, -4, message, _bufs(hb, **kw))


def _query(hb, which, bufs):
    bufs = list(bufs)
    bufs[which] = hb.HalideBuffer.bounds_query(np.float32, 1 if which == 2 else 4)
    assert _call(hb, bufs) == 0
    return bufs[which].shape()


def test_nonzero_mins_are_accepted_when_the_regions_cover(hb):
    """Larger buffers whose mins are not 0.  The regions follow relu's mins (shown by a bounds query, which needs no GPU),
    and moving any one buffer by an element so that its region sticks out is refused."""
    kw = dict(inp=(CI + 2, W + 5, H + 4, N + 1), in_mins=(-1, -9, 18, 3), filt=(CO + 3, 4, 5, CI + 1), f_mins=(10, -1, -2, 0),
              bias=(CO + 4,), b_mins=(9,), relu=(CO, W, H, N), out_mins=(11, -8, 19, 3))
    bufs = _bufs(hb, **kw)
    assert _query(hb, 0, bufs) == [(0, CI + 1, 1), (-8, W + 2, CI + 1), (19, H + 2, (CI + 1) * (W + 2)),
                                   (3, N, (CI + 1) * (W + 2) * (H + 2))]
    # the same buffers moved by one so that one region sticks out
    for name, mins in [("in_mins", (-1, -9, 18, 4)), ("f_mins", (12, -1, -2, 0)), ("b_mins", (12,)), ("in_mins", (-1, -7, 18, 3))]:
        assert _call(hb, _bufs(hb, **dict(kw, **{name: mins}))) == -4


def test_inner_stride_must_be_one(hb):
    for i in range(4):
        bufs = _bufs(hb)
        bufs[i].dims[0].stride = 2
        _fails(hb, -8, ".stride.0 (2) == 1 (1)", bufs)


def test_bounds_query_on_each_buffer(hb):
    mins = (11, -8, 19, 3)
    bufs = _bufs(hb, in_mins=(0, -8, 19, 3), f_mins=(11, 0, 0, 0), b_mins=(11,), out_mins=mins)
    assert _query(hb, 0, bufs) == [(0, CI, 1), (-8, W + 2, CI), (19, H + 2, CI * (W + 2)), (3, N, CI * (W + 2) * (H + 2))]
    # the filter's CI comes from the input when the filter is the buffer being queried
    assert _query(hb, 1, bufs) == [(11, CO, 1), (0, 3, CO), (0, 3, 3 * CO), (0, CI, 9 * CO)]
    assert _query(hb, 2, bufs) == [(11, CO, 1)]
    # relu without memory keeps the region its dim array states and gets dense strides
    bufs[3] = hb.HalideBuffer(np.float32, (CO, W, H, N), strides=(1, CO + 1, (CO + 1) * W + 3, 4096), mins=mins)
    assert _call(hb, bufs) == 0
    assert bufs[3].shape() == [(11, CO, 1), (-8, W, CO), (19, H, CO * W), (3, N, CO * W * H)]
    # a query comes before the region checks: the other buffers may be anything of the right type and rank
    bufs = _bufs(hb, inp=(1, 1, 1, 1), bias=(1,))
    assert _query(hb, 1, bufs) == [(0, CO, 1), (0, 3, CO), (0, 3, 3 * CO), (0, 1, 9 * CO)]


@pytest.mark.parametrize("d", range(4))
def test_zero_extent_output_does_nothing(hb, d):
    bufs = _bufs(hb)
    bufs[3].dims[d].extent = 0
    assert _call(hb, bufs) == 0
    assert not bufs[3].device_dirty


def test_conv_layer_still_refuses_other_shapes(hb):
    from halide_b200.lib import capture_errors, last_error_message
    with capture_errors():
        assert _call(hb, _bufs(hb), entry="conv_layer") == -8
        assert "Constraint violated: relu.dim(0)" in last_error_message(), last_error_message()


@pytest.mark.parametrize("shape", [(1, 1, 1, 1, 1), (2, 5, 7, 6, 4), (3, 37, 11, 9, 5)], ids=str)
def test_restatements_agree(oracle, shape):
    from oracle import np_restatement as npr
    n, ci, co, w, h = shape
    inp, filt, bias = (f32_frame(s, sum(shape) + i) - np.float32(0.25) for i, s in
                       enumerate([(n, h + 2, w + 2, ci), (ci, 3, 3, co), (co,)]))
    a, b = oracle.conv_layer(inp, filt, bias), npr.conv_layer(inp, filt, bias)
    assert a.shape == (n, h, w, co)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), float(np.abs(a - b).max())
