"""Argument checks of the 8-bit local_laplacian entry points: halide_b200_local_laplacian_u8 (3-D (x, y, c) uint8 buffers)
and halide_b200_local_laplacian_u8_batch (4-D (x, y, c, n)).  Every case returns before the library makes a CUDA call,
so none needs a GPU."""
import ctypes

import numpy as np
import pytest

SINGLE, BATCH = "halide_b200_local_laplacian_u8", "halide_b200_local_laplacian_u8_batch"
# the same (y, x) frame shape seen by either entry point: numpy shape, batch adds the leading frame dimension
SHAPES = {SINGLE: (3, 8, 10), BATCH: (2, 3, 8, 10)}


def _call(hb, fn, bi, bo, levels=8):
    l = hb.load_library()
    return getattr(l, fn)(None if bi is None else bi.ptr, ctypes.c_int32(levels), ctypes.c_float(1 / 7),
                          ctypes.c_float(1.0), None if bo is None else bo.ptr)


def _buf(hb, shape, dtype=np.uint8, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


@pytest.fixture(params=[SINGLE, BATCH])
def fn(request):
    return request.param


def test_null_buffers(hb, fn):
    s = SHAPES[fn]
    assert _call(hb, fn, None, _buf(hb, s, host_dirty=False)) == -12
    assert _call(hb, fn, _buf(hb, s), None) == -12


@pytest.mark.parametrize("tin,tout", [
    (np.uint16, np.uint16), (np.float32, np.float32),   # other element types
    (np.uint8, np.uint16), (np.uint16, np.uint8),       # mixed pairs
    (np.int8, np.int8), (np.float32, np.uint8),
])
def test_wrong_type(hb, fn, tin, tout):
    s = SHAPES[fn]
    assert _call(hb, fn, _buf(hb, s, tin), _buf(hb, s, tout, host_dirty=False)) == -3


def test_u16_entry_points_refuse_uint8(hb):
    """The uint16 entry points keep refusing 8-bit buffers."""
    l = hb.load_library()
    args = (ctypes.c_int32(8), ctypes.c_float(1 / 7), ctypes.c_float(1.0))
    bi, bo = _buf(hb, (3, 8, 10)), _buf(hb, (3, 8, 10), host_dirty=False)
    assert l.local_laplacian(bi.ptr, *args, bo.ptr) == -3
    bi, bo = _buf(hb, (2, 3, 8, 10)), _buf(hb, (2, 3, 8, 10), host_dirty=False)
    assert l.halide_b200_local_laplacian_batch(bi.ptr, *args, bo.ptr) == -3


def test_dimension_mixups(hb):
    three, four = (3, 8, 10), (2, 3, 8, 10)
    assert _call(hb, SINGLE, _buf(hb, four), _buf(hb, four, host_dirty=False)) == -43
    assert _call(hb, SINGLE, _buf(hb, three), _buf(hb, four, host_dirty=False)) == -43
    assert _call(hb, BATCH, _buf(hb, three), _buf(hb, three, host_dirty=False)) == -43
    assert _call(hb, BATCH, _buf(hb, four), _buf(hb, three, host_dirty=False)) == -43


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((3, 8, 10), None, (3, 9, 10), None),                 # rows
    ((3, 8, 10), None, (3, 8, 11), None),                 # columns
    ((2, 8, 10), None, (3, 8, 10), None),                 # channels
    ((3, 8, 10), (1, 0, 0), (3, 8, 10), (0, 0, 0)),       # columns shifted
    ((3, 8, 10), (0, -1, 0), (3, 8, 10), (0, 0, 0)),      # rows shifted
])
def test_single_output_not_covered_by_the_input(hb, in_shape, in_mins, out_shape, out_mins):
    assert _call(hb, SINGLE, _buf(hb, in_shape, mins=in_mins), _buf(hb, out_shape, mins=out_mins, host_dirty=False)) == -4


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((2, 3, 8, 10), None, (3, 3, 8, 10), None),                            # one frame too few
    ((3, 3, 8, 10), (0, 0, 0, 1), (3, 3, 8, 10), (0, 0, 0, 0)),            # frames shifted by one
    ((3, 3, 8, 10), (0, 0, 0, -2), (2, 3, 8, 10), (0, 0, 0, 0)),           # input frames -2..0, output 0..1
    ((3, 3, 8, 10), None, (3, 3, 9, 10), None),                            # rows
    ((3, 3, 8, 10), None, (3, 3, 8, 11), None),                            # columns
    ((3, 2, 8, 10), None, (3, 3, 8, 10), None),                            # channels
])
def test_batch_output_not_covered_by_the_input(hb, in_shape, in_mins, out_shape, out_mins):
    assert _call(hb, BATCH, _buf(hb, in_shape, mins=in_mins), _buf(hb, out_shape, mins=out_mins, host_dirty=False)) == -4


def test_input_larger_than_the_output_passes_the_checks(hb):
    """An input covering more than the output is accepted up to the levels check (levels = 1 fails there, before any
    CUDA call), so the coverage check did not refuse it."""
    bi = _buf(hb, (4, 12, 14), mins=(-1, -1, -1))
    assert _call(hb, SINGLE, bi, _buf(hb, (3, 8, 10), host_dirty=False), levels=1) == -9
    bi = _buf(hb, (5, 4, 12, 14), mins=(-1, -1, -1, -1))
    assert _call(hb, BATCH, bi, _buf(hb, (3, 3, 8, 10), host_dirty=False), levels=1) == -9


@pytest.mark.parametrize("levels,code", [(1, -9), (33, -10), (0, -9), (-5, -9)])
def test_levels_out_of_range(hb, fn, levels, code):
    s = SHAPES[fn]
    assert _call(hb, fn, _buf(hb, s), _buf(hb, s, host_dirty=False), levels) == code


def test_empty_output_returns_zero(hb):
    backing = np.zeros(16, np.uint8)
    for shape in [(10, 8, 0), (10, 0, 3), (0, 8, 3)]:  # (x, y, c), dense strides
        bo = hb.HalideBuffer(np.uint8, shape)
        bo.buf.host = backing.ctypes.data
        assert _call(hb, SINGLE, _buf(hb, (3, 8, 10)), bo) == 0
    for shape in [(10, 8, 3, 0), (10, 0, 3, 2), (10, 8, 0, 2)]:  # (x, y, c, n)
        bo = hb.HalideBuffer(np.uint8, shape)
        bo.buf.host = backing.ctypes.data
        assert _call(hb, BATCH, _buf(hb, (2, 3, 8, 10)), bo) == 0


def test_size_limits(hb):
    """The -5 / -6 limits of the other filters: per-dimension span and product of extents."""
    backing = np.zeros(16, np.uint8)  # (never read: the checks return before any copy)
    big = hb.HalideBuffer(np.uint8, (4, 4, 3), strides=(1, 4, 1 << 30))
    big.buf.host = backing.ctypes.data
    big.buf.flags = 1
    assert _call(hb, SINGLE, big, _buf(hb, (3, 4, 4), host_dirty=False)) == -5
    huge = hb.HalideBuffer(np.uint8, (1 << 16, 1 << 16, 1), strides=(1, 0, 0))
    huge.buf.host = backing.ctypes.data
    huge.buf.flags = 1
    assert _call(hb, SINGLE, huge, _buf(hb, (1, 4, 4), host_dirty=False)) == -6
    big4 = hb.HalideBuffer(np.uint8, (4, 4, 3, 2), strides=(1, 4, 16, 1 << 30))
    big4.buf.host = backing.ctypes.data
    big4.buf.flags = 1
    assert _call(hb, BATCH, big4, _buf(hb, (2, 3, 4, 4), host_dirty=False)) == -5
    huge4 = hb.HalideBuffer(np.uint8, (1 << 16, 1 << 16, 1, 1), strides=(1, 0, 0, 0))
    huge4.buf.host = backing.ctypes.data
    huge4.buf.flags = 1
    assert _call(hb, BATCH, huge4, _buf(hb, (1, 1, 4, 4), host_dirty=False)) == -6


def test_bounds_query_fills_the_input_region(hb):
    """A bounds query on the input proposes the output's region with dense strides; the output is left as it was."""
    bi = hb.HalideBuffer.bounds_query(np.uint8, 3)
    bo = _buf(hb, (3, 20, 30), mins=(5, -3, 0), host_dirty=False)
    assert _call(hb, SINGLE, bi, bo) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600)]
    assert bo.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600)]
    bi = hb.HalideBuffer.bounds_query(np.uint8, 4)
    bo = _buf(hb, (4, 3, 20, 30), mins=(5, -3, 0, -2), host_dirty=False)
    assert _call(hb, BATCH, bi, bo) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600), (-2, 4, 1800)]
    assert bo.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600), (-2, 4, 1800)]
