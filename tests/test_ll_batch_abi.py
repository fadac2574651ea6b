"""Argument checks of halide_b200_local_laplacian_batch (4-D (x, y, c, n) uint16 buffers).  Every case returns before the
library makes a CUDA call, so none needs a GPU."""
import ctypes

import numpy as np
import pytest

BATCH = "halide_b200_local_laplacian_batch"


def _call(hb, bi, bo, levels=8):
    l = hb.load_library()
    return getattr(l, BATCH)(None if bi is None else bi.ptr, ctypes.c_int32(levels), ctypes.c_float(1 / 7),
                             ctypes.c_float(1.0), None if bo is None else bo.ptr)


def _buf(hb, shape, dtype=np.uint16, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def test_null_buffers(hb):
    bo = _buf(hb, (2, 3, 8, 10), host_dirty=False)
    assert _call(hb, None, bo) == -12
    assert _call(hb, _buf(hb, (2, 3, 8, 10)), None) == -12


def test_wrong_type(hb):
    assert _call(hb, _buf(hb, (2, 3, 8, 10), np.float32), _buf(hb, (2, 3, 8, 10), host_dirty=False)) == -3
    assert _call(hb, _buf(hb, (2, 3, 8, 10)), _buf(hb, (2, 3, 8, 10), np.uint8, host_dirty=False)) == -3


def test_three_dimensional_buffers_are_refused(hb):
    assert _call(hb, _buf(hb, (3, 8, 10)), _buf(hb, (3, 8, 10), host_dirty=False)) == -43
    assert _call(hb, _buf(hb, (2, 3, 8, 10)), _buf(hb, (3, 8, 10), host_dirty=False)) == -43


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((2, 3, 8, 10), None, (3, 3, 8, 10), None),                            # one frame too few
    ((3, 3, 8, 10), (0, 0, 0, 1), (3, 3, 8, 10), (0, 0, 0, 0)),            # frames shifted by one
    ((3, 3, 8, 10), (0, 0, 0, -2), (2, 3, 8, 10), (0, 0, 0, 0)),           # input frames -2..0, output 0..1
    ((3, 3, 8, 10), None, (3, 3, 9, 10), None),                            # rows
    ((3, 3, 8, 10), None, (3, 3, 8, 11), None),                            # columns
    ((3, 2, 8, 10), None, (3, 3, 8, 10), None),                            # channels
])
def test_output_not_covered_by_the_input(hb, in_shape, in_mins, out_shape, out_mins):
    assert _call(hb, _buf(hb, in_shape, mins=in_mins), _buf(hb, out_shape, mins=out_mins, host_dirty=False)) == -4


def test_input_larger_than_the_output_passes_the_checks(hb):
    """An input covering more than the output in every dimension is accepted up to the levels check (levels = 1 fails
    there, before any CUDA call), so the coverage check did not refuse it."""
    bi = _buf(hb, (5, 4, 12, 14), mins=(-1, -1, -1, -1))
    bo = _buf(hb, (3, 3, 8, 10), mins=(0, 0, 0, 0), host_dirty=False)
    assert _call(hb, bi, bo, levels=1) == -9


@pytest.mark.parametrize("levels,code", [(1, -9), (33, -10), (0, -9), (-5, -9)])
def test_levels_out_of_range(hb, levels, code):
    assert _call(hb, _buf(hb, (2, 3, 8, 10)), _buf(hb, (2, 3, 8, 10), host_dirty=False), levels) == code


def test_empty_output_returns_zero(hb):
    backing = np.zeros(16, np.uint16)
    for shape in [(10, 8, 3, 0), (10, 0, 3, 2), (10, 8, 0, 2)]:  # (x, y, c, n), dense strides
        bo = hb.HalideBuffer(np.uint16, shape)
        bo.buf.host = backing.ctypes.data
        assert _call(hb, _buf(hb, (2, 3, 8, 10)), bo) == 0


def test_size_limits(hb):
    """The -5 / -6 limits of the other filters apply to the 4-D buffers: per-dimension span and product of extents."""
    backing = np.zeros(16, np.uint16)  # (never read: the checks return before any copy)
    big = hb.HalideBuffer(np.uint16, (4, 4, 3, 2), strides=(1, 4, 16, 1 << 30))
    big.buf.host = backing.ctypes.data
    big.buf.flags = 1
    assert _call(hb, big, _buf(hb, (2, 3, 4, 4), host_dirty=False)) == -5
    huge = hb.HalideBuffer(np.uint16, (1 << 16, 1 << 16, 1, 1), strides=(1, 0, 0, 0))
    huge.buf.host = big.buf.host
    huge.buf.flags = 1
    assert _call(hb, huge, _buf(hb, (1, 1, 4, 4), host_dirty=False)) == -6


def test_bounds_query_fills_the_input_region(hb):
    """A bounds query on the input proposes the output's 4-D region with dense strides."""
    bi = hb.HalideBuffer.bounds_query(np.uint16, 4)
    bo = _buf(hb, (4, 3, 20, 30), mins=(5, -3, 0, -2), host_dirty=False)
    assert _call(hb, bi, bo) == 0
    assert bi.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600), (-2, 4, 1800)]
    # the output untouched
    assert bo.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600), (-2, 4, 1800)]
