"""local_laplacian at pyramid depths other than 8, without a GPU: the bordered oracle (each level stored only inside its
constant border) against the literal one at every depth the literal one can afford, the numpy restatement against the
C++ oracle, halide_b200_local_laplacian_pyramid_levels's argument checks (all of which return before any CUDA call), and
which levels of a very wide frame get launches of their own."""
import ctypes

import numpy as np
import pytest

import ll_bordered
from util import smooth_u16_frame, u16_frame

ENTRY = "halide_b200_local_laplacian_pyramid_levels"

# (name, numpy input shape [c, h, w], oracle keywords): whole frames, inputs larger than the output at negative and
# positive mins, and channel crops
FRAMES = [
    ("1x1", (3, 1, 1), {}),
    ("1xN", (3, 1, 23), {}),
    ("Nx1", (3, 19, 1), {}),
    ("5x3", (3, 3, 5), {}),
    ("37x29", (3, 29, 37), {}),
    ("64x64", (3, 64, 64), {}),
    ("crop_neg", (3, 30, 41), dict(out_shape=(3, 17, 22), in_mins=(-13, -7, 0), out_mins=(-9, -5, 0))),
    ("crop_pos", (3, 25, 33), dict(out_shape=(3, 11, 9), in_mins=(100, 37, 0), out_mins=(117, 45, 0))),
    ("channels_1_3", (3, 21, 26), dict(out_shape=(2, 21, 26), out_mins=(0, 0, 1))),
    ("channel_0_of_1", (1, 13, 15), dict(out_shape=(1, 13, 15))),
]


@pytest.mark.parametrize("J", range(1, 12))
@pytest.mark.parametrize("name,shape,kw", FRAMES, ids=[f[0] for f in FRAMES])
def test_bordered_oracle_equals_literal(oracle, J, name, shape, kw):
    img = u16_frame(shape, 11 * J + len(name)) if J % 2 else smooth_u16_frame(shape, J)
    for levels, alpha, beta in [(8, 1.0 / 7.0, 1.0), (3, 0.75, 0.5)]:
        a = oracle.local_laplacian(img, levels, alpha, beta, pyramid_levels=J, **kw)
        b = ll_bordered.local_laplacian(img, levels, alpha, beta, pyramid_levels=J, **kw)
        assert np.array_equal(a, b), (levels, int(np.count_nonzero(a != b)))


@pytest.mark.parametrize("J", [1, 2, 3, 5])
def test_restatement_agrees(oracle, J):
    from oracle import np_restatement as npr
    img = smooth_u16_frame((3, 23, 31), J)
    for levels, alpha, beta, kw in [(8, 1.0 / 7.0, 1.0, {}), (5, 0.5, 0.5, {}),
                                    (8, 1.0 / 7.0, 1.0, dict(out_shape=(2, 11, 13), in_mins=(-4, 3, 0), out_mins=(-1, 6, 1)))]:
        a = oracle.local_laplacian(img, levels, alpha, beta, pyramid_levels=J, **kw)
        b = npr.local_laplacian(img, levels, alpha, beta, J=J, **kw)
        assert np.array_equal(a, b), (levels, kw)


# ---- argument checks ------------------------------------------------------------------------------------------------

def _call(hb, bi, bo, J=5, levels=8):
    l = hb.load_library()
    return getattr(l, ENTRY)(None if bi is None else bi.ptr, ctypes.c_int32(J), ctypes.c_int32(levels), ctypes.c_float(1 / 7),
                             ctypes.c_float(1.0), None if bo is None else bo.ptr)


def _buf(hb, shape, dtype=np.uint16, mins=None, host_dirty=True):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, dtype), mins, host_dirty=host_dirty)


def _fails(hb, code, message, *args, **kw):
    from halide_b200.lib import capture_errors, last_error_message
    with capture_errors():
        assert _call(hb, *args, **kw) == code
        assert message in last_error_message(), last_error_message()


def test_null_buffers(hb):
    assert _call(hb, None, _buf(hb, (3, 8, 10), host_dirty=False)) == -12
    assert _call(hb, _buf(hb, (3, 8, 10)), None) == -12


@pytest.mark.parametrize("tin,tout", [(np.uint8, np.uint8), (np.float32, np.float32), (np.uint16, np.uint8), (np.uint8, np.uint16)])
def test_wrong_type(hb, tin, tout):
    assert _call(hb, _buf(hb, (3, 8, 10), tin), _buf(hb, (3, 8, 10), tout, host_dirty=False)) == -3


def test_wrong_dimensions(hb):
    assert _call(hb, _buf(hb, (8, 10)), _buf(hb, (3, 8, 10), host_dirty=False)) == -43
    assert _call(hb, _buf(hb, (3, 8, 10)), _buf(hb, (2, 3, 8, 10), host_dirty=False)) == -43


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((3, 8, 10), None, (3, 9, 10), None),                 # rows
    ((3, 8, 10), None, (3, 8, 11), None),                 # columns
    ((2, 8, 10), None, (3, 8, 10), None),                 # channels
    ((3, 8, 10), (1, 0, 0), (3, 8, 10), (0, 0, 0)),       # shifted by one column
    ((3, 8, 10), (0, -2, 0), (3, 8, 10), (0, -3, 0)),     # shifted by one row
])
def test_output_not_covered_by_the_input(hb, in_shape, in_mins, out_shape, out_mins):
    for J in (1, 2, 8, 20):
        assert _call(hb, _buf(hb, in_shape, mins=in_mins), _buf(hb, out_shape, mins=out_mins, host_dirty=False), J) == -4


@pytest.mark.parametrize("J,code", [(0, -9), (-1, -9), (21, -10)])
def test_pyramid_levels_out_of_range(hb, J, code):
    _fails(hb, code, f"Parameter pyramid_levels is {J} but must be in [1, 20]", _buf(hb, (3, 8, 10)),
           _buf(hb, (3, 8, 10), host_dirty=False), J)


@pytest.mark.parametrize("levels,code", [(1, -9), (33, -10)])
def test_levels_out_of_range(hb, levels, code):
    for J in (1, 2, 5, 20):
        _fails(hb, code, f"Parameter levels is {levels} but must be in [2, 32]", _buf(hb, (3, 8, 10)),
               _buf(hb, (3, 8, 10), host_dirty=False), J, levels)


def test_bounds_query_answers_the_output_region(hb):
    for J in (1, 3, 14):
        bi = hb.HalideBuffer.bounds_query(np.uint16, 3)
        bo = _buf(hb, (3, 20, 30), mins=(5, -3, 0), host_dirty=False)
        assert _call(hb, bi, bo, J) == 0
        assert bi.shape() == bo.shape() == [(5, 30, 1), (-3, 20, 30), (0, 3, 600)]


def test_bounds_query_comes_before_the_parameter_checks(hb):
    bi = hb.HalideBuffer.bounds_query(np.uint16, 3)
    assert _call(hb, bi, _buf(hb, (3, 4, 6), host_dirty=False), 0, 1) == 0
    assert bi.shape() == [(0, 6, 1), (0, 4, 6), (0, 3, 24)]


@pytest.mark.parametrize("shape", [(10, 8, 0), (10, 0, 3), (0, 8, 3)])  # (x, y, c), dense strides
def test_empty_output(hb, shape):
    backing = np.zeros(16, np.uint16)
    bo = hb.HalideBuffer(np.uint16, shape)
    bo.buf.host = backing.ctypes.data
    for J in (1, 2, 9, 20):
        assert _call(hb, _buf(hb, (3, 8, 10)), bo, J) == 0


# ---- which levels get launches of their own --------------------------------------------------------------------------

def test_last_own_level(hb):
    """Levels of at most 40 K pixels share the cooperative coarse tail.  On a 2^22 x 1 frame level 8 is still 16 K columns
    by a few rows, so at J = 14 it has launches of its own (ll_down_rows / ll_up2 at a level index past the 8 slots of the
    kernels' per-level stride arrays); on 4K it is inside the tail."""
    l = hb.load_library()
    assert l.halide_b200_ll_last_own_level(1 << 22, 1, 14) >= 8
    assert l.halide_b200_ll_last_own_level(3840, 2160, 14) < 8
    assert l.halide_b200_ll_last_own_level(3840, 2160, 8) == l.halide_b200_ll_last_own_level(3840, 2160, 20)
    assert l.halide_b200_ll_last_own_level(3840, 2160, 1) == 0
    assert l.halide_b200_ll_last_own_level(3840, 2160, 21) == -1
