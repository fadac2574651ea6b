"""Strides the filters refuse, checked before the library makes any CUDA call (no GPU needed).

A planar buffer may have any stride but dim[0].stride == 1, so a reversed (-1) or broadcast (0) innermost dimension is
refused with constraint_violated (-8) by every planar entry point, on the input and on the output.  The interleaved
entry points need positive row and frame strides (dim[1], dim[3]), and the fixed-shape conv_layer a dense layout.  The
refused buffers carry a host pointer that is never read: a null one would make the call a bounds query.  Each planar
case also makes the same call on dense buffers, which gets as far as the device allocation (and runs where there is a
GPU)."""
import ctypes

import numpy as np
import pytest

CONSTRAINT_VIOLATED, OUT_OF_BOUNDS = -8, -4  # halide_error_code_t
H, W = 20, 24


def _buf(hb, dtype, shape_xyz, strides=None, mins=None, dense=False):
    """A host buffer of shape (x, y, ...) with the given strides over a small array that is never read, or (dense) over a
    zero array it spans exactly."""
    b = hb.HalideBuffer(dtype, shape_xyz, strides, mins)
    keep = np.zeros(int(np.prod(shape_xyz)) if dense else 16, dtype)
    b.buf.host = keep.ctypes.data
    b.buf.flags = 0
    b._keep = keep
    return b


def _planar(hb):
    """(name, buffer shapes (x, y, ...) and dtypes, call) per planar entry point: valid shapes, dense strides."""
    l = hb.load_library()
    u16, u8, f32 = np.uint16, np.uint8, np.float32
    m = ((4, 3), f32)

    def ll(fn):
        return lambda bi, bo: fn(bi.ptr, 8, ctypes.c_float(1 / 7), ctypes.c_float(1.0), bo.ptr)
    return {
        "halide_blur": ([((W + 2, H + 2), u16), ((W, H), u16)], lambda bi, bo: l.halide_blur(bi.ptr, bo.ptr)),
        "local_laplacian": ([((W, H, 3), u16)] * 2, ll(l.local_laplacian)),
        "local_laplacian_batch": ([((W, H, 3, 2), u16)] * 2, ll(l.halide_b200_local_laplacian_batch)),
        "local_laplacian_u8": ([((W, H, 3), u8)] * 2, ll(l.halide_b200_local_laplacian_u8)),
        "local_laplacian_u8_batch": ([((W, H, 3, 2), u8)] * 2, ll(l.halide_b200_local_laplacian_u8_batch)),
        "local_laplacian_pyramid_levels": ([((W, H, 3), u16)] * 2, lambda bi, bo: l.halide_b200_local_laplacian_pyramid_levels(
            bi.ptr, 4, 8, ctypes.c_float(1 / 7), ctypes.c_float(1.0), bo.ptr)),
        "bilateral_grid": ([((W, H), f32)] * 2, lambda bi, bo: l.bilateral_grid(bi.ptr, ctypes.c_float(0.1), bo.ptr)),
        "bilateral_grid_s_sigma": ([((W, H), f32)] * 2, lambda bi, bo: l.halide_b200_bilateral_grid_s_sigma(
            bi.ptr, 3, ctypes.c_float(0.1), bo.ptr)),
        "nl_means": ([((W, H, 3), f32)] * 2, lambda bi, bo: l.nl_means(bi.ptr, 3, 7, ctypes.c_float(0.12), bo.ptr)),
        "stencil_chain": ([((W, H), u16)] * 2, lambda bi, bo: l.stencil_chain(bi.ptr, bo.ptr)),
        "stencil_chain_stencils": ([((W, H), u16)] * 2, lambda bi, bo: l.halide_b200_stencil_chain_stencils(bi.ptr, 5, bo.ptr)),
        "camera_pipe": ([((96, 64), u16), m, m, ((32, 16, 3), u8)], lambda br, b32, b70, bo: l.camera_pipe(
            br.ptr, b32.ptr, b70.ptr, ctypes.c_float(3700), ctypes.c_float(2), ctypes.c_float(50), ctypes.c_float(1), 25, 1023,
            bo.ptr)),
        "conv_layer_any_shape": ([((5, 6, 6, 1), f32), ((7, 3, 3, 5), f32), ((7,), f32), ((7, 4, 4, 1), f32)],
                                 lambda bi, bf, bb, bo: l.halide_b200_conv_layer_any_shape(bi.ptr, bf.ptr, bb.ptr, bo.ptr)),
    }


PLANAR = ["halide_blur", "local_laplacian", "local_laplacian_batch", "local_laplacian_u8", "local_laplacian_u8_batch",
          "local_laplacian_pyramid_levels", "bilateral_grid", "bilateral_grid_s_sigma", "nl_means", "stencil_chain",
          "stencil_chain_stencils", "camera_pipe", "conv_layer_any_shape"]


@pytest.mark.parametrize("stride0", [-1, 0])
@pytest.mark.parametrize("name", PLANAR)
def test_planar_entry_points_refuse_innermost_stride(hb, name, stride0):
    """Each buffer of the call in turn gets dim[0].stride = -1 or 0: -8, and the message names the stride.  The same call
    on dense buffers gets past the shape and bounds checks (it runs, or fails later for want of a device), so the
    refusal is the stride's alone."""
    shapes, call = _planar(hb)[name]
    with hb.capture_errors() as err:
        rc = call(*[_buf(hb, t, s, dense=True) for s, t in shapes])
    assert rc not in (CONSTRAINT_VIOLATED, OUT_OF_BOUNDS) and "stride" not in err.msg, (name, rc, err.msg)
    for k in range(len(shapes)):
        bufs = [_buf(hb, t, s) for s, t in shapes]
        bufs[k].dims[0].stride = stride0
        with hb.capture_errors() as err:
            rc = call(*bufs)
        assert rc == CONSTRAINT_VIOLATED, (name, k, rc, err.msg)
        assert f"stride.0 ({stride0}) == 1" in err.msg, err.msg


IL = ["halide_b200_local_laplacian_interleaved", "halide_b200_local_laplacian_interleaved_batch",
      "halide_b200_local_laplacian_u8_interleaved", "halide_b200_local_laplacian_u8_interleaved_batch"]


@pytest.mark.parametrize("stride", [-1, 0])
@pytest.mark.parametrize("dim", [1, 3])
@pytest.mark.parametrize("fn", IL)
def test_interleaved_entry_points_refuse_non_positive_row_and_frame_strides(hb, fn, dim, stride):
    """Interleaved (x, y, c[, n]) buffers with strides (3, 3W, 1[, 3WH]): a row stride (dim 1) or frame stride (dim 3)
    negated or 0, on the input or the output, is refused with -8 (the header: "dim[1].stride (and dim[3].stride)
    positive")."""
    batch = fn.endswith("batch")
    if dim == 3 and not batch:
        pytest.skip("no frame dimension")
    dtype = np.uint8 if "_u8_" in fn else np.uint16
    shape = (W, H, 3, 2) if batch else (W, H, 3)
    dense = (3, 3 * W, 1, 3 * W * H)[:len(shape)]
    bad = stride * dense[dim]  # -1: the row (frame) order reversed; 0: one row (frame) repeated
    for k in range(2):
        bufs = [_buf(hb, dtype, shape, dense) for _ in range(2)]
        bufs[k].dims[dim].stride = bad
        with hb.capture_errors() as err:
            rc = getattr(hb.load_library(), fn)(bufs[0].ptr, 8, ctypes.c_float(1 / 7), ctypes.c_float(1.0), bufs[1].ptr)
        assert rc == CONSTRAINT_VIOLATED, (fn, k, rc, err.msg)
        assert f"stride.{dim} ({bad}) > 0" in err.msg, err.msg


@pytest.mark.parametrize("which,dim", [(0, 1), (0, 2), (0, 3), (1, 3), (3, 1), (3, 2)])
def test_conv_layer_refuses_negative_strides(hb, which, dim):
    """conv_layer's buffers are its fixed shapes, densely packed: a negative stride on the input, filter or output is a
    constraint violation that names it."""
    CI, CO, WW, HH, N = 128, 128, 100, 80, 5
    shapes = [(CI, WW + 2, HH + 2, N), (CO, 3, 3, CI), (CO,), (CO, WW, HH, N)]

    def dense(s):
        return [int(np.prod(s[:d])) for d in range(len(s))]
    bufs = [_buf(hb, np.float32, s, dense(s)) for s in shapes]
    bufs[which].dims[dim].stride = -dense(shapes[which])[dim]
    name = ["input", "filter", "bias", "relu"][which]
    with hb.capture_errors() as err:
        rc = hb.load_library().conv_layer(*(b.ptr for b in bufs))
    assert rc == CONSTRAINT_VIOLATED, (rc, err.msg)
    assert err.msg.startswith(f"Constraint violated: {name}.dim({dim})") and f"stride {-dense(shapes[which])[dim]}" in err.msg, \
        err.msg
