"""local_laplacian at any pyramid depth on batch, 8-bit and pixel-interleaved frames: the seven forms of
:func:`halide_b200.filters.local_laplacian_pyramid_levels`, one per fixed-depth entry point it generalises (same names
with ``_pyramid_levels`` inserted, arguments ``(input, pyramid_levels, levels, alpha, beta, output)``).  Each frame is, bit
for bit, ``local_laplacian_pyramid_levels`` on a planar uint16 copy (8-bit frames converted as
``local_laplacian_u8`` converts them); J = 8 is the fixed-depth entry point, with the same launches."""
import ctypes

from .filters import _INTERLEAVED_LAYOUT
from .lib import lib, check


def _call(entry, input, pyramid_levels, levels, alpha, beta, output):
    return check(entry(input.ptr, ctypes.c_int32(pyramid_levels), ctypes.c_int32(levels), ctypes.c_float(alpha),
                       ctypes.c_float(beta), output.ptr))


def local_laplacian_pyramid_levels_batch(input, pyramid_levels, levels, alpha, beta, output):
    """local_laplacian_batch with the pyramid depth J chosen per call, 1 <= J <= 20: output frame n =
    local_laplacian_pyramid_levels(input frame n, J), bit for bit, in one launch sequence for the whole batch.  Buffers
    and error codes as local_laplacian_batch; J = 8 is local_laplacian_batch itself."""
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_batch, input, pyramid_levels, levels, alpha, beta,
                 output)


def local_laplacian_pyramid_levels_u8(input, pyramid_levels, levels, alpha, beta, output):
    """local_laplacian_u8 with the pyramid depth J chosen per call, 1 <= J <= 20: output =
    to_u8(local_laplacian_pyramid_levels(to_u16(input), J)) bit for bit, with local_laplacian_u8's conversions done inside
    the kernels.  Buffers and error codes as local_laplacian_u8; J = 8 is local_laplacian_u8 itself."""
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_u8, input, pyramid_levels, levels, alpha, beta, output)


def local_laplacian_pyramid_levels_u8_batch(input, pyramid_levels, levels, alpha, beta, output):
    """local_laplacian_u8_batch with the pyramid depth J chosen per call, 1 <= J <= 20: output frame n =
    local_laplacian_pyramid_levels_u8(input frame n, J).  Buffers and error codes as local_laplacian_u8_batch; J = 8 is
    local_laplacian_u8_batch itself."""
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_u8_batch, input, pyramid_levels, levels, alpha, beta,
                 output)


def local_laplacian_pyramid_levels_interleaved(input, pyramid_levels, levels, alpha, beta, output):
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_interleaved, input, pyramid_levels, levels, alpha,
                 beta, output)


def local_laplacian_pyramid_levels_interleaved_batch(input, pyramid_levels, levels, alpha, beta, output):
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_interleaved_batch, input, pyramid_levels, levels,
                 alpha, beta, output)


def local_laplacian_pyramid_levels_u8_interleaved(input, pyramid_levels, levels, alpha, beta, output):
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_u8_interleaved, input, pyramid_levels, levels, alpha,
                 beta, output)


def local_laplacian_pyramid_levels_u8_interleaved_batch(input, pyramid_levels, levels, alpha, beta, output):
    return _call(lib.halide_b200_local_laplacian_pyramid_levels_u8_interleaved_batch, input, pyramid_levels, levels,
                 alpha, beta, output)


_J = " with the pyramid depth J chosen per call, 1 <= J <= 20 (J = 8: that entry point itself).\n"
local_laplacian_pyramid_levels_interleaved.__doc__ = "local_laplacian_interleaved" + _J + _INTERLEAVED_LAYOUT
local_laplacian_pyramid_levels_interleaved_batch.__doc__ = "local_laplacian_interleaved_batch" + _J + _INTERLEAVED_LAYOUT
local_laplacian_pyramid_levels_u8_interleaved.__doc__ = "local_laplacian_u8_interleaved" + _J + _INTERLEAVED_LAYOUT
local_laplacian_pyramid_levels_u8_interleaved_batch.__doc__ = "local_laplacian_u8_interleaved_batch" + _J + _INTERLEAVED_LAYOUT
