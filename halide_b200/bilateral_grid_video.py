"""Python call sites of the batch bilateral_grid entry points (float32 and uint8): bilateral_grid on video clips,
``(N, H, W)`` tensors or arrays.

The one-frame entry points, ``bilateral_grid``, ``bilateral_grid_s_sigma`` and ``bilateral_grid_u8``, are in
:mod:`halide_b200.filters`; these take the same arguments and report errors the same way (a negative halide_error_code_t
becomes a :class:`HalideError`).  They live in a module of their own, as the clip entry points of nl_means do in
:mod:`halide_b200.nl_means_video`, because :mod:`halide_b200.filters` holds exactly the call sites that
tests/test_concurrent_callers_gpu.py runs as concurrent jobs (it checks that set, 23 functions, against its jobs)."""
import ctypes

from .filters import _U8_CONVERSIONS
from .lib import lib, check


def bilateral_grid_batch(input, r_sigma, output):
    return check(lib.halide_b200_bilateral_grid_batch(input.ptr, ctypes.c_float(r_sigma), output.ptr))


def bilateral_grid_s_sigma_batch(input, s_sigma, r_sigma, output):
    return check(lib.halide_b200_bilateral_grid_s_sigma_batch(input.ptr, ctypes.c_int32(s_sigma), ctypes.c_float(r_sigma),
                                                              output.ptr))


def bilateral_grid_u8_batch(input, r_sigma, output):
    return check(lib.halide_b200_bilateral_grid_u8_batch(input.ptr, ctypes.c_float(r_sigma), output.ptr))


_BATCH = ("Output frame n is, bit for bit, {one}(input frame n); frames are independent.  output.dim[2].min selects the "
          "input frame each output frame reads, and the input's frames must cover the output's, else -4.  Rows may be "
          "padded, frames may be crops of a larger array, and the frame stride may be negative (a reversed clip) or, on "
          "the input, 0 (one frame for every output frame).  The frames run in groups whose two scratch grids stay "
          "within 256 MiB, three launches a group; frames so large that fewer than 3 fit (7680 x 4320 at r_sigma 0.1) "
          "run one at a time, three launches each.  Arguments, buffer rules and error codes as {one}.")
bilateral_grid_batch.__doc__ = ("bilateral_grid on every frame of 3-D (x, y, n) float32 buffers, e.g. an (N, H, W) "
                                "float32 torch tensor (a clip).\n" + _BATCH.format(one="bilateral_grid"))
bilateral_grid_s_sigma_batch.__doc__ = ("bilateral_grid_s_sigma on every frame of 3-D (x, y, n) float32 buffers, with "
                                        "the same s_sigma (1 <= s_sigma <= 128) for every frame.\n" +
                                        _BATCH.format(one="bilateral_grid_s_sigma"))
bilateral_grid_u8_batch.__doc__ = ("bilateral_grid_u8 on every frame of 3-D (x, y, n) uint8 buffers, e.g. a decoded "
                                   "(N, H, W) uint8 clip.\n" + _BATCH.format(one="bilateral_grid_u8") + _U8_CONVERSIONS)
