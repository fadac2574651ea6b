"""Python call sites of the batch and interleaved nl_means entry points (float32 and uint8): nl_means on video clips,
``(N, 3, H, W)`` tensors, and on pixel-interleaved frames, ``(H, W, 3)`` arrays and ``channels_last`` tensors.

The one-frame planar entry points, ``nl_means`` and ``nl_means_u8``, are in :mod:`halide_b200.filters`; these take the
same arguments and report errors the same way (a negative halide_error_code_t becomes a :class:`HalideError`)."""
import ctypes

from .filters import _INTERLEAVED_LAYOUT, _U8_CONVERSIONS
from .lib import lib, check


def _nl_means_args(patch_size, search_area, sigma):
    return ctypes.c_int32(patch_size), ctypes.c_int32(search_area), ctypes.c_float(sigma)


def nl_means_batch(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_batch(input.ptr, *_nl_means_args(patch_size, search_area, sigma), output.ptr))


def nl_means_interleaved(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_interleaved(input.ptr, *_nl_means_args(patch_size, search_area, sigma), output.ptr))


def nl_means_interleaved_batch(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_interleaved_batch(input.ptr, *_nl_means_args(patch_size, search_area, sigma),
                                                            output.ptr))


def nl_means_u8_batch(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_u8_batch(input.ptr, *_nl_means_args(patch_size, search_area, sigma), output.ptr))


def nl_means_u8_interleaved(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_u8_interleaved(input.ptr, *_nl_means_args(patch_size, search_area, sigma),
                                                         output.ptr))


def nl_means_u8_interleaved_batch(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_u8_interleaved_batch(input.ptr, *_nl_means_args(patch_size, search_area, sigma),
                                                               output.ptr))


_NL_MEANS_BATCH = ("Output frame n is, bit for bit, {one}(input frame n), with x, y and c clamped inside each frame; the "
                   "input's frames must cover the output's, else -4.  Every frame runs in one launch.  Arguments, buffer "
                   "rules (output channels exactly [0, 3)) and error codes as {one}.")
nl_means_batch.__doc__ = ("nl_means on every frame of 4-D (x, y, c, n) float32 buffers, e.g. an (N, 3, H, W) float32 "
                          "torch tensor (a clip).\n" + _NL_MEANS_BATCH.format(one="nl_means"))
nl_means_u8_batch.__doc__ = ("nl_means_u8 on every frame of 4-D (x, y, c, n) uint8 buffers, e.g. a decoded (N, 3, H, W) "
                             "uint8 clip.\n" + _NL_MEANS_BATCH.format(one="nl_means_u8") + _U8_CONVERSIONS)
nl_means_interleaved.__doc__ = ("nl_means on 3-D (x, y, c) float32 interleaved buffers (an RGBA input's alpha is never "
                                "read; the output's channels are exactly [0, 3)).\n" + _INTERLEAVED_LAYOUT)
nl_means_interleaved_batch.__doc__ = ("nl_means_batch on 4-D (x, y, c, n) float32 interleaved buffers, e.g. an (N, 3, H, W) "
                                      "channels_last tensor.\n" + _INTERLEAVED_LAYOUT)
nl_means_u8_interleaved.__doc__ = ("nl_means_u8 on 3-D (x, y, c) uint8 interleaved buffers, e.g. a decoded (H, W, 3) photo."
                                   "\n" + _INTERLEAVED_LAYOUT + _U8_CONVERSIONS)
nl_means_u8_interleaved_batch.__doc__ = ("nl_means_u8_batch on 4-D (x, y, c, n) uint8 interleaved buffers, e.g. a decoded "
                                         "(N, 3, H, W) channels_last clip.\n" + _INTERLEAVED_LAYOUT + _U8_CONVERSIONS)
