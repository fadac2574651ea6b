"""Python call site of the batch blur entry point: halide_blur on video clips, ``(N, H, W)`` uint16 tensors or arrays.

The one-frame entry point, ``halide_blur``, is in :mod:`halide_b200.filters`; this takes the same buffers and reports
errors the same way (a negative halide_error_code_t becomes a :class:`HalideError`).  It lives in a module of its own, as
the clip entry points of the other filters do, because :mod:`halide_b200.filters` holds exactly the call sites that
tests/test_concurrent_callers_gpu.py runs as concurrent jobs (it checks that set, 23 functions, against its jobs)."""
from .lib import lib, check


def blur_batch(input, blur_y):
    """halide_blur on every frame of 3-D (x, y, n) uint16 buffers, e.g. an (N, H, W) uint16 torch tensor (a clip).

    Output frame n is, bit for bit, halide_blur(input frame n); frames are independent.  blur_y.dim[2].min selects the
    input frame each output frame reads, and the input's frames must cover the output's, else -4 naming dimension 2.  In
    x and y the input must cover [ox, ox + W + 1] x [oy, oy + H + 1] of every output frame, else -4.  Rows may be padded,
    frames may be crops of a larger array, and the frame stride may be negative (a reversed clip) or, on the input, 0
    (one frame for every output frame).  The whole clip is one launch.  Buffer rules and error codes as halide_blur."""
    return check(lib.halide_b200_blur_batch(input.ptr, blur_y.ptr))
