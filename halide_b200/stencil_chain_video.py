"""Python call sites of the batch stencil_chain entry points: stencil_chain on video clips, ``(N, H, W)`` uint16 tensors
or arrays.

The one-frame entry points, ``stencil_chain`` and ``stencil_chain_stencils``, are in :mod:`halide_b200.filters`; these
take the same arguments and report errors the same way (a negative halide_error_code_t becomes a :class:`HalideError`).
They live in a module of their own, as the clip entry points of the other filters do, because
:mod:`halide_b200.filters` holds exactly the call sites that tests/test_concurrent_callers_gpu.py runs as concurrent jobs
(it checks that set, 23 functions, against its jobs)."""
import ctypes

from .lib import lib, check


def stencil_chain_batch(input, output):
    return check(lib.halide_b200_stencil_chain_batch(input.ptr, output.ptr))


def stencil_chain_stencils_batch(input, stencils, output):
    return check(lib.halide_b200_stencil_chain_stencils_batch(input.ptr, ctypes.c_int32(stencils), output.ptr))


_BATCH = ("Output frame n is, bit for bit, {one}(input frame n); frames are independent: repeat_edge applies in x and y "
          "within each frame, never across frames.  output.dim[2].min selects the input frame each output frame reads, "
          "and the input's frames must cover the output's, else -4 naming dimension 2; in x and y the input need only be "
          "non-empty.  Rows may be padded, frames may be crops of a larger array, and the frame stride may be negative "
          "(a reversed clip) or, on the input, 0 (one frame for every output frame).  The frames run in groups whose "
          "scratch planes stay within 256 MiB (at most 65 535 frames), ceil(stencils / 4) launches a group.  Arguments, "
          "buffer rules and error codes as {one}.")
stencil_chain_batch.__doc__ = ("stencil_chain (32 stages) on every frame of 3-D (x, y, n) uint16 buffers, e.g. an "
                               "(N, H, W) uint16 torch tensor (a clip).\n" + _BATCH.format(one="stencil_chain"))
stencil_chain_stencils_batch.__doc__ = ("stencil_chain_stencils on every frame of 3-D (x, y, n) uint16 buffers, with the "
                                        "same stencils (1 <= stencils <= 100) for every frame.\n" +
                                        _BATCH.format(one="stencil_chain_stencils"))
