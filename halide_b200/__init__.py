"""halide_b200 — H100-native drop-in for Halide's canonical apps/ pipelines.

The product is ``libhalide_b200.so``: hand-written sm_90a CUDA kernels behind the exact C ABI a
Halide AOT filter exports (``int local_laplacian(halide_buffer_t*, int, float, float,
halide_buffer_t*)`` ...; see ``include/*.h``).  This Python package is only the thin ctypes
binding the tests and ``bench.py`` use to call that C ABI; it contains no compute and no
fallback: importing :mod:`halide_b200.lib` raises if the shared library has not been built.
:mod:`halide_b200.image_io` is the host-side image reader / writer with the reference's
conversion rules (``tools/halide_image_io.h``), for natural-image runs of the filters.
"""
from .buffer import HalideBuffer, halide_buffer_t, halide_dimension_t  # noqa: F401
from .lib import lib as capi, load_library, HalideError, capture_errors  # noqa: F401
from . import lib  # noqa: F401  (module: loader + profile helpers)
from . import filters  # noqa: F401
from . import nl_means_video  # noqa: F401  (batch and interleaved nl_means)
from . import bilateral_grid_video  # noqa: F401  (batch bilateral_grid)
from . import blur_video  # noqa: F401  (batch halide_blur)
from . import stencil_chain_video  # noqa: F401  (batch stencil_chain)
from . import local_laplacian_depth  # noqa: F401  (local_laplacian at any pyramid depth on batch / 8-bit / interleaved frames)
from .pipeline import FramePipeline  # noqa: F401
from . import image_io  # noqa: F401  (host-side: file formats + the reference's type-conversion rules)
