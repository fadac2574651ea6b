"""ctypes binding of tests/ll_bordered_oracle.cpp — TEST INFRASTRUCTURE: local_laplacian at any pyramid depth with each
level stored only inside its constant border (same bits as the literal oracle, memory about the frame's).

The library is compiled on first use into a private temporary directory, with the parity flags of oracle/Makefile (no
FMA contraction, no fast-math), so the tree is never written to."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
# oracle/Makefile's CXX and CXXFLAGS: the float expressions must round exactly as in liboracle.so
_CXX = "/usr/bin/g++"
_CXXFLAGS = ["-O3", "-mavx2", "-fPIC", "-std=c++17", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall",
             "-Wno-unknown-pragmas"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="ll_bordered_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libll_bordered.so")
        subprocess.check_call([_CXX, *_CXXFLAGS, "-shared", "-I", _ORACLE, "-o", so,
                               os.path.join(_HERE, "ll_bordered_oracle.cpp")])
        _lib = ctypes.CDLL(so)
    return _lib


def local_laplacian(inp, levels, alpha, beta, out_shape=None, in_mins=None, out_mins=None, pyramid_levels=8):
    """As oracle.pyoracle.local_laplacian (inp: uint16 [c, h, w]), evaluated by oracle_local_laplacian_bordered."""
    from oracle import pyoracle
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.uint16)
    r = lib().oracle_local_laplacian_bordered(ctypes.byref(pyoracle.image(inp, in_mins)), ctypes.c_int(levels),
                                              ctypes.c_float(alpha), ctypes.c_float(beta),
                                              ctypes.byref(pyoracle.image(out, out_mins)), ctypes.c_int(pyramid_levels))
    if r != 0:
        raise RuntimeError(f"oracle_local_laplacian_bordered returned {r}")
    return out
