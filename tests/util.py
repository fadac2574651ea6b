"""Shared helpers for the parity tests: seeded synthetic frames, C-ABI call wrappers and the stored digests of what the
reference produced."""
import hashlib
import json
import os
from contextlib import contextmanager

import numpy as np

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests.json")


def array_digest(a):
    """SHA-256 of an array's type, shape and bytes: the form in which golden/reference_digests.json holds what the reference
    produced (golden/make_reference_digests.py)."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str} {a.shape}".encode() + a.tobytes()).hexdigest()


def bytes_digest(b):
    return hashlib.sha256(b).hexdigest()


def reference_digest(key):
    with open(DIGESTS) as f:
        return json.load(f)[key]


def u16_frame(shape, seed, bits=16):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 16, shape, dtype=np.uint16)
    if bits < 16:
        a &= np.uint16((1 << bits) - 1)
    return a


def smooth_u16_frame(shape, seed):
    """Low-frequency content + mild noise: exercises coherent LUT / plane selection paths."""
    rng = np.random.default_rng(seed)
    c, h, w = shape
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = np.empty(shape, np.uint16)
    for ch in range(c):
        base = 0.5 + 0.45 * np.sin(xx / (7.0 + ch) + seed) * np.cos(yy / (11.0 - ch))
        base += rng.normal(0, 0.02, (h, w))
        out[ch] = np.clip(base * 65535.0, 0, 65535).astype(np.uint16)
    return out


def f32_frame(shape, seed):
    rng = np.random.default_rng(seed)
    return rng.random(shape, dtype=np.float32)


@contextmanager
def kernels_run(hb):
    """Collects {kernel name: (launches, ms)} of the launches made inside the block (the library's profile mode), so a
    test can assert which kernel variant a call took."""
    report = {}
    hb.lib.profile_reset()
    hb.lib.profile(True)
    try:
        yield report
        report.update(hb.lib.profile_report())
    finally:
        hb.lib.profile(False)
        hb.lib.profile_reset()


@contextmanager
def nl_means_variant(hb, v):
    """halide_b200_nl_means_variant(v) for the duration of the block (1 = nl_means's generic kernel for every patch /
    search size), then the default (0) again."""
    l = hb.load_library()
    l.halide_b200_nl_means_variant(v)
    try:
        yield
    finally:
        l.halide_b200_nl_means_variant(0)


# ---- camera_pipe ---------------------------------------------------------------------------------------------------
# The harness's colour matrices (apps/camera_pipe/process.cpp:43-49), its scalar arguments, and each scalar at the
# extremes the filter accepts, one at a time.  Left out: a zero or non-finite color_temp, whose matrix entries convert inf
# or NaN to int16, which Halide leaves undefined (the GPU saturates, x86 gives INT_MIN), so the oracle and the kernel may
# both be right and still disagree.  Zero and non-finite gamma, contrast and sharpen_strength are defined in both copies
# (halide_exp's exponent goes through exp_k, NaN -> 0 and clamped) and test_hl_math_gpu.py checks their tables bit for
# bit; they stay out of this list because the float64 formulas of test_camera_pipe_tables.py mean nothing there.
CP_M3200 = np.array([[1.6697, -0.2693, -0.4004, -42.4346], [-0.3576, 1.0615, 1.5949, -37.1158],
                     [-0.2175, -1.8751, 6.9640, -26.6970]], np.float32)
CP_M7000 = np.array([[2.2997, -0.4478, 0.1706, -39.0923], [-0.3826, 1.5906, -0.2080, -25.4311],
                     [-0.0888, -0.7344, 2.2832, -20.0826]], np.float32)
CP_DEFAULTS = dict(color_temp=3700.0, gamma=2.0, contrast=50.0, sharpen=1.0, black=25, white=1023)
CP_EXTREMES = ([dict(color_temp=t) for t in (3200.0, 7000.0, 1000.0, 2000.0, 20000.0, 1e5)] +
               [dict(gamma=g) for g in (0.25, 0.5, 1.0, 4.0, 10.0)] +
               [dict(contrast=c) for c in (-100.0, 0.0, 100.0, 200.0)] +
               [dict(sharpen=s) for s in (-1.0, 0.0, 0.03, 1 / 32, 7.96875, 100.0)] +
               [dict(black=b, white=w) for b, w in ((0, 1023), (0, 1), (1022, 1023), (25, 4000), (-100, 1023), (500, 500),
                                                    (600, 400))])


def cp_params(overrides):
    """CP_DEFAULTS with `overrides` applied, as the filter's positional scalars (color_temp .. whiteLevel)."""
    p = dict(CP_DEFAULTS, **overrides)
    return (p["color_temp"], p["gamma"], p["contrast"], p["sharpen"], p["black"], p["white"])


def cp_param_id(overrides):
    return ",".join(f"{k}={v:g}" for k, v in overrides.items()) or "defaults"


def cp_matrix_q88(m3200, m7000, color_temp):
    """The Q8.8 colour matrix camera_pipe derives for `color_temp`, restated in float32 (alpha from the folded reciprocal
    of 1/7000 - 1/3200, as the generator's simplifier leaves it), after asserting the two limits inside which Halide
    defines the result: every val * 256 converts to int16 without overflow, and each row's magnitudes sum below 2^16, so
    m3 + m0 * r + m1 * g + m2 * b stays inside int32 for any int16 r, g, b."""
    f = np.float32
    c3200 = f(1) / f(3200)
    inv_c_diff = f(1.0 / float(f(1) / f(7000) - c3200))
    alpha = (f(1) / f(color_temp) - c3200) * inv_c_diff
    scaled = (np.asarray(m3200, f) * alpha + np.asarray(m7000, f) * (f(1) - alpha)) * f(256)
    assert (scaled > -32769).all() and (scaled < 32768).all(), f"matrix * 256 leaves int16 at color_temp {color_temp}"
    q = np.trunc(scaled).astype(np.int64)
    assert (np.abs(q).sum(axis=1) < 1 << 16).all(), f"matrix rows may overflow int32 at color_temp {color_temp}"
    return q


def run_blur(hb, inp, out_shape, in_mins=None, out_mins=None):
    out = np.zeros(out_shape, np.uint16)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.halide_blur(bi, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out


def run_local_laplacian(hb, inp, levels, alpha, beta, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.uint16)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.local_laplacian(bi, levels, alpha, beta, bo)
    bo.copy_to_host()
    return out
