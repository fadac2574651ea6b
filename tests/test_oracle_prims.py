"""CPU tests pinning the oracle's primitives (SURVEY.md Appendix A) and the blur oracle against
the reference's own C implementation (oracle/_ref, built from apps/blur/test.cpp)."""
import math

import numpy as np
import pytest


def test_euclidean_div_mod(oracle):
    l = oracle.lib()
    # src/IROperator.h:253-311: a/b rounds toward -inf for b>0, 0 <= a%b < |b|, x/0 == 0, x%0 == 0
    for a in range(-9, 10):
        for b in (1, 2, 3, 8):
            assert l.oracle_div_floor(a, b) == a // b
            assert l.oracle_mod_floor(a, b) == a % b
    assert l.oracle_div_floor(-1, 2) == -1 and l.oracle_mod_floor(-1, 2) == 1
    assert l.oracle_div_floor(5, 0) == 0 and l.oracle_mod_floor(5, 0) == 0


def _ulps(a, b):
    ia = np.float32(a).view(np.int32).astype(np.int64)
    ib = np.float32(b).view(np.int32).astype(np.int64)
    return abs(int(ia) - int(ib))


def test_halide_exp_log_accuracy_bounds(oracle):
    # test/correctness/vector_math.cpp:548-640: exp within 32, fast_exp within 64 mantissa units of libm
    l = oracle.lib()
    for x in np.linspace(-20, 20, 401, dtype=np.float32):
        assert _ulps(l.oracle_halide_exp(float(x)), np.exp(np.float32(x))) <= 32, x
    for x in np.linspace(-10, 10, 201, dtype=np.float32):
        assert _ulps(l.oracle_fast_exp(float(x)), np.exp(np.float32(x))) <= 64 * 4, x  # loose: degree-5 poly
    for x in np.geomspace(1e-6, 1e6, 200, dtype=np.float32):
        got = l.oracle_halide_log(float(x))
        assert abs(got - math.log(float(x))) <= 2e-6 * max(1.0, abs(math.log(float(x)))), x
    assert l.oracle_halide_exp(0.0) == 1.0
    assert l.oracle_halide_exp(-200.0) == 0.0 and math.isinf(l.oracle_halide_exp(200.0))
    assert math.isnan(l.oracle_halide_log(-1.0)) and l.oracle_halide_log(0.0) == -math.inf
    assert l.oracle_halide_pow(0.0, 2.2) == 0.0 and l.oracle_halide_pow(3.0, 0.0) == 1.0
    assert abs(l.oracle_halide_pow(2.0, 0.5) - math.sqrt(2.0)) < 1e-6


def test_folded_constants_match_device_constants():
    # hl_math.cuh hard-codes logf(2), 1/logf(2) and float(1.0/65535.0); check them against numpy f32
    ln2 = np.float32(np.log(np.float32(2.0)))
    assert ln2.view(np.uint32) == 0x3F317218
    assert (np.float32(1.0) / ln2).view(np.uint32) == 0x3FB8AA3B
    assert np.float32(1.0 / float(ln2)).view(np.uint32) == 0x3FB8AA3B  # fast_exp's x / logf(2) fold
    assert np.float32(1.0 / 65535.0) == np.float32(1.525902189314365386962890625e-05)


def test_remap_lut_is_odd_and_matches_closed_form(oracle):
    l = oracle.lib()
    alpha = np.float32(1.0 / 7.0)
    for i in (-1792, -300, -1, 0, 1, 255, 256, 1792):
        v = l.oracle_ll_remap(i, float(alpha))
        assert v == -l.oracle_ll_remap(-i, float(alpha))
        fx = i / 256.0
        assert abs(v - float(alpha) * fx * math.exp(-fx * fx / 2)) < 1e-6


def test_blur_oracle_matches_numpy_wraparound(oracle):
    rng = np.random.default_rng(3)
    a = rng.integers(0, 65536, (37, 53), dtype=np.uint16)  # full range: sums wrap mod 2^16
    got = oracle.blur(a)
    bx = ((a[:, :-2] + a[:, 1:-1]) + a[:, 2:]) // np.uint16(3)
    want = ((bx[:-2] + bx[1:-1]) + bx[2:]) // np.uint16(3)
    assert got.dtype == np.uint16 and np.array_equal(got, want)


@pytest.mark.parametrize("fast", [False, True])
def test_blur_oracle_matches_reference_c_implementation(oracle, fast):
    """apps/blur/test.cpp:165-191 compares on 12-bit inputs (rand() & 0xfff); so do we, against the
    reference's own code compiled into oracle/_ref/libref_blur.so — or, where that is not built, what it returned for
    this input (tests/golden/reference_digests.json)."""
    from util import array_digest, reference_digest
    rng = np.random.default_rng(11)
    a = (rng.integers(0, 65536, (98, 264), dtype=np.uint16) & 0xFFF).astype(np.uint16)
    got = oracle.blur(a)[:, : a.shape[1] - 8]   # oracle computes w-2 columns; the reference's C blur w-8
    if not oracle.ref_blur_available():
        assert array_digest(got) == reference_digest(f"ref_blur/98x264/{int(fast)}")
        return
    want = oracle.ref_blur(a, fast)             # [h-2, w-8]
    assert np.array_equal(got, want)


def test_local_laplacian_oracle_properties(oracle):
    # identity-ish behaviour: alpha = 0, beta = 1 makes remap == 0 so every gPyramid[0] plane equals
    # gray and the filter returns the input up to the f32 round trip of the colour ratio.
    rng = np.random.default_rng(5)
    img = rng.integers(2000, 60000, (3, 40, 56), dtype=np.uint16)
    out = oracle.local_laplacian(img, 8, 0.0, 1.0)
    assert np.max(np.abs(out.astype(np.int64) - img.astype(np.int64))) <= 40
    # constant frames stay constant (all pyramid levels are flat)
    flat = np.full((3, 33, 47), 30000, np.uint16)
    o2 = oracle.local_laplacian(flat, 8, 1.0 / 7.0, 1.0)
    assert len(np.unique(o2)) == 1 and abs(int(o2[0, 0, 0]) - 30000) <= 1000


def test_strict_float_switch_builds_and_stays_close():
    """oracle/Makefile also builds the restatement with Halide's `strict_float` semantics (x / c stays a divide instead of
    x * fold(1/c), src/Simplify_Div.cpp:204 vs src/StrictifyFloat.cpp): the switch SURVEY.md §8c asks to keep.  It is not
    the parity target; it must build, run, and differ from the default realisation by at most a rare +-1 LSB."""
    import ctypes

    import numpy as np

    from oracle import pyoracle
    strict = pyoracle.strict_float_lib()
    rng = np.random.default_rng(5)
    img = rng.integers(0, 65536, (3, 64, 96), dtype=np.uint16)
    want = pyoracle.local_laplacian(img, 8, 1.0 / 7.0, 1.0)
    out = np.zeros_like(img)
    r = strict.oracle_local_laplacian(ctypes.byref(pyoracle.image(img)), ctypes.c_int(8), ctypes.c_float(1.0 / 7.0), ctypes.c_float(1.0),
                                      ctypes.byref(pyoracle.image(out)), ctypes.c_int(8))
    assert r == 0
    diff = np.abs(out.astype(np.int64) - want.astype(np.int64))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.02
