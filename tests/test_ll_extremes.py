"""local_laplacian at extreme and non-finite alpha and beta on the CPU (ll_extremes.CASES): the C++ oracle and the numpy
restatement agree byte for byte on every case, the NaN-mixed cases keep their mix, and every case would show at least
one named mistake of the kind a kernel could make, so comparing bytes on these cases means something."""
import functools

import numpy as np
import pytest

import ll_extremes as E
from oracle import np_restatement as R

F = np.float32


def nan_to_zero(color):
    """The final clamp as a float-to-integer conversion would do it: NaN -> 0 (cvt.rzi, and numpy on x86)."""
    with np.errstate(invalid="ignore"):
        return np.maximum(np.minimum(color, F(65535.0)), F(0.0)).astype(np.uint16)


def lerp_one_mul(zero, one, w):
    """lerp as zero + (one - zero) * w: one multiply instead of Halide's zero * (1 - w) + one * w."""
    return zero + (one - zero) * w


def down4_paired(a, b, c, d):
    """The 1-3-3-1 tap with its outer and inner pairs summed first: ((a + d) + 3 * (b + c)) / 8."""
    return ((a + d) + F(3.0) * (b + c)) * F(0.125)


MUTATIONS = ("nan_to_zero", "lerp", "down4")


@functools.lru_cache(maxsize=None)
def results(case_id):
    """(colour, output, {mutation: output under it}) of the restatement on a case."""
    c = CASES[case_id]
    img = E.frame()
    color = R.local_laplacian_color(img, c.levels, c.alpha, c.beta)
    out = {"nan_to_zero": nan_to_zero(color)}
    mp = pytest.MonkeyPatch()
    try:
        for name, attr, fn in (("lerp", "_lerp", lerp_one_mul), ("down4", "_down4", down4_paired)):
            mp.setattr(R, attr, fn)
            out[name] = R.local_laplacian(img, c.levels, c.alpha, c.beta)
            mp.undo()
    finally:
        mp.undo()
    return color, R.clamp_u16(color), out


CASES = {c.id: c for c in E.CASES}


def test_clamp_selects_like_halide():
    """min(v, 65535) then max(., 0), each a compare-and-select: NaN and +inf give 65535, -inf and -0.0 give 0."""
    v = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 0.9, 65534.99, 65535.0, 1e30, -1.0], F)
    assert R.clamp_u16(v).tolist() == [65535, 65535, 0, 0, 0, 0, 65534, 65535, 65535, 0]


@pytest.mark.parametrize("c", E.CASES, ids=E.CASE_IDS)
def test_oracle_and_restatement_agree(oracle, c):
    _, want, _ = results(c.id)
    got = oracle.local_laplacian(E.frame(), c.levels, c.alpha, c.beta)
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} samples differ, first at {np.argwhere(bad)[0]}"


@pytest.mark.parametrize("c", E.mixed(), ids=lambda c: c.id)
def test_mixed_cases_keep_their_mix(c):
    """At least MIXED_SHARE of the colours are NaN, and as many are positive and negative (finite or infinite)."""
    color, out, _ = results(c.id)
    shares = {"nan": np.isnan(color).mean(), "positive": (color > 0).mean(), "negative": (color < 0).mean()}
    assert min(shares.values()) >= E.MIXED_SHARE, shares
    assert (out[np.isnan(color)] == 65535).all()


@pytest.mark.parametrize("c", E.CASES, ids=E.CASE_IDS)
def test_every_case_shows_a_mistake(c):
    """Under at least one of the mutations the case's output changes: a kernel making that mistake fails on it.  The
    saturated cases (ll_extremes.SATURATED) instead have every colour beyond [0, 65535], none NaN, and both signs."""
    color, out, mutated = results(c.id)
    changed = {m: int((mutated[m] != out).sum()) for m in MUTATIONS}
    if c.saturated:
        assert not any(changed.values()), changed
        assert not np.isnan(color).any() and not ((color > 0) & (color < 65535)).any()
        assert (out == 0).any() and (out == 65535).any()
    else:
        assert any(changed.values()), changed


def test_every_mutation_is_caught():
    """Each mutation changes the output of some case; the counts of cases it shows on are reported on failure."""
    seen = {m: [c.id for c in E.CASES if (results(c.id)[2][m] != results(c.id)[1]).any()] for m in MUTATIONS}
    assert all(seen.values()), {m: len(v) for m, v in seen.items()}
