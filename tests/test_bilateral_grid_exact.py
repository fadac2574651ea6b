"""On the CPU, for the cases the bit-exact GPU tests of bilateral_grid run (bilateral_grid_exact.CASES): the premise that
makes s_sigma = 8 bit-exact holds on their content, the oracle agrees with an independent float64 restatement (and maps
NaN pixels to 1, as Halide's clamp does), and the row halo dist.halo_rows gives is the one the filter needs."""
import numpy as np
import pytest

import bilateral_grid_exact as E
from halide_b200 import dist


def bin_sums32(vals, zi, nb, order):
    """float32 sums [GH, GW, nb] of each cell's values by bin, in one order: "forward" (rows, then columns: the
    generator's), "reverse", or "split" (bg_hist_blurz: columns 0-3 and 4-7 of a cell summed apart, rows outer, then
    added)."""
    v32 = vals.astype(np.float32)
    bins = np.arange(nb)
    zero = np.float32(0)
    s = vals.shape[-1]

    def total(pixels):
        acc = np.zeros(vals.shape[:2] + (nb,), np.float32)
        for ry, rx in pixels:
            acc = acc + np.where(zi[:, :, ry, rx, None] == bins, v32[:, :, ry, rx, None], zero)
        return acc

    walk = [(ry, rx) for ry in range(s) for rx in range(s)]
    if order == "forward":
        return total(walk)
    if order == "reverse":
        return total(walk[::-1])
    return total([p for p in walk if p[1] < 4]) + total([p for p in walk if p[1] >= 4])


@pytest.mark.parametrize("c", [c for c in E.CASES if c.s == 8], ids=lambda c: c.id)
def test_s8_bin_sums_are_exact_in_any_order(c):
    """Every s_sigma = 8 case: after the clamp the frame holds multiples of 2^-16 in [0, 1], so a bin's 64 terms and
    every partial sum of them are multiples of 2^-16 below 2^6, 22 bits, exact in float32 (24).  The bin sums in the
    generator's order, in reverse, and as bg_hist_blurz's two 4-column halves all equal the float64 sums: the kernel's
    re-association cannot change a bit on this content."""
    assert 64 * 2 ** 16 < 2 ** 24
    inp, kw = E.frame(c)
    clamped = E.clamp01(inp.astype(np.float64))
    assert np.array_equal(clamped * 65536, np.round(clamped * 65536))
    vals, zi, _ = E.cells(inp, c.s, c.r_sigma, **kw)
    nb = E.params(c.r_sigma)[1] + 1
    exact = np.zeros(vals.shape[:2] + (nb,))
    for b in range(nb):
        exact[..., b] = np.where(zi == b, vals, 0.0).sum(axis=(2, 3))
    for order in ("forward", "reverse", "split"):
        got = bin_sums32(vals, zi, nb, order)
        assert np.array_equal(got.astype(np.float64), exact), order


def test_every_s8_case_is_dyadic():
    cs = [c for c in E.CASES if c.s == 8]
    assert cs and all(c.content["kind"] == "dyadic" for c in cs)
    assert all(c.kernels == E.KERNELS_8 for c in cs)
    assert all(c.kernels == E.KERNELS_S for c in E.CASES if c.s != 8)


@pytest.mark.parametrize("c", E.CASES, ids=lambda c: c.id)
def test_oracle_within_float64_bound(oracle, c):
    inp, kw = E.frame(c)
    got = oracle.bilateral_grid(inp, c.r_sigma, s_sigma=c.s, **kw)
    assert np.isfinite(got).all()
    assert E.rel(got, E.bilateral_grid64(inp, c.s, c.r_sigma, **kw)) <= E.oracle_bound(c.s)


def test_clamp01_selects():
    """NaN -> 1, +inf -> 1, -inf -> 0, -0.0 -> +0.0, and values inside [0, 1] unchanged."""
    v = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, 0.25, -3.0, 7.0, E.DENORMAL], np.float64)
    got = E.clamp01(v)
    assert np.array_equal(got, [1, 1, 0, 0, 0, 1, 0.25, 0, 1, float(E.DENORMAL)])
    assert not np.signbit(got[3])


@pytest.mark.parametrize("c", E.group("specials"), ids=lambda c: c.id)
def test_oracle_clamps_special_pixels_like_halide(oracle, c):
    """The specials frames hold NaN, +-inf and -0.0 pixels.  The oracle's output on them equals its output on the frame
    with those pixels replaced by what Halide's clamp makes of them (NaN and +inf -> 1, -inf and -0.0 -> 0), bit for
    bit, and bilateral_grid64 within the bound.  Mapping NaN to 0 instead, as a saturating add does, changes it."""
    inp, kw = E.frame(c)
    assert np.isnan(inp).any() and np.isposinf(inp).any() and np.isneginf(inp).any()
    assert ((inp == 0) & np.signbit(inp)).any()
    if c.s != 8:
        assert (inp == E.DENORMAL).any()
    want = oracle.bilateral_grid(inp, c.r_sigma, s_sigma=c.s, **kw)
    clamped = E.clamp01(inp.astype(np.float64)).astype(np.float32)
    assert np.array_equal(want, oracle.bilateral_grid(clamped, c.r_sigma, s_sigma=c.s, **kw))
    assert E.rel(want, E.bilateral_grid64(inp, c.s, c.r_sigma, **kw)) <= E.oracle_bound(c.s)
    nan_to_0 = np.where(np.isnan(inp), np.float32(0), clamped)
    assert not np.array_equal(want, oracle.bilateral_grid(nan_to_0, c.r_sigma, s_sigma=c.s, **kw))


@pytest.mark.parametrize("c", E.group("specials"), ids=lambda c: c.id)
def test_specials_sit_on_bin_boundaries(c):
    """The bin-boundary values put val * inv_r + 0.5 exactly on an integer, in float32, for every bin."""
    inv_r, zmax = E.params(c.r_sigma)
    vals = E.special_values(c.s, c.r_sigma)
    t = vals[(vals > E.DENORMAL) & (vals < 1)] * inv_r + np.float32(0.5)
    assert np.array_equal(t, np.round(t)) and sorted(t.astype(int)) == list(range(1, zmax + 1))


@pytest.mark.parametrize("s", range(1, 129))
def test_halo_rows_cover_the_derivation(s):
    """dist.halo_rows("bilateral_grid") gives 4 s rows each way; an output row reads 3 s - 1 + s / 2 above and
    4 s - 1 - s / 2 below (counted here over every row offset within a cell)."""
    above, below = dist.halo_rows("bilateral_grid", s_sigma=s)
    assert (above, below) == (4 * s, 4 * s)
    reach = []
    for y in range(-2 * s, 2 * s):
        yi = y // s
        first = (yi - 2) * s - s // 2          # first row of cell yi - 2
        last = (yi + 3) * s - s // 2 + s - 1   # last row of cell yi + 3
        reach.append((y - first, last - y))
    assert tuple(max(r) for r in zip(*reach)) == E.halo_derived(s)
    assert E.halo_derived(s)[0] <= above and E.halo_derived(s)[1] <= below


@pytest.mark.parametrize("s", [1, 2, 3, 5, 8, 16])
def test_halo_derivation_is_tight_in_float64(s):
    """On bilateral_grid64, output bands ending at rows = 0 and = 1 (mod s) and starting at a row = s - 1: computed from
    exactly the derived rows they equal the whole-frame result bit for bit; from one row fewer above, they do not.
    Below, one row fewer still gives the same bits (that row weighs nothing: E.halo_derived) and two rows fewer do
    not."""
    h, w = 12 * s + 5, 2 * s + 7
    inp = E.noise((h, w), 40 + s)
    whole = E.bilateral_grid64(inp, s, 0.1)
    above, below = E.halo_derived(s)
    for lo, hi in ((5 * s - 1, 6 * s), (5 * s - 1, 6 * s + 1)):
        def band(a, b):
            return E.bilateral_grid64(inp[a:b + 1], s, 0.1, out_shape=(hi - lo + 1, w), in_mins=(0, a),
                                      out_mins=(0, lo))

        want = whole[lo:hi + 1]
        assert 0 < lo - above and hi + below < h - 1
        assert np.array_equal(band(lo - above, hi + below), want)
        assert not np.array_equal(band(lo - above + 1, hi + below), want)
        # a band ending at a row = 1 (mod s) depends on every derived row but the last; one ending at a row = 0 (mod s)
        # (s > 1) on none of the last s, since its last row weighs no cell row past the one its row above reaches
        short_ok = 1 if hi % s == 1 % s else s
        assert np.array_equal(band(lo - above, hi + below - short_ok), want)
        assert not np.array_equal(band(lo - above, hi + below - short_ok - 1), want)
