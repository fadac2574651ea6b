"""nl_means against the oracle bit for bit, on content where every search offset carries weight (nl_means_exact.CASES).

Both kernels perform the oracle's float operations in the oracle's order: d = ((0 + e0^2) + e1^2) + e2^2, the vertical
patch sum before the horizontal one, both ascending, search rows outer and dx inner, the same fast_exp, an IEEE divide,
and no contraction (the library builds with --fmad=false, the oracle with -ffp-contract=off).  So every case compares
with np.array_equal, NaN equal to NaN, and runs the default kernel choice and the generic kernel (variant 1 of
halide_b200_nl_means_variant), asserting which kernel ran.  test_nl_means_exact checks on the CPU that the content makes
a wrong offset, neighbour or patch window move the result far beyond rounding."""
import numpy as np
import pytest

import nl_means_exact as E
from halide_b200 import dist
from test_param_extremes_gpu import nl_nd, nl_variant
from util import kernels_run

pytestmark = pytest.mark.gpu
WINDOW = {(3, 7), (7, 7)}  # the (patch, search) pairs the default takes to the register-window kernel


def kernel(patch, search, variant):
    return "nl_means_window" if variant == 0 and (patch, search) in WINDOW else "nl_means"


def run(hb, inp, patch, search, sigma, variant, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros((3,) + inp.shape[1:] if out_shape is None else out_shape, np.float32)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    with nl_variant(hb, variant), kernels_run(hb) as ran:
        hb.filters.nl_means(bi, patch, search, sigma, bo)
    assert list(ran) == [kernel(patch, search, variant)], sorted(ran)
    bo.copy_to_host()
    return out


def same(got, want, what=""):
    assert got.shape == want.shape
    if not np.array_equal(got, want, equal_nan=True):
        bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
        i = np.unravel_index(bad.argmax(), bad.shape)
        pytest.fail(f"{what}: {bad.sum()} of {bad.size} samples differ, first at {i}: {got[i]!r} vs {want[i]!r}")


def check(hb, oracle, c):
    """Both kernels against the oracle on case c; returns the results by variant."""
    inp, kw = E.frame(c)
    want = oracle.nl_means(inp, c.patch, c.search, c.sigma, **kw)
    got = {v: run(hb, inp, c.patch, c.search, c.sigma, v, **kw) for v in (0, 1)}
    for v in (0, 1):
        same(got[v], want, f"{c.id} variant {v}")
    return inp, kw, want, got


@pytest.mark.parametrize("c", E.group("seams") + E.group("mins") + E.group("channels") + E.group("clamp"),
                         ids=lambda c: c.id)
def test_frames(hb, oracle, c):
    """Ragged frames around the 32 x 16 tile (1 to 97 wide, 1 to 33 high), output mins away from the input's on each
    side and below zero, an output larger than its input, an input smaller than the apron, inputs of 1, 2 and 4
    channels and one whose channels start at 1, and inputs in [-0.5, 1.5], whose results the final clamp cuts."""
    inp, _, want, _ = check(hb, oracle, c)
    if c.group == "clamp":
        assert (want == 0).mean() > 0.05 and (want == 1).mean() > 0.05


@pytest.mark.parametrize("c", E.group("grid"), ids=lambda c: c.id)
def test_patch_search_grid(hb, oracle, c):
    """Every patch in {1, 2, 3, 4, 5, 7, 9, 15, 31} with every search in {1, 2, 3, 4, 7, 8, 13, 31, 63}: even sizes
    make the windows asymmetric ([-n/2, n/2 - 1]), patch 1 a single pixel.  At search 1 the centre is the only offset,
    whose weight is 1, so the result is the input, clamped."""
    inp, kw, want, got = check(hb, oracle, c)
    if c.search == 1:
        assert "out_mins" not in kw
        same(got[0], np.clip(inp, 0, 1), "search 1 against clip(input)")


@pytest.mark.parametrize("c", E.group("dx"), ids=lambda c: c.id)
def test_dx_batches(hb, oracle, c):
    """The generic kernel batches a search row's dx offsets within 100 KB of shared memory: for each patch, the last
    search with one batch per row and the first with two, partial last batches, and shared memory either side of 48 KB
    (the opt-in).  The sides are restated from nl_nd and asserted, so a retuned budget fails here."""
    nd, smem = nl_nd(c.patch, c.search)
    sides = {  # (one batch per row, > 48 KB, partial last batch)
        (3, 7): (True, False, False), (3, 8): (True, True, False), (3, 17): (True, True, False),
        (3, 18): (False, True, True), (7, 14): (True, True, False), (7, 15): (False, True, True),
        (15, 9): (True, True, False), (15, 10): (False, True, True), (15, 11): (False, True, True),
        (31, 4): (True, True, False), (31, 5): (False, True, True), (9, 31): (False, True, True)}
    assert sides[(c.patch, c.search)] == (nd == c.search, smem > 48 * 1024, c.search % nd != 0)
    check(hb, oracle, c)


def test_sigma(hb, oracle):
    """sigma across its range, on each kernel:
    -0.12 gives +0.12's bits (only sigma^2 is used);
    1e-4 (on noise of amplitude 0.2) makes every off-centre weight underflow to exactly 0, so the result is the input,
    clamped (at the frame edges too: a clamped patch still differs from the centre's in a row or column);
    1e4 and inf make every weight 1 (or within rounding of it): the box mean over the search window;
    1e-20 makes every weight NaN (test_nl_means_exact.test_oracle_nan_weights_give_one); clamp(NaN, 0, 1) is 1.0 in
    the oracle, by Halide's compare-and-select min / max.  The kernels once gave 0.0 there: ptxas turned their
    fmaxf(fminf(v, 1), 0) into a saturating add, which maps NaN to 0."""
    res = {}
    for c in E.group("sigma"):
        inp, kw, want, got = check(hb, oracle, c)
        res[c.sigma] = got
        if c.sigma == 1e-20:
            assert (want == 1.0).all()
        if c.sigma == 1e-4:
            same(got[0], np.clip(inp, 0, 1), "sigma 1e-4 against clip(input)")
        if c.sigma >= 1e4:
            box = E.nl_means64(inp, c.patch, c.search, float("inf"), **kw)
            assert E.rel(got[0], box) <= E.oracle_bound(c.search)
    for v in (0, 1):
        same(res[-0.12][v], res[0.12][v], f"sigma -0.12 against 0.12, variant {v}")


# ---- config 4: 3840 x 2160 x 3, patch 3, search 7, sigma 0.12 ------------------------------------------------------

@pytest.fixture(scope="module")
def frame_4k(hb):
    """The whole sensitive frame and each kernel's whole-frame result."""
    c = E.group("config4")[0]
    inp = E.sensitive_frame(*c.shape, c.sigma, c.seed)
    return c, inp, {v: run(hb, inp, c.patch, c.search, c.sigma, v) for v in (0, 1)}


def test_4k_regions(oracle, frame_4k):
    """Regions of the whole-frame result, at the frame's corners and across 32 x 16 tile seams, against the oracle on
    the crop that determines each (footprint: search/2 + patch/2 = 4 pixels; margin 16)."""
    _, inp, whole = frame_4k
    for c in E.group("config4"):
        crop, kw = E.frame(c)
        ya, xa = kw["in_mins"][1], kw["in_mins"][0]
        want = oracle.nl_means(crop, c.patch, c.search, c.sigma, **kw)
        y0, x0 = (int(t) for t in c.id.split("_")[1:])
        n = E.REGION
        for v in (0, 1):
            same(whole[v][:, y0:y0 + n, x0:x0 + n], want[:, y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n], f"{c.id} variant {v}")


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_4k_row_bands(hb, frame_4k, world):
    """Row bands cut with dist.band_rows, each run alone with its mins over its rows plus dist.halo_rows of input, put
    together, equal the whole-frame call bit for bit.  With the halo one row short, some band differs: the content
    sees a halo error."""
    c, inp, whole = frame_4k
    h = inp.shape[1]
    above, below = dist.halo_rows("nl_means", patch_size=c.patch, search_area=c.search)
    assert (above, below) == (4, 4)
    for v in (0, 1):
        for short in (0, 1):
            out = np.empty_like(whole[v])
            for rank in range(world):
                lo, hi = dist.band_rows(rank, world, h)
                a, b = max(0, lo - above + short), min(h - 1, hi + below - short)
                band = np.ascontiguousarray(inp[:, a:b + 1])
                out[:, lo:hi + 1] = run(hb, band, c.patch, c.search, c.sigma, v, out_shape=(3, hi - lo + 1, inp.shape[2]),
                                        in_mins=(0, a, 0), out_mins=(0, lo, 0))
            if short:
                assert not np.array_equal(out, whole[v]), f"{world} bands, variant {v}: a short halo went unseen"
            else:
                same(out, whole[v], f"{world} bands, variant {v}")
