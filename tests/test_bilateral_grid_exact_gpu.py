"""bilateral_grid against the oracle bit for bit, on every case of bilateral_grid_exact.CASES.

The kernels perform the oracle's float operations in the oracle's order (bin sums rows then columns, the same blur5
association, the lerp nest x -> y -> z, an IEEE divide, no contraction: --fmad=false in the library, -ffp-contract=off in
the oracle) and clamp input pixels as Halide does, NaN to 1.  The one re-association, bg_hist_blurz's two 4-column halves
of a cell at s_sigma = 8, is exact on the dyadic frames every s_sigma = 8 case uses (test_bilateral_grid_exact checks
that premise on the CPU).  So every case compares with np.array_equal, NaN equal to NaN, and asserts which kernels ran."""
import numpy as np
import pytest

import bilateral_grid_exact as E
from halide_b200 import dist
from util import kernels_run

pytestmark = pytest.mark.gpu


def call(hb, bi, s, r_sigma, bo):
    """bilateral_grid itself at s = 8, halide_b200_bilateral_grid_s_sigma otherwise; asserts the kernels that ran."""
    with kernels_run(hb) as ran:
        if s == 8:
            hb.filters.bilateral_grid(bi, r_sigma, bo)
        else:
            hb.filters.bilateral_grid_s_sigma(bi, s, r_sigma, bo)
    assert set(ran) == E.kernels(s), sorted(ran)


def run(hb, inp, s, r_sigma, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.float32)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    call(hb, bi, s, r_sigma, bo)
    bo.copy_to_host()
    return out


def same(got, want, what="", inp=None):
    """Bit for bit, NaN equal to NaN; on failure names the first differing sample (and the input pixel there, for an
    output that starts where the input does)."""
    assert got.shape == want.shape
    if not np.array_equal(got, want, equal_nan=True):
        bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
        i = np.unravel_index(bad.argmax(), bad.shape)
        px = f", input {inp[i]!r}" if inp is not None and inp.shape == got.shape else ""
        pytest.fail(f"{what}: {bad.sum()} of {bad.size} samples differ, first at {i}: {got[i]!r} vs {want[i]!r}{px}")


@pytest.mark.parametrize("c", [c for c in E.CASES if c.group != "config3"], ids=lambda c: c.id)
def test_case(hb, oracle, c):
    """Frames from 1 x 1 to 240 x 519 at s_sigma 1 to 128; crops with negative, unaligned and mismatched mins, one
    starting inside a cell; r_sigma from 1 / 199 (200 bins) to inf (one bin); and frames holding NaN, +-inf, -0.0, the
    smallest denormal (not at s_sigma = 8), 0, 1 and values on bin boundaries at cell corners, interiors and edges."""
    inp, kw = E.frame(c)
    want = oracle.bilateral_grid(inp, c.r_sigma, s_sigma=c.s, **kw)
    same(run(hb, inp, c.s, c.r_sigma, **kw), want, c.id, inp)


@pytest.mark.parametrize("s", E.S_CONFIG3)
def test_8k_regions(hb, oracle, s):
    """7680 x 4320 (BASELINE.json config 3): regions of the whole-frame result, at the corners, the centre and off any
    alignment, against the oracle on the crop that determines each (margin 5 s: the blurs reach 2 cells, the slice 1);
    the crops keep their frame coordinates as mins, since cell boundaries are absolute."""
    cs = [c for c in E.group("config3") if c.s == s]
    whole = run(hb, E.content(cs[0]), s, cs[0].r_sigma)
    for c in cs:
        crop, kw = E.frame(c)
        ya, xa = kw["in_mins"][1], kw["in_mins"][0]
        y0, x0 = E.region(c)
        n = E.REGION
        want = oracle.bilateral_grid(crop, c.r_sigma, s_sigma=s, **kw)
        same(whole[y0:y0 + n, x0:x0 + n], want[y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n], c.id)


@pytest.mark.parametrize("s", [3, 8, 16])
def test_row_bands(hb, s):
    """Row bands cut with dist.band_rows (2, 3, 4 and 8 bands), each run alone over exactly the rows the derivation
    gives (3 s - 1 + s / 2 above, 4 s - 1 - s / 2 below), put together equal the whole-frame call bit for bit.  With one
    row fewer above, some band differs: the derivation is tight there.  Below, the last derived row is read but weighs
    nothing (yf = 0 on rows = 0 mod s: bilateral_grid_exact.halo_derived), so one row fewer gives the same bits and two
    rows fewer differ in some band.  The frame height puts band edges where each of these shows."""
    h, w = E.band_height(s), 523
    inp = E.dyadic((h, w), 70 + s) if s == 8 else E.noise((h, w), 70 + s)
    whole = run(hb, inp, s, 0.1)
    above, below = E.halo_derived(s)
    assert above + below <= 2 * dist.halo_rows("bilateral_grid", s_sigma=s)[0]
    differs = {"above": False, "below2": False}
    for world in E.BAND_WORLDS:
        for short, (da, db) in {"exact": (0, 0), "above": (1, 0), "below1": (0, 1), "below2": (0, 2)}.items():
            out = np.empty_like(whole)
            for rank in range(world):
                lo, hi = dist.band_rows(rank, world, h)
                a, b = max(0, lo - above + da), min(h - 1, hi + below - db)
                out[lo:hi + 1] = run(hb, np.ascontiguousarray(inp[a:b + 1]), s, 0.1, out_shape=(hi - lo + 1, w),
                                     in_mins=(0, a), out_mins=(0, lo))
            if short in differs:
                differs[short] |= not np.array_equal(out, whole)
            else:
                same(out, whole, f"{world} bands, halo {short}")
    assert all(differs.values()), f"a short halo went unseen: {differs}"


# (input pitch, input offset, output pitch, output offset), in floats; the frame is 133 wide
LAYOUTS = [(152, 0, 140, 0),   # 16-byte rows, aligned bases: the float4 paths
           (152, 1, 140, 3),   # misaligned bases: the scalar paths
           (141, 0, 137, 0),   # odd pitches: rows alternate between the two
           (152, 0, 141, 2),   # aligned input, odd output pitch and misaligned base
           (139, 3, 136, 0)]


@pytest.mark.parametrize("s", [3, 8, 16])
def test_device_layouts(hb, oracle, s):
    """Device-resident torch views with padded and odd row pitches and bases off 16-byte alignment, so both the float4
    and the scalar loads of the histogram and slice kernels run: bit for bit against the oracle, and the output's
    padding keeps its sentinel."""
    import torch
    h, w = 75, 133
    sentinel = -7.25
    for k, (pin, oin, pout, oout) in enumerate(LAYOUTS):
        base = E.dyadic((h, pin), 50 + k, spread=True) if s == 8 else E.noise((h, pin), 50 + k, spread=True)
        tin = torch.from_numpy(base).cuda()
        tout = torch.full((h, pout), sentinel, dtype=torch.float32, device="cuda")
        vin, vout = tin[:, oin:oin + w], tout[:, oout:oout + w]
        call(hb, hb.HalideBuffer.from_torch(vin), s, 0.1, hb.HalideBuffer.from_torch(vout))
        torch.cuda.synchronize()
        inp = np.ascontiguousarray(base[:, oin:oin + w])
        same(vout.cpu().numpy(), oracle.bilateral_grid(inp, 0.1, s_sigma=s), f"layout {k}", inp)
        pad = tout.cpu().numpy()
        assert (pad[:, :oout] == sentinel).all() and (pad[:, oout + w:] == sentinel).all(), f"layout {k}: padding written"
