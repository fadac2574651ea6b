"""GPU parity tests for stencil_chain through the C ABI: bit-exact uint16 (ring arithmetic mod 2^16)."""
import numpy as np
import pytest

from util import u16_frame

pytestmark = pytest.mark.gpu


def run(hb, inp, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.uint16)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.stencil_chain(bi, bo)
    bo.copy_to_host()
    return out


@pytest.mark.parametrize("h,w", [(1, 1), (5, 3), (17, 40), (64, 64), (65, 129), (200, 333)])
def test_matches_oracle(hb, oracle, h, w):
    inp = u16_frame((h, w), h * 7 + w)
    assert np.array_equal(run(hb, inp), oracle.stencil_chain(inp))


def test_small_values_no_wrap_first_stage_scale(hb, oracle):
    # a constant frame c maps to c * 225^32 mod 2^16 (sum of weights = 225 per stage)
    inp = np.full((70, 90), 3, np.uint16)
    got = run(hb, inp)
    assert (got == (3 * pow(225, 32, 1 << 16)) % (1 << 16)).all()


def test_output_larger_than_input_and_offsets(hb, oracle):
    """All input accesses are clamped, so the output may extend beyond the input (SURVEY.md §8b)."""
    inp = u16_frame((40, 50), 3)
    got = run(hb, inp, out_shape=(60, 80), in_mins=(3, -2), out_mins=(-10, -9))
    want = oracle.stencil_chain(inp, out_shape=(60, 80), in_mins=(3, -2), out_mins=(-10, -9))
    assert np.array_equal(got, want)


def test_harness_size_linearity(hb):
    """1536x2560 (the harness frame): the pipeline is linear over Z/2^16, so
    f(a + b) == f(a) + f(b) (mod 2^16) at full size without needing the oracle."""
    a = u16_frame((2560, 1536), 1)
    b = u16_frame((2560, 1536), 2)
    fa, fb, fab = run(hb, a), run(hb, b), run(hb, (a + b).astype(np.uint16))
    assert np.array_equal(fab, (fa + fb).astype(np.uint16))


def test_harness_size_regions_vs_oracle(hb, oracle):
    """1536 x 2560 (the harness frame) against the oracle by region: 32 stages of a 5x5 stencil reach 64 px, so the
    oracle on a crop with an 80 px margin (ending exactly at the frame edges it touches) determines the region."""
    h, w = 2560, 1536
    inp = u16_frame((h, w), 4)
    got = run(hb, inp)
    for (y0, x0) in [(0, 0), (h - 96, w - 96), (1200, 700), (2048 - 48, 1024 - 48)]:
        n, m = 96, 80
        ya, yb, xa, xb = max(0, y0 - m), min(h, y0 + n + m), max(0, x0 - m), min(w, x0 + n + m)
        crop = np.ascontiguousarray(inp[ya:yb, xa:xb])
        want = oracle.stencil_chain(crop, in_mins=(xa, ya), out_mins=(xa, ya))
        assert np.array_equal(got[y0:y0 + n, x0:x0 + n], want[y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n])


@pytest.mark.parametrize("seed", [100, 200])
def test_tile_kernel_edge_cases_match_oracle(hb, oracle, seed):
    """Ragged sizes, odd widths (odd row strides: the 16-bit load / store paths), an output larger than the input and a
    crop with odd offsets."""
    for h, w in ((1, 1), (17, 40), (65, 129), (200, 333), (130, 256)):
        inp = u16_frame((h, w), seed + h + w)
        assert np.array_equal(run(hb, inp), oracle.stencil_chain(inp)), (seed, h, w)
    inp = u16_frame((40, 50), 3)
    got = run(hb, inp, out_shape=(60, 80), in_mins=(3, -2), out_mins=(-10, -9))
    assert np.array_equal(got, oracle.stencil_chain(inp, out_shape=(60, 80), in_mins=(3, -2), out_mins=(-10, -9)))
    got = run(hb, inp, out_shape=(21, 33), in_mins=(0, 0), out_mins=(7, 5))
    assert np.array_equal(got, oracle.stencil_chain(inp, out_shape=(21, 33), in_mins=(0, 0), out_mins=(7, 5)))
