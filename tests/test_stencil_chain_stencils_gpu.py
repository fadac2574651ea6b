"""halide_b200_stencil_chain_stencils on the GPU: stencil_chain with the generator's stencils (the number of chained 5x5
stages) chosen per call, against oracle/oracle_stencil_chain.cpp run with the same depth.  uint16 ring arithmetic: bit
for bit.  A chain of S stages runs floor(S / 4) launches of 4 stages and, when S mod 4 is not 0, one launch of the rest;
S = 32 must be stencil_chain itself."""
import numpy as np
import pytest

from util import kernels_run, u16_frame

pytestmark = pytest.mark.gpu
EDGE_S = [1, 2, 3, 5, 6, 7, 32, 33, 99, 100]


def run(hb, inp, stencils, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.uint16)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.stencil_chain_stencils(bi, stencils, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out


def test_every_depth_on_a_ragged_frame(hb, oracle):
    """S = 1 .. 100 on a 23 x 37 frame (odd width: odd row strides) placed at odd mins, the output offset from it."""
    inp = u16_frame((37, 23), 2337)
    kw = dict(out_shape=(37, 23), in_mins=(-5, 13), out_mins=(-3, 9))
    for s in range(1, 101):
        assert np.array_equal(run(hb, inp, s, **kw), oracle.stencil_chain(inp, stencils=s, **kw)), s


@pytest.mark.parametrize("s", EDGE_S)
def test_edge_shapes(hb, oracle, s):
    """Ragged sizes (odd widths take the 16-bit load / store paths), an output larger than the input at negative mins and
    a crop with odd offsets."""
    for h, w in ((1, 1), (17, 40), (65, 129), (200, 333)):
        inp = u16_frame((h, w), 10 * s + h + w)
        assert np.array_equal(run(hb, inp, s), oracle.stencil_chain(inp, stencils=s)), (h, w)
    inp = u16_frame((40, 50), s)
    for kw in (dict(out_shape=(60, 80), in_mins=(3, -2), out_mins=(-10, -9)),
               dict(out_shape=(21, 33), in_mins=(0, 0), out_mins=(7, 5))):
        assert np.array_equal(run(hb, inp, s, **kw), oracle.stencil_chain(inp, stencils=s, **kw)), kw


@pytest.mark.parametrize("s", EDGE_S)
def test_odd_strides_and_base_on_the_device(hb, oracle, s):
    """Device-resident torch views with odd row pitches and bases one pixel past a 4-byte boundary: no launch may use
    the 32-bit path on the frame's own buffers."""
    import torch
    h, w = 45, 71
    base = u16_frame((h, w + 6), 90 + s)  # row pitch 77: odd
    tin = torch.from_numpy(base.view(np.int16)).cuda().view(torch.uint16)
    for off in (0, 1):
        ref = oracle.stencil_chain(np.ascontiguousarray(base[:, off:off + w]), stencils=s)
        tout_full = torch.zeros((h, w + 4), dtype=torch.uint16, device="cuda")  # row pitch 75
        view_out = tout_full[:, off:off + w]
        hb.filters.stencil_chain_stencils(hb.HalideBuffer.from_torch(tin[:, off:off + w]), s,
                                          hb.HalideBuffer.from_torch(view_out))
        torch.cuda.synchronize()
        full = tout_full.view(torch.int16).cpu().numpy().view(np.uint16)
        assert np.array_equal(full[:, off:off + w], ref), off
        assert not full[:, :off].any() and not full[:, off + w:].any()


def test_constant_frame(hb):
    """A constant frame c maps to c * 225^S mod 2^16 (the weights of one stage sum to 225), at every depth."""
    inp = np.full((70, 90), 3, np.uint16)
    for s in range(1, 101):
        got = run(hb, inp, s)
        assert (got == (3 * pow(225, s, 1 << 16)) % (1 << 16)).all(), s


def _launches(hb):
    return hb.capi.halide_b200_kernel_launch_count()


def test_32_is_stencil_chain(hb):
    inp = u16_frame((130, 257), 32)
    want = np.zeros_like(inp)
    bi, bo = hb.HalideBuffer.from_numpy(inp), hb.HalideBuffer.from_numpy(want, host_dirty=False)
    hb.filters.stencil_chain(bi, bo)
    bo.copy_to_host()
    n0 = _launches(hb)
    with kernels_run(hb) as ran:
        got = run(hb, inp, 32)
    assert _launches(hb) - n0 == 8
    assert set(ran) == {"stencil_chain_window"} and ran["stencil_chain_window"][0] == 8, ran
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("s", [1, 3, 4, 5, 99, 100])
def test_launches_per_depth(hb, oracle, s):
    inp = u16_frame((61, 107), s)
    n0 = _launches(hb)
    with kernels_run(hb) as ran:
        got = run(hb, inp, s)
    assert _launches(hb) - n0 == -(-s // 4)
    assert set(ran) == {"stencil_chain_window"} and ran["stencil_chain_window"][0] == -(-s // 4), ran
    assert np.array_equal(got, oracle.stencil_chain(inp, stencils=s))


@pytest.mark.parametrize("s", [1, 3, 33, 100])
def test_harness_size_linearity(hb, s):
    """1536 x 2560 (the harness frame): every stage is linear over Z/2^16, so f(a + b) == f(a) + f(b) (mod 2^16)."""
    a = u16_frame((2560, 1536), 1 + s)
    b = u16_frame((2560, 1536), 2 + s)
    fa, fb, fab = run(hb, a, s), run(hb, b, s), run(hb, (a + b).astype(np.uint16), s)
    assert np.array_equal(fab, (fa + fb).astype(np.uint16))


@pytest.mark.parametrize("s,corners", [(33, [(0, 0), (2560 - 96, 1536 - 96), (1200, 700), (2048 - 48, 1024 - 48)]),
                                       (100, [(0, 0), (1201, 703)])])
def test_harness_size_regions_vs_oracle(hb, oracle, s, corners):
    """1536 x 2560 against the oracle by region: S stages of a 5x5 stencil reach 2S px, so the oracle on a crop with a
    2S + 16 px margin (ending exactly at the frame edges it touches) determines the region."""
    h, w = 2560, 1536
    inp = u16_frame((h, w), 40 + s)
    got = run(hb, inp, s)
    n, m = 96, 2 * s + 16
    for (y0, x0) in corners:
        ya, yb, xa, xb = max(0, y0 - m), min(h, y0 + n + m), max(0, x0 - m), min(w, x0 + n + m)
        crop = np.ascontiguousarray(inp[ya:yb, xa:xb])
        want = oracle.stencil_chain(crop, in_mins=(xa, ya), out_mins=(xa, ya), stencils=s)
        assert np.array_equal(got[y0:y0 + n, x0:x0 + n], want[y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n]), (y0, x0)


def test_alternating_depths_on_the_same_buffers(hb, oracle):
    """Scratch is sized per call: a deep chain after a shallow one on the same buffers is still right."""
    import torch
    inp = u16_frame((150, 263), 7)
    tin = torch.from_numpy(inp.view(np.int16)).cuda().view(torch.uint16)
    tout = torch.empty_like(tin)
    bi, bo = hb.HalideBuffer.from_torch(tin), hb.HalideBuffer.from_torch(tout)
    for s in (100, 1, 37, 100):
        tout.fill_(0)
        hb.filters.stencil_chain_stencils(bi, s, bo)
        torch.cuda.synchronize()
        got = tout.view(torch.int16).cpu().numpy().view(np.uint16)
        assert np.array_equal(got, oracle.stencil_chain(inp, stencils=s)), s
