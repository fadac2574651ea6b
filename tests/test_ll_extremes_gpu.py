"""local_laplacian at extreme and non-finite alpha and beta (ll_extremes.CASES) against the oracle, byte for byte, through
every kernel path and entry point, asserting which kernels ran.

Two things go wrong there when a kernel departs from Halide's arithmetic.  A NaN colour must clamp to 65535 (Halide's
min / max select on a comparison), not 0 as a float-to-integer conversion gives it.  And the pyramid's sums must round
and overflow as the generator's do: the fast down kernels (ll_level1, ll_down_rows) defer the downsample's first * 1/8
to one * 1/64 after the second pass, which overflows at an eighth of the generator's range, so the library sends alpha
or beta of magnitude 2^100 and up (and non-finite ones) to the generic down kernels, which scale as the generator does.

Frames sit in rows padded to 80 samples (160 bytes) where a path needs 16-byte rows: the final kernel's TMA frame tile,
the vector tone kernel, the interleaved TMA path."""
import functools
from contextlib import contextmanager

import numpy as np
import pytest

import ll_bordered
import ll_extremes as E
from halide_b200.image_io import convert
from util import kernels_run

pytestmark = pytest.mark.gpu
PITCH = 80  # padded row length (elements, or pixels for interleaved frames)
FAST = [c for c in E.CASES if c.levels == 8]  # levels 8: the fast kernels


def fast_sums(c):
    """The fast down kernels run (levels 8, J >= 3) only for these scalars (local_laplacian.cu: fast_down)."""
    return abs(c.alpha) < 2.0 ** 100 and abs(c.beta) < 2.0 ** 100


def expected_kernels(c, mask=0, J=8):
    """The level-1 and final kernels a call on case c runs under force-generic mask `mask` at pyramid depth J >= 2."""
    fast = c.levels == 8 and J >= 3
    down = "ll_level1" if fast and fast_sums(c) and not mask & 1 else "ll_level1_generic"
    final = "ll_final2" if fast and not mask & 4 else "ll_final"
    return {down, final}


@contextmanager
def force_generic(hb, mask):
    l = hb.load_library()
    l.halide_b200_ll_force_generic(mask)
    try:
        yield
    finally:
        l.halide_b200_ll_force_generic(0)


def padded(a, pitch=PITCH):
    """A view of the planar frame(s) `a` ([..., h, w]) whose rows are `pitch` samples long."""
    v = np.zeros(a.shape[:-1] + (pitch,), a.dtype)[..., :a.shape[-1]]
    v[...] = a
    return v


def padded_pixels(a, pitch=PITCH):
    """A view of the interleaved frame `a` ([h, w, c]) whose rows are `pitch` pixels long."""
    v = np.zeros((a.shape[0], pitch, a.shape[2]), a.dtype)[:, :a.shape[1]]
    v[...] = a
    return v


@functools.lru_cache(maxsize=None)
def want(oracle, case_id, J=8):
    """The oracle's output on the case frame (the bordered evaluation past J = 11, as in test_ll_pyramid_levels_gpu)."""
    c = CASES[case_id]
    evaluate = ll_bordered.local_laplacian if J > 11 else oracle.local_laplacian
    return evaluate(E.frame(), c.levels, c.alpha, c.beta, pyramid_levels=J)


CASES = {c.id: c for c in E.CASES}


def same(got, ref, what):
    bad = got != ref
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} samples differ, first at {i}: {got[i]} vs {ref[i]}")


def call(hb, fn, inp, out, *args):
    bi = hb.HalideBuffer.from_numpy(inp)
    bo = hb.HalideBuffer.from_numpy(out, host_dirty=False)
    with kernels_run(hb) as ran:
        fn(bi, *args, bo)
    bo.copy_to_host()
    return set(ran)


# ---- local_laplacian under each force-generic mask ---------------------------------------------------------------------
# 0: TMA frame tile in the final kernel; 64: aligned loads instead; 16 | 64: the general-layout final kernel; 4: the
# generic final kernel; 1: the generic down kernels; 8: every level its own launches (no fused tail), so ll_up2 runs the
# up-sweep; 2 | 8: the generic up-sweep kernel instead (on this frame every level past the first fits the fused tail,
# so bit 2 alone changes nothing).
MASKS = [0, 64, 16 | 64, 4, 1, 8, 2 | 8]


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("c", FAST, ids=lambda c: c.id)
def test_masks(hb, oracle, c, mask):
    out = padded(np.zeros(E.SHAPE, np.uint16))
    with force_generic(hb, mask):
        ran = call(hb, hb.filters.local_laplacian, padded(E.frame()), out, c.levels, c.alpha, c.beta)
    same(out, want(oracle, c.id), f"mask {mask}")
    assert expected_kernels(c, mask) <= ran, sorted(ran)
    assert ("ll_coarse_fused" in ran) == (not mask & 8), sorted(ran)
    if mask & 8:
        assert ("ll_up2" in ran) != bool(mask & 2), sorted(ran)


@pytest.mark.parametrize("c", [c for c in E.CASES if c.levels != 8], ids=lambda c: c.id)
def test_other_levels(hb, oracle, c):
    """levels 2 and 32: the generic kernels, and remap tables of 513 and 15873 entries."""
    out = np.zeros(E.SHAPE, np.uint16)
    ran = call(hb, hb.filters.local_laplacian, E.frame(), out, c.levels, c.alpha, c.beta)
    same(out, want(oracle, c.id), f"levels {c.levels}")
    assert expected_kernels(c) <= ran, sorted(ran)


# ---- pyramid depths ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("J,mask", [(1, 0), (1, 16), (2, 0), (3, 0), (20, 0)], ids=["J1vec", "J1px", "J2", "J3", "J20"])
@pytest.mark.parametrize("c", FAST, ids=lambda c: c.id)
def test_pyramid_levels(hb, oracle, c, J, mask):
    """J = 1: the tone kernel, its 16-byte vector form on the padded rows and its per-pixel form (mask 16); J = 2: the
    generic kernels; J = 3 and 20: the fast kernels at the shallowest and the deepest pyramid."""
    out = padded(np.zeros(E.SHAPE, np.uint16))
    with force_generic(hb, mask):
        ran = call(hb, hb.filters.local_laplacian_pyramid_levels, padded(E.frame()), out, J, c.levels, c.alpha, c.beta)
    same(out, want(oracle, c.id, J), f"J {J}")
    if J == 1:
        assert "ll_tone" in ran and ran <= {"ll_lut", "ll_tone"}, sorted(ran)
    else:
        assert expected_kernels(c, 0, J) <= ran, sorted(ran)


# ---- 8-bit and interleaved entry points -------------------------------------------------------------------------------

def want_u8(oracle, c, frame8):
    return convert(oracle.local_laplacian(convert(frame8, np.uint16), c.levels, c.alpha, c.beta), np.uint8)


@pytest.mark.parametrize("c", FAST, ids=lambda c: c.id)
def test_u8(hb, oracle, c):
    """to_u8(oracle(to_u16(x))): a NaN colour is 65535, so 255."""
    x = convert(E.frame(), np.uint8)
    out = padded(np.zeros(E.SHAPE, np.uint8))
    ran = call(hb, hb.filters.local_laplacian_u8, padded(x), out, c.levels, c.alpha, c.beta)
    same(out, want_u8(oracle, c, x), "u8")
    assert expected_kernels(c) <= ran, sorted(ran)


@pytest.mark.parametrize("dtype", [np.uint16, np.uint8])
@pytest.mark.parametrize("c", FAST, ids=lambda c: c.id)
def test_interleaved(hb, oracle, c, dtype):
    """RGB frames, pixel-interleaved, in rows of 80 pixels: the final kernel's interleaved TMA path."""
    x = E.frame() if dtype == np.uint16 else convert(E.frame(), np.uint8)
    out = padded_pixels(np.zeros(E.SHAPE[1:] + (3,), dtype))
    fn = hb.filters.local_laplacian_interleaved if dtype == np.uint16 else hb.filters.local_laplacian_u8_interleaved
    bi = hb.HalideBuffer.from_numpy(padded_pixels(x.transpose(1, 2, 0)).transpose(2, 0, 1))
    bo = hb.HalideBuffer.from_numpy(out.transpose(2, 0, 1), host_dirty=False)
    with kernels_run(hb) as ran:
        fn(bi, c.levels, c.alpha, c.beta, bo)
    bo.copy_to_host()
    ref = want(oracle, c.id) if dtype == np.uint16 else want_u8(oracle, c, x)
    same(np.ascontiguousarray(out.transpose(2, 0, 1)), ref, f"interleaved {np.dtype(dtype).name}")
    assert expected_kernels(c) <= set(ran), sorted(ran)


# ---- batches -----------------------------------------------------------------------------------------------------------

def batch_frames():
    """Three frames of different content: the case frame, another seed, and the case frame turned by 180 degrees."""
    a = E.frame()
    return np.stack([a, E.frame(seed=E.SEED + 1), np.ascontiguousarray(a[:, ::-1, ::-1])])


@pytest.mark.parametrize("dtype", [np.uint16, np.uint8])
@pytest.mark.parametrize("c", FAST, ids=lambda c: c.id)
def test_batch(hb, oracle, c, dtype):
    x = batch_frames() if dtype == np.uint16 else convert(batch_frames(), np.uint8)
    out = padded(np.zeros(x.shape, dtype))
    fn = hb.filters.local_laplacian_batch if dtype == np.uint16 else hb.filters.local_laplacian_u8_batch
    ran = call(hb, fn, padded(x), out, c.levels, c.alpha, c.beta)
    for k in range(x.shape[0]):
        if dtype == np.uint16:
            ref = oracle.local_laplacian(x[k], c.levels, c.alpha, c.beta)
        else:
            ref = want_u8(oracle, c, x[k])
        same(out[k], ref, f"batch {np.dtype(dtype).name} frame {k}")
    assert expected_kernels(c) <= ran, sorted(ran)


# ---- a video frame ---------------------------------------------------------------------------------------------------

def test_1080p_at_the_mixed_alpha(hb, oracle):
    """One 1920 x 1080 frame at levels 8's NaN-mixed alpha, compared whole: level 2 is too large for the fused tail here,
    so its own down- and up-sweep launches run as well.  Its colours are +-inf, and NaN on about 2900 samples."""
    alpha = E.f32(E.MIXED[8][0])
    img = E.frame((3, 1080, 1920))
    out = np.zeros_like(img)
    ran = call(hb, hb.filters.local_laplacian, img, out, 8, alpha, 1.0)
    ref = oracle.local_laplacian(img, 8, alpha, 1.0)
    same(out, ref, "1080p")
    assert (ref == 65535).mean() > 0.05 and (ref == 0).mean() > 0.05, "the frame lost its mix"
    assert {"ll_level1_generic", "ll_down", "ll_up2", "ll_final2"} <= ran, sorted(ran)
