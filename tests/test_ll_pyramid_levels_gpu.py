"""GPU tests of halide_b200_local_laplacian_pyramid_levels: every pyramid depth J in [1, 20] bit for bit against the oracle
(the literal evaluation up to J = 11, the bordered one of tests/ll_bordered.py above, which tests/test_ll_pyramid_levels.py
checks against the literal one), crops and layouts, a frame wide enough that levels past the eighth get launches of their own, J = 8 against
local_laplacian itself, which kernels each depth runs, and back-to-back calls at changing depths."""
import numpy as np
import pytest

import ll_bordered
from util import kernels_run, smooth_u16_frame, u16_frame

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (2, 3), (17, 33), (255, 129), (480, 270)]  # (W, H)
PARAMS = [(levels, alpha, beta) for levels in (8, 3, 5) for alpha in (1.0 / (levels - 1), 0.5) for beta in (1.0, 0.5)]


def run(hb, img, J, levels, alpha, beta, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(img.shape if out_shape is None else out_shape, np.uint16)
    bi = hb.HalideBuffer.from_numpy(img, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.local_laplacian_pyramid_levels(bi, J, levels, alpha, beta, bo)
    bo.copy_to_host()
    return out


def want(oracle, img, J, levels, alpha, beta, **kw):
    evaluate = ll_bordered.local_laplacian if J > 11 else oracle.local_laplacian
    return evaluate(img, levels, alpha, beta, pyramid_levels=J, **kw)


def check(hb, oracle, img, J, levels, alpha, beta, **kw):
    got = run(hb, img, J, levels, alpha, beta, **kw)
    ref = want(oracle, img, J, levels, alpha, beta, **kw)
    assert np.array_equal(got, ref), (J, levels, alpha, beta, kw, int(np.count_nonzero(got != ref)))


@pytest.mark.parametrize("J", range(1, 21))
@pytest.mark.parametrize("W,H", SIZES)
def test_every_depth(hb, oracle, J, W, H):
    img = smooth_u16_frame((3, H, W), J) if (W * H) % 2 else u16_frame((3, H, W), J + W)
    for levels, alpha, beta in PARAMS:
        check(hb, oracle, img, J, levels, alpha, beta)


@pytest.mark.parametrize("J", [1, 3, 10, 14])
def test_4k(hb, oracle, J):
    img = smooth_u16_frame((3, 2160, 3840), J)
    check(hb, oracle, img, J, 8, 1.0 / 7.0, 1.0)


@pytest.mark.parametrize("J", [1, 2, 3, 9, 14])
def test_crops_channels_and_strides(hb, oracle, J):
    img = u16_frame((3, 61, 83), 7 * J)
    # an input larger than the output, at negative and at nonzero positive mins
    check(hb, oracle, img, J, 8, 1.0 / 7.0, 1.0, out_shape=(3, 40, 57), in_mins=(-20, -11, 0), out_mins=(-13, -3, 0))
    check(hb, oracle, img, J, 5, 0.5, 0.5, out_shape=(3, 29, 33), in_mins=(1000, 37, 0), out_mins=(1031, 50, 0))
    # output channel ranges
    for c0, c1 in [(0, 1), (1, 3), (0, 3)]:
        check(hb, oracle, img, J, 8, 1.0 / 7.0, 1.0, out_shape=(c1 - c0, 61, 83), out_mins=(0, 0, c0))
    # an input row stride that is not dense (and not a 16-byte multiple)
    wide = u16_frame((3, 45, 77), 3 * J)
    check(hb, oracle, wide[:, :, :70], J, 8, 1.0 / 7.0, 1.0)
    check(hb, oracle, wide[:, :, 3:67], J, 3, 0.5, 1.0)


@pytest.mark.parametrize("J", [1, 3, 14])
def test_general_layout_paths(hb, oracle, J):
    """The general-layout final and tone kernels (the force-generic hook's 16) on a frame the aligned ones would take."""
    img = smooth_u16_frame((3, 64, 96), J)
    ref = want(oracle, img, J, 8, 1.0 / 7.0, 1.0)
    l = hb.load_library()
    l.halide_b200_ll_force_generic(16)
    try:
        got = run(hb, img, J, 8, 1.0 / 7.0, 1.0)
    finally:
        l.halide_b200_ll_force_generic(0)
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("levels", [8, 3])
def test_levels_past_the_eighth_with_launches_of_their_own(hb, oracle, levels):
    """A 2^22 x 1 frame: at J = 14 levels 8 and up are still too big for the fused tail (tests/test_ll_pyramid_levels.py
    checks the host's choice), so they run ll_down_rows / ll_up2 (levels 8) or the generic kernels (levels 3) on a level
    index past the 8 slots of the per-level stride arrays."""
    l = hb.load_library()
    assert l.halide_b200_ll_last_own_level(1 << 22, 1, 14) >= 8
    img = smooth_u16_frame((3, 1, 1 << 22), levels)
    with kernels_run(hb) as ran:
        got = run(hb, img, 14, levels, 1.0 / (levels - 1), 1.0)
    ref = want(oracle, img, 14, levels, 1.0 / (levels - 1), 1.0)
    assert np.array_equal(got, ref), int(np.count_nonzero(got != ref))
    assert ("ll_down_rows" if levels == 8 else "ll_down") in ran, ran


@pytest.mark.parametrize("W,H,levels", [(480, 270, 8), (3840, 2160, 8), (255, 129, 3)])
def test_depth_8_is_local_laplacian(hb, W, H, levels):
    img = smooth_u16_frame((3, H, W), W)
    alpha = 1.0 / (levels - 1)
    out = np.zeros_like(img)
    bi, bo = hb.HalideBuffer.from_numpy(img), hb.HalideBuffer.from_numpy(out, host_dirty=False)
    hb.filters.local_laplacian(bi, levels, alpha, 1.0, bo)  # (the remap table exists for both calls below)
    with kernels_run(hb) as plain:
        hb.filters.local_laplacian(bi, levels, alpha, 1.0, bo)
    bo.copy_to_host()
    a = out.copy()
    with kernels_run(hb) as deep:
        hb.filters.local_laplacian_pyramid_levels(bi, 8, levels, alpha, 1.0, bo)
    bo.copy_to_host()
    assert np.array_equal(a, out)
    assert {k: v[0] for k, v in plain.items()} == {k: v[0] for k, v in deep.items()}


def _names(hb, J, levels, alpha):
    img = smooth_u16_frame((3, 270, 480), 5)
    with kernels_run(hb) as ran:
        run(hb, img, J, levels, alpha, 1.0)
    return {k: v[0] for k, v in ran.items()}


@pytest.mark.parametrize("J", [3, 4, 8, 12, 20])
def test_fast_kernels_from_depth_3(hb, J):
    ran = _names(hb, J, 8, 1.0 / 7.0)
    assert ran.get("ll_level1") and ran.get("ll_final2"), ran
    assert not {"ll_level1_generic", "ll_final", "ll_tone"} & set(ran), ran


def test_depth_2_runs_the_generic_kernels(hb):
    ran = _names(hb, 2, 8, 1.0 / 7.0)
    assert ran.get("ll_level1_generic") == 1 and ran.get("ll_up") == 1 and ran.get("ll_final") == 1, ran
    assert not {"ll_level1", "ll_final2", "ll_up2", "ll_coarse_fused", "ll_tone"} & set(ran), ran


def test_depth_1_runs_only_the_tone_kernel(hb):
    alpha = 0.3125  # a table no other test builds: the first call builds it
    assert _names(hb, 1, 8, alpha) == {"ll_lut": 1, "ll_tone": 1}
    assert _names(hb, 1, 8, alpha) == {"ll_tone": 1}


def test_depth_1_tables_above_48k_in_turn(hb, oracle):
    """ll_tone stages the remap table, (2 * 256 * (levels - 1) + 1) floats, in shared memory: more than 48 KB at levels 30
    and 26 alike.  The 26-level call must not leave the kernel's limit below what the following 30-level call needs.  (No
    other test runs ll_tone at these level counts.)"""
    img = u16_frame((3, 61, 83), 30)
    for levels in (30, 26, 30):
        alpha = 1.0 / (levels - 1)
        with kernels_run(hb) as ran:
            got = run(hb, img, 1, levels, alpha, 1.0)
        assert "ll_tone" in ran, (levels, ran)
        assert np.array_equal(got, want(oracle, img, 1, levels, alpha, 1.0)), levels


def test_alternating_depths_leak_nothing(hb):
    img = u16_frame((3, 133, 201), 99)
    seq = [(1, 8), (14, 3), (2, 8), (8, 5), (20, 8), (3, 3), (1, 5), (11, 8), (2, 3)]
    fresh = {}
    for J, levels in reversed(seq):
        fresh[J, levels] = run(hb, img, J, levels, 1.0 / (levels - 1), 0.5)
    for _ in range(2):
        for J, levels in seq:
            assert np.array_equal(run(hb, img, J, levels, 1.0 / (levels - 1), 0.5), fresh[J, levels]), (J, levels)
