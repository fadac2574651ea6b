"""GPU parity tests for local_laplacian through the C ABI: bit-exact uint16 against the oracle
(oracle/oracle_local_laplacian.cpp, a restatement of apps/local_laplacian/local_laplacian_generator.cpp)."""
import os

import numpy as np
import pytest

from util import run_local_laplacian, smooth_u16_frame, u16_frame

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _check(hb, oracle, img, levels, alpha, beta, **kw):
    got = run_local_laplacian(hb, img, levels, alpha, beta, **kw)
    want = oracle.local_laplacian(img, levels, alpha, beta, **kw)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{len(bad)} mismatching samples, first at (c,y,x)={bad[0]}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


@pytest.mark.parametrize("h,w", [(1, 1), (2, 3), (7, 5), (16, 16), (33, 47), (64, 96), (100, 130), (255, 257)])
def test_small_and_ragged_frames(hb, oracle, h, w):
    _check(hb, oracle, u16_frame((3, h, w), h * 1000 + w), 8, 1.0 / 7.0, 1.0)


@pytest.mark.parametrize("seed", [0, 42, 1, 2])
def test_random_full_range(hb, oracle, seed):
    _check(hb, oracle, u16_frame((3, 192, 320), seed), 8, 1.0 / 7.0, 1.0)


@pytest.mark.parametrize("seed", [0, 1])
def test_smooth_content(hb, oracle, seed):
    _check(hb, oracle, smooth_u16_frame((3, 200, 264), seed), 8, 1.0 / 7.0, 1.0)


@pytest.mark.parametrize("levels,alpha,beta", [(2, 1.0, 1.0), (4, 0.5, 0.7), (8, 2.0 / 7.0, 1.5), (8, 0.0, 1.0),
                                               (16, 1.0 / 15.0, 0.3)])
def test_parameter_sweep(hb, oracle, levels, alpha, beta):
    _check(hb, oracle, u16_frame((3, 72, 104), levels), levels, alpha, beta)


def test_extreme_pixels(hb, oracle):
    img = u16_frame((3, 64, 80), 9)
    img[:, :8] = 0
    img[:, 8:16] = 65535
    img[0, 16:24] = 0
    img[1, 16:24] = 65535
    _check(hb, oracle, img, 8, 1.0 / 7.0, 1.0)


def test_output_crop_with_offsets(hb, oracle):
    """Output region strictly inside a larger input with non-zero mins: the pyramid is clamped at the
    INPUT's edges (repeat_edge uses the buffer's own bounds, src/BoundaryConditions.cpp:15-35)."""
    img = u16_frame((3, 90, 120), 4)
    _check(hb, oracle, img, 8, 1.0 / 7.0, 1.0, out_shape=(3, 50, 61), in_mins=(-7, 3, 0), out_mins=(10, 21, 0))
    _check(hb, oracle, img, 8, 1.0 / 7.0, 1.0, out_shape=(3, 90, 120), in_mins=(5, -4, 0), out_mins=(5, -4, 0))


def test_golden_fixture(hb):
    """Committed vectors (tests/golden/make_golden.py ran the oracle once): guards both the oracle and
    the kernels against drifting together."""
    z = np.load(os.path.join(GOLDEN, "local_laplacian_small.npz"))
    got = run_local_laplacian(hb, z["input"], int(z["levels"]), float(z["alpha"]), float(z["beta"]))
    assert np.array_equal(got, z["output"])


def test_idempotent_and_deterministic(hb):
    img = u16_frame((3, 300, 420), 77)
    a = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    b = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    assert np.array_equal(a, b)


def test_4k_tile_consistency(hb, oracle):
    """Config 2 size (3840x2160x3).  The oracle needs ~1 min for a full 4K frame, so the full-size
    check is by region: the top-left and bottom-right 256x256 corners of the 4K result must equal
    the oracle run on the enlarged crop that determines them (footprint of 8 levels < 2*256+64 px)."""
    h, w = 2160, 3840
    img = u16_frame((3, h, w), 0)
    got = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    m = 1024  # margin: level-7 taps reach < 2^8 * 3 px; the crop keeps the true frame edge on two sides
    tl = oracle.local_laplacian(np.ascontiguousarray(img[:, :m, :m]), 8, 1.0 / 7.0, 1.0)
    assert np.array_equal(got[:, :160, :160], tl[:, :160, :160])
    # pyramid coordinates are absolute (parity of x,y matters in down/upsample): keep the crop's mins
    br = oracle.local_laplacian(np.ascontiguousarray(img[:, h - m:, w - m:]), 8, 1.0 / 7.0, 1.0,
                                in_mins=(w - m, h - m, 0), out_mins=(w - m, h - m, 0))
    assert np.array_equal(got[:, h - 160:, w - 160:], br[:, m - 160:, m - 160:])


def _region_vs_oracle(oracle, img, got, y0, x0, n=128, margin=896):
    """`got` = the filter's result on the whole frame `img`; compare its n x n region at (y0, x0) with the oracle run on
    the crop that determines it (the footprint of 8 pyramid levels stays well inside `margin` px; pyramid coordinates
    are absolute — the parity of x, y matters in down/upsample — so the crop keeps its frame coordinates as mins; where
    the crop touches a frame edge it ends exactly there, so repeat_edge acts where it would on the whole frame)."""
    _, h, w = img.shape
    ya, yb = max(0, y0 - margin), min(h, y0 + n + margin)
    xa, xb = max(0, x0 - margin), min(w, x0 + n + margin)
    crop = np.ascontiguousarray(img[:, ya:yb, xa:xb])
    want = oracle.local_laplacian(crop, 8, 1.0 / 7.0, 1.0, in_mins=(xa, ya, 0), out_mins=(xa, ya, 0))
    w_reg = want[:, y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n]
    g_reg = got[:, y0:y0 + n, x0:x0 + n]
    bad = np.argwhere(g_reg != w_reg)
    assert bad.size == 0, f"region ({y0},{x0}): {len(bad)} mismatching samples, first at {bad[0]}"


def test_4k_interior_regions(hb, oracle):
    """Config 2 size, away from the frame edges: where the strip / chunk / tile seams of the kernels and the balanced
    work partition live (the corners alone never see them)."""
    h, w = 2160, 3840
    img = u16_frame((3, h, w), 5)
    got = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    for (y0, x0) in [(1000, 1850), (1016, 3600), (37, 2001), (2032, 64)]:
        _region_vs_oracle(oracle, img, got, y0, x0)


def test_16k_regions(hb, oracle):
    """North-star size (16384 x 16384 x 3): corners, an interior region, and regions straddling rows 2048*k and the
    2^31-byte marks of the level buffers (the kernels use 32-bit element / 64-bit byte addressing at this size)."""
    n = 16384
    rng = np.random.default_rng(16)
    img = rng.integers(0, 1 << 16, (3, n, n), dtype=np.uint16)
    got = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    for (y0, x0) in [(0, 0), (n - 128, n - 128), (8131, 9000), (3 * 2048 - 64, 5000), (6 * 2048 - 64, 16384 - 200),
                     (10923, 123), (16384 - 128, 7777)]:
        _region_vs_oracle(oracle, img, got, y0, x0)


def test_generic_kernels_agree_with_fast_path(hb, oracle):
    """levels == 8 takes the fast kernels; any other `levels` (and this hook) takes the generic per-pixel kernels.
    Both must equal the oracle; so must every mix of them (the up-sweep then picks its planes out of the level instead
    of the pair plane the fast down-sweep emits)."""
    img = u16_frame((3, 131, 203), 31)
    want = oracle.local_laplacian(img, 8, 1.0 / 7.0, 1.0)
    l = hb.load_library()
    try:
        l.halide_b200_ll_force_generic(7)
        got_generic = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    finally:
        l.halide_b200_ll_force_generic(0)
    got_fast = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    assert np.array_equal(got_generic, want) and np.array_equal(got_fast, want)
    # 64: no TMA frame tile in the final kernel
    for mask in (1, 2, 4, 8, 1 | 8, 2 | 4, 64, 16 | 64):
        try:
            l.halide_b200_ll_force_generic(mask)
            got = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
        finally:
            l.halide_b200_ll_force_generic(0)
        assert np.array_equal(got, want), f"force_generic mask {mask}"


def test_beta_not_one_takes_the_general_kernels(hb, oracle):
    """beta == 1 (the harness default) selects kernel variants without the beta multiply (1 * x is exact); any other
    beta takes the general variants."""
    img = u16_frame((3, 150, 260), 12)
    for beta in (0.5, 1.0, 2.0):
        _check(hb, oracle, img, 8, 1.0 / 7.0, beta)


def test_wide_frame_many_strips(hb, oracle):
    """A frame wide enough for several 30-column strips and 64-column tiles per row, odd sizes."""
    _check(hb, oracle, u16_frame((3, 77, 1031), 8), 8, 1.0 / 7.0, 1.0)


@pytest.mark.parametrize("shape", [(3, 130, 256), (3, 97, 198), (3, 64, 66)])
def test_final_kernel_simple_and_general_layout_paths(hb, oracle, shape):
    """Even-width 3-channel frames with 4-byte aligned rows take the final kernel's aligned path (32-bit addressing,
    one aligned word per thread and channel); hook bit 16 forces the general-layout path on the same frame.
    Both must equal the oracle; a crop with odd column offsets must fall back to the general path by itself."""
    img = u16_frame(shape, 77)
    want = oracle.local_laplacian(img, 8, 1.0 / 7.0, 1.0)
    l = hb.load_library()
    got_simple = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    try:
        l.halide_b200_ll_force_generic(16)
        got_general = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0)
    finally:
        l.halide_b200_ll_force_generic(0)
    assert np.array_equal(got_simple, want) and np.array_equal(got_general, want)
    c, h, w = shape
    out_shape = (3, h - 9, w - 12)  # even width, output columns start at an odd input column
    want_crop = oracle.local_laplacian(img, 8, 1.0 / 7.0, 1.0, out_shape=out_shape, in_mins=(0, 0, 0), out_mins=(5, 4, 0))
    got_crop = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0, out_shape=out_shape, in_mins=(0, 0, 0), out_mins=(5, 4, 0))
    assert np.array_equal(got_crop, want_crop)
    out_shape = (3, h - 8, w - 12)  # even offsets: SIMPLE path on a crop (row pointer no longer at the buffer start)
    want_crop = oracle.local_laplacian(img, 8, 1.0 / 7.0, 1.0, out_shape=out_shape, in_mins=(0, 0, 0), out_mins=(6, 4, 0))
    got_crop = run_local_laplacian(hb, img, 8, 1.0 / 7.0, 1.0, out_shape=out_shape, in_mins=(0, 0, 0), out_mins=(6, 4, 0))
    assert np.array_equal(got_crop, want_crop)


@pytest.mark.parametrize("h,w,beta,crop", [(150, 256, 1.0, False), (101, 136, 0.7, False), (49, 64, 1.0, False),
                                          (140, 264, 1.0, True)])
def test_tma_final_kernel(hb, oracle, h, w, beta, crop):
    """Frames whose rows are 16-byte multiples take the final kernel's TMA frame tile: heights that are no multiple of
    its 32-row tiles, beta == 1 and beta != 1, and a crop starting 8 columns / 5 rows inside the input."""
    img = u16_frame((3, h, w), h)
    if crop:
        _check(hb, oracle, img, 8, 1.0 / 7.0, beta, out_shape=(3, h - 20, w - 24), in_mins=(0, 0, 0), out_mins=(8, 5, 0))
    else:
        _check(hb, oracle, img, 8, 1.0 / 7.0, beta)
