"""The largest parameters the filters accept, and the kernel branches only they reach, against the oracle.

bilateral_grid's shared-memory opt-ins (histogram beyond 48 bins, slice staging beyond 126) and its 200-bin limit;
nl_means' generic kernel batching a search row's dx offsets over several passes, the largest patch / search pair, and
inputs whose channels are not [0, 3); local_laplacian at 3..32 levels, negative alpha, and a sweep of alphas long
enough to make the remap-table cache evict.  Where a host-side formula picks the branch, the test restates it and
asserts which side the case falls on, so a retuned budget fails here instead of silently losing the coverage."""
from contextlib import contextmanager

import numpy as np
import pytest

from nl_means_exact import sensitive_frame
from util import f32_frame, kernels_run, run_local_laplacian, smooth_u16_frame, u16_frame

pytestmark = pytest.mark.gpu
RTOL = 1e-4  # the float pipelines' tolerance, as in test_bilateral_grid_gpu.py / test_nl_means_gpu.py
PARAM_TOO_SMALL = -9  # halide_error_code_t


def close(got, want, floor):
    assert np.isfinite(got).all()
    err = np.abs(got - want) / np.maximum(np.abs(want), floor)
    assert err.max() <= RTOL, f"max rel err {err.max()} at {np.unravel_index(err.argmax(), err.shape)}"


# ---- bilateral_grid -------------------------------------------------------------------------------------------------

def bg_zmax(r_sigma):
    """bilateral_grid.cu: inv_r = 1 / r_sigma, zmax = int(1 * inv_r + 0.5), all in float32."""
    inv_r = np.float32(1.0) / np.float32(r_sigma)
    return int(np.float32(np.float32(1.0) * inv_r) + np.float32(0.5))


def bg_hist_bytes(zmax):  # (zmax + 1) bins x 2 channels x 128 threads of float
    return (zmax + 1) * 2 * 128 * 4


def bg_slice_bytes(zmax):  # nz = zmax + 2 planes x 2 cell rows x 24 cells of float2
    return (zmax + 2) * 2 * 24 * 8


def r_sigma_for(zmax):
    r = float(np.float32(1.0) / np.float32(zmax))
    assert bg_zmax(r) == zmax
    return r


def bg_frame(kind, h, w):
    if kind == "noise":
        return f32_frame((h, w), h * w)
    if kind == "ramp":  # every bin from 0 to zmax, 0 and 1 exactly included
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        return ((xx / (w - 1)) * 0.75 + (yy / (h - 1)) * 0.25).astype(np.float32)
    return (f32_frame((h, w), h + w) * 3.0 - 1.0).astype(np.float32)  # values in [-1, 2]: clamped into [0, 1]


def run_bg(hb, inp, r_sigma, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.float32)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.bilateral_grid(bi, r_sigma, bo)
    bo.copy_to_host()
    return out


# zmax 47 / 48: the last histogram without and the first with the > 48 KB opt-in; 126 / 127: the same for the slice's
# staging; 199: the largest grid accepted (200 bins, 200 KB of histogram)
@pytest.mark.parametrize("kind", ["noise", "ramp", "outside"])
@pytest.mark.parametrize("zmax", [47, 48, 126, 127, 199])
def test_bilateral_grid_bin_count_thresholds(hb, oracle, zmax, kind):
    """r_sigma on both sides of each shared-memory threshold of the histogram and slice kernels, and at the largest
    accepted grid."""
    r = r_sigma_for(zmax)
    assert (bg_hist_bytes(zmax) > 48 * 1024) == (zmax >= 48)
    assert (bg_slice_bytes(zmax) > 48 * 1024) == (zmax >= 127)
    assert bg_hist_bytes(zmax) <= 200 * 1024
    inp = bg_frame(kind, 61, 107)
    close(run_bg(hb, inp, r), oracle.bilateral_grid(inp, r), 1e-6)


def test_bilateral_grid_rejects_201_bins(hb):
    """One bin past the largest grid: param_too_small, nothing launched."""
    from halide_b200 import HalideError
    r = r_sigma_for(200)
    assert bg_hist_bytes(200) > 200 * 1024
    inp = f32_frame((16, 16), 0)
    with kernels_run(hb) as ran, pytest.raises(HalideError) as e:
        run_bg(hb, inp, r)
    assert e.value.code == PARAM_TOO_SMALL
    assert not any(k.startswith("bg_") for k in ran), sorted(ran)


@pytest.mark.parametrize("r_sigma", [0.1, r_sigma_for(127), r_sigma_for(199)])
def test_bilateral_grid_negative_output_mins(hb, oracle, r_sigma):
    """Output mins below zero and no multiple of 8: the grid's first cell is a floor division, and the slice tiles start
    at (min & ~7), which must round towards minus infinity too."""
    inp = f32_frame((90, 130), 12)
    kw = dict(out_shape=(70, 101), in_mins=(-29, -21), out_mins=(-19, -11))
    close(run_bg(hb, inp, r_sigma, **kw), oracle.bilateral_grid(inp, r_sigma, **kw), 1e-6)


# ---- nl_means ------------------------------------------------------------------------------------------------------

def nl_nd(patch, search):
    """nl_means.cu: the generic kernel's dx offsets per pass and its shared memory (32 x 16 output tiles; the input tile
    and every dx's D and V tiles within a 100 KB budget, at least one dx)."""
    tx, ty = 32, 16
    iw, ih = tx + patch + search - 2, ty + patch + search - 2
    dw, dh = tx + patch - 1, ty + patch - 1
    fixed, per_dx = 3 * iw * ih * 4, (dh + ty) * dw * 4
    nd = search
    while nd > 1 and fixed + nd * per_dx > 100 * 1024:
        nd -= 1
    return nd, fixed + nd * per_dx


@contextmanager
def nl_variant(hb, v):
    l = hb.load_library()
    l.halide_b200_nl_means_variant(v)
    try:
        yield
    finally:
        l.halide_b200_nl_means_variant(0)


def run_nl(hb, inp, patch, search, sigma, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros((3,) + inp.shape[1:] if out_shape is None else out_shape, np.float32)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.nl_means(bi, patch, search, sigma, bo)
    bo.copy_to_host()
    return out


def nl_check(hb, oracle, inp, patch, search, sigma, kernel, variant=0, **kw):
    kw.setdefault("out_shape", (3,) + inp.shape[1:])
    with nl_variant(hb, variant), kernels_run(hb) as ran:
        got = run_nl(hb, inp, patch, search, sigma, **kw)
    assert list(ran) == [kernel], sorted(ran)
    want = oracle.nl_means(inp, patch, search, sigma, **kw)
    close(got, want, 1e-3)
    return got


def smooth_f32(c, h, w, seed):
    """Smooth content plus noise: patch distances spread over a range where many weights matter."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([0.5 + 0.4 * np.sin(xx / (5.0 + k) + k) * np.cos(yy / (4.0 + k)) for k in range(c)])
    return (base + 0.1 * f32_frame((c, h, w), seed)).astype(np.float32)


@pytest.mark.parametrize("patch,search,h,w", [(9, 31, 21, 45), (15, 21, 19, 40)])
def test_nl_means_dx_batches(hb, oracle, patch, search, h, w):
    """Search rows wider than one pass of the generic kernel: patch 9 / search 31 runs dx batches of 8, 8, 8 and 7 (the
    partial last batch), patch 15 / search 21 three batches of 7.  Every batch after the first reads its neighbours at
    column offset dx0 > 0."""
    nd, smem = nl_nd(patch, search)
    assert nd < search and smem > 48 * 1024
    assert (search % nd != 0) == (patch == 9)
    inp = smooth_f32(3, h, w, patch)
    nl_check(hb, oracle, inp, patch, search, 0.4, "nl_means")


def test_nl_means_largest_patch_and_search(hb, oracle):
    """patch 31 / search 63, the largest accepted pair: one dx per pass and 176 080 bytes of shared memory.  A tiny
    frame (the oracle costs search^2 x patch^2 per pixel)."""
    nd, smem = nl_nd(31, 63)
    assert nd == 1 and smem == 176080
    inp = smooth_f32(3, 12, 20, 31)
    nl_check(hb, oracle, inp, 31, 63, 0.5, "nl_means")


@pytest.mark.parametrize("variant,kernel", [(0, "nl_means_window"), (1, "nl_means")])
@pytest.mark.parametrize("in_c,c0", [(1, 0), (4, 0), (3, 1)])
def test_nl_means_input_channels(hb, oracle, in_c, c0, variant, kernel):
    """Inputs of 1 and 4 channels and one whose channels are [1, 4): both kernels read channel clamp(c, c0, c0 + in_c - 1)
    for c = 0..2 (the output always has channels [0, 3)).  Patch 3 / search 7 takes the window kernel by default; the
    variant hook forces the generic one."""
    inp = smooth_f32(in_c, 37, 53, 10 * in_c + c0)
    nl_check(hb, oracle, inp, 3, 7, 0.12, kernel, variant, in_mins=(0, 0, c0))


@pytest.mark.parametrize("patch", [3, 7])
@pytest.mark.parametrize("h,w", [(1, 1), (17, 33), (37, 53), (70, 101)])
def test_nl_means_window_kernel_bit_identical_to_generic(hb, patch, h, w):
    """The window kernel performs the generic kernel's float operations in the same order: the two must agree bit for
    bit on ragged frames, not only each within tolerance of the oracle.  Content on which every offset carries weight
    (on uniform noise at sigma 0.12 only the centre does, and a shared mistake in an off-centre offset would not show)."""
    inp = sensitive_frame(3, h, w, 0.12, 1000 * patch + h + w)
    with nl_variant(hb, 0), kernels_run(hb) as ran:
        a = run_nl(hb, inp, patch, 7, 0.12)
    assert list(ran) == ["nl_means_window"], sorted(ran)
    with nl_variant(hb, 1), kernels_run(hb) as ran:
        b = run_nl(hb, inp, patch, 7, 0.12)
    assert list(ran) == ["nl_means"], sorted(ran)
    assert np.array_equal(a, b), f"{np.count_nonzero(a != b)} samples differ"


# ---- local_laplacian -------------------------------------------------------------------------------------------------

def ll_check(hb, oracle, img, levels, alpha, beta=1.0):
    got = run_local_laplacian(hb, img, levels, alpha, beta)
    want = oracle.local_laplacian(img, levels, alpha, beta)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"levels {levels} alpha {alpha}: {len(bad)} mismatching samples, first at (c,y,x)={bad[0]}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


@pytest.fixture(scope="module")
def frame_300x500():
    return smooth_u16_frame((3, 300, 500), 3)


@pytest.mark.parametrize("levels", [3, 9, 31, 32])
def test_local_laplacian_level_counts(hb, oracle, frame_300x500, levels):
    """Intensity level counts far from 8, up to the largest accepted: the generic kernels (the fast ones are built for
    8), K planes per pyramid pixel, a remap table of 2 * 256 * (levels - 1) + 1 entries (15 873 at 32)."""
    with kernels_run(hb) as ran:
        ll_check(hb, oracle, frame_300x500, levels, 1.0 / (levels - 1))
    assert "ll_level1_generic" in ran and "ll_final" in ran and "ll_final2" not in ran, sorted(ran)


@pytest.mark.parametrize("levels,alpha,beta", [(8, -1.0 / 7.0, 1.0), (8, -3.0 / 7.0, 0.6), (5, -0.25, 1.0)])
def test_local_laplacian_negative_alpha(hb, oracle, levels, alpha, beta):
    """alpha < 0 flattens detail instead of enhancing it: the remap table changes sign."""
    ll_check(hb, oracle, u16_frame((3, 90, 130), 17), levels, alpha, beta)


def test_local_laplacian_remap_cache_eviction(hb, oracle):
    """The remap tables are cached per (device, levels, alpha) and all freed once 64 are held.  65 alphas never used
    elsewhere in the suite guarantee at least one eviction, whatever the cache held before; every result must equal
    the oracle, and so must the first alpha again (rebuilt after the eviction) and the same alpha at another level
    count (a different key)."""
    img = u16_frame((3, 24, 40), 65)
    alphas = [0.0123 + 0.0071 * i for i in range(65)]
    for a in alphas:
        ll_check(hb, oracle, img, 8, a)
    ll_check(hb, oracle, img, 8, alphas[0])
    ll_check(hb, oracle, img, 5, alphas[0])
    ll_check(hb, oracle, img, 8, alphas[1])
