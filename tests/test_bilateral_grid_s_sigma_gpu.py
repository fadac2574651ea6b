"""halide_b200_bilateral_grid_s_sigma on the GPU: bilateral_grid with the generator's s_sigma (grid cell size) chosen per
call, against oracle/oracle_bilateral_grid.cpp run with the same s_sigma.  Float pipeline: 1e-4 relative, the tolerance
of test_bilateral_grid_gpu.py.  s_sigma = 8 must be bilateral_grid itself, bit for bit; every other cell size runs the
any-S kernels (bg_hist_blurz_s, bg_slice_s)."""
import numpy as np
import pytest

from util import f32_frame, kernels_run

pytestmark = pytest.mark.gpu
RTOL = 1e-4
S_VALUES = [1, 2, 3, 4, 5, 7, 9, 12, 16, 31, 32, 64, 100, 128]


def close(got, want, floor=1e-6):
    assert np.isfinite(got).all()
    err = np.abs(got - want) / np.maximum(np.abs(want), floor)
    assert err.max() <= RTOL, f"max rel err {err.max()} at {np.unravel_index(err.argmax(), err.shape)}"


def run(hb, inp, s_sigma, r_sigma, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.float32)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.bilateral_grid_s_sigma(bi, s_sigma, r_sigma, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out


def bg_zmax(r_sigma):  # bilateral_grid.cu: inv_r = 1 / r_sigma, zmax = int(1 * inv_r + 0.5), in float32
    inv_r = np.float32(1.0) / np.float32(r_sigma)
    return int(np.float32(np.float32(1.0) * inv_r) + np.float32(0.5))


def r_sigma_for(zmax):
    r = float(np.float32(1.0) / np.float32(zmax))
    assert bg_zmax(r) == zmax
    return r


def bg_frame(kind, h, w):  # the frames of test_param_extremes_gpu.py
    if kind == "noise":
        return f32_frame((h, w), h * w)
    if kind == "ramp":
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        return ((xx / (w - 1)) * 0.75 + (yy / (h - 1)) * 0.25).astype(np.float32)
    return (f32_frame((h, w), h + w) * 3.0 - 1.0).astype(np.float32)


@pytest.mark.parametrize("s", S_VALUES)
def test_matches_oracle_across_sizes(hb, oracle, s):
    for h, w in [(1, 1), (max(1, s - 1), s + 1), (61, 107), (240, 519)]:
        inp = f32_frame((h, w), 1000 * s + h + w)
        close(run(hb, inp, s, 0.1), oracle.bilateral_grid(inp, 0.1, s_sigma=s))


@pytest.mark.parametrize("s", [1, 16, 128])
@pytest.mark.parametrize("kind", ["noise", "ramp", "outside"])
def test_r_sigma_and_bin_counts(hb, oracle, s, kind):
    """r_sigma 0.05 / 0.25 / 1.0, and zmax on both sides of each shared-memory opt-in (47 / 48 histogram, 126 / 127
    bilateral_grid's slice) up to the largest accepted grid (199: 200 bins)."""
    inp = bg_frame(kind, 61, 107)
    for r in [0.05, 0.25, 1.0] + [r_sigma_for(z) for z in (47, 48, 126, 127, 199)]:
        close(run(hb, inp, s, r), oracle.bilateral_grid(inp, r, s_sigma=s))


@pytest.mark.parametrize("s", [3, 5, 12, 33])
def test_crops_with_negative_unaligned_mins(hb, oracle, s):
    inp = f32_frame((130, 170), s)
    kw = dict(out_shape=(70, 101), in_mins=(-29, -21), out_mins=(-19, -11))
    close(run(hb, inp, s, 0.1, **kw), oracle.bilateral_grid(inp, 0.1, s_sigma=s, **kw))
    kw = dict(out_shape=(45, 61), in_mins=(-13, 5), out_mins=(-6, 23))
    close(run(hb, inp, s, 0.25, **kw), oracle.bilateral_grid(inp, 0.25, s_sigma=s, **kw))


@pytest.mark.parametrize("s", [2, 6, 16])
def test_padded_stride_and_misaligned_base_on_the_device(hb, oracle, s):
    """Device-resident torch views: rows padded to a wider pitch, and input and output starting one float past a
    16-byte boundary (no float4 path for any pixel)."""
    import torch
    h, w = 75, 133
    base = f32_frame((h, w + 19), 40 + s)  # row pitches of 152 and 140 floats: 16-byte multiples, so off = 0 is aligned
    tin = torch.from_numpy(base).cuda()
    for off in (0, 1, 3):
        view_in = tin[:, off:off + w]
        ref = oracle.bilateral_grid(np.ascontiguousarray(base[:, off:off + w]), 0.1, s_sigma=s)
        tout_full = torch.zeros((h, w + 7), dtype=torch.float32, device="cuda")
        view_out = tout_full[:, off:off + w]
        hb.filters.bilateral_grid_s_sigma(hb.HalideBuffer.from_torch(view_in), s, 0.1, hb.HalideBuffer.from_torch(view_out))
        torch.cuda.synchronize()
        close(view_out.cpu().numpy(), ref)
        assert not tout_full[:, :off].any() and not tout_full[:, off + w:].any()


@pytest.mark.parametrize("s", [4, 16, 64])
def test_8k_random_frame_regions(hb, oracle, s):
    """7680 x 4320 (BASELINE.json config 3) random frame: regions of the full result against the oracle on the crop
    that determines them (cells of s px, the blurs reach 2 cells and the slice 1: a margin of 5 s px is enough); the
    crops keep their frame coordinates as mins, since cell boundaries are absolute."""
    h, w = 4320, 7680
    inp = f32_frame((h, w), 21 + s)
    got = run(hb, inp, s, 0.1)
    m = 5 * s
    for (y0, x0) in [(0, 0), (h - 96, w - 96), (2001, 3333), (4096 - 45, 4096 - 51)]:
        n = 96
        ya, yb, xa, xb = max(0, y0 - m), min(h, y0 + n + m), max(0, x0 - m), min(w, x0 + n + m)
        crop = np.ascontiguousarray(inp[ya:yb, xa:xb])
        want = oracle.bilateral_grid(crop, 0.1, in_mins=(xa, ya), out_mins=(xa, ya), s_sigma=s)
        close(got[y0:y0 + n, x0:x0 + n], want[y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n])


@pytest.mark.parametrize("s", [3, 16, 128])
def test_constant_8k_frame_is_a_fixed_point(hb, oracle, s):
    """A constant frame comes back constant: every cell of it is the same, so the whole output is the tile of one cell's
    s x s outputs, bit for bit, and that cell matches the oracle on a small constant frame within the float tolerance.
    The value itself is 0.37 only up to the rounding of the generator's sequential cell sums (s^2 float additions of
    0.37: 2.1e-4 relative at s = 128), which the oracle shares."""
    h, w = 4320, 7680
    inp = np.full((h, w), 0.37, np.float32)
    got = run(hb, inp, s, 0.1)
    cell = got[:s, :s]
    assert np.array_equal(got, np.tile(cell, (-(-h // s), -(-w // s)))[:h, :w])
    m = 2 * s + 7
    close(got[:m, :m], oracle.bilateral_grid(np.full((m, m), 0.37, np.float32), 0.1, s_sigma=s))
    assert np.allclose(got, 0.37, rtol=max(1e-5, s * s * 2.0 ** -24))


@pytest.mark.parametrize("s", [2, 8, 13, 64])
def test_repeated_calls_give_identical_bytes(hb, s):
    inp = f32_frame((300, 517), 77 + s)
    a, b = run(hb, inp, s, 0.1), run(hb, inp, s, 0.1)
    assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("s", [1, 4, 5, 8, 9, 128])
def test_kernels_launched(hb, s):
    """s_sigma = 8 runs bilateral_grid's kernels and equals bilateral_grid bit for bit; any other s_sigma runs the any-S
    histogram and slice kernels."""
    inp = f32_frame((97, 203), 5)
    with kernels_run(hb) as ran:
        got = run(hb, inp, s, 0.1)
    if s == 8:
        assert set(ran) == {"bg_hist_blurz", "bg_blur_xy", "bg_slice"}, sorted(ran)
        want = np.zeros_like(inp)
        bi, bo = hb.HalideBuffer.from_numpy(inp), hb.HalideBuffer.from_numpy(want, host_dirty=False)
        hb.filters.bilateral_grid(bi, 0.1, bo)
        bo.copy_to_host()
        assert got.tobytes() == want.tobytes()
    else:
        assert set(ran) == {"bg_hist_blurz_s", "bg_blur_xy", "bg_slice_s"}, sorted(ran)


def test_device_resident_torch_tensors(hb, oracle):
    import torch
    inp = f32_frame((120, 250), 9)
    tin = torch.from_numpy(inp).cuda()
    tout = torch.empty_like(tin)
    hb.filters.bilateral_grid_s_sigma(hb.HalideBuffer.from_torch(tin), 11, 0.1, hb.HalideBuffer.from_torch(tout))
    torch.cuda.synchronize()
    close(tout.cpu().numpy(), oracle.bilateral_grid(inp, 0.1, s_sigma=11))
