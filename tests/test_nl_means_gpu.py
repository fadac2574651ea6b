"""GPU parity tests for nl_means through the C ABI against oracle/oracle_nl_means.cpp, within a 1e-4 relative tolerance
(BASELINE.json north_star).  The kernels match the oracle bit for bit; test_nl_means_exact_gpu.py holds them to that, on
content where every search offset carries weight.  Uniform noise in [0, 1) at sigma 0.12 is not such content (every
off-centre weight is about exp(-35)), so the tests here that compare kernels with each other or at config 4's size use
nl_means_exact.sensitive_frame."""
import numpy as np
import pytest

from nl_means_exact import sensitive_frame
from util import f32_frame

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def run(hb, inp, patch, search, sigma, out_shape=None, in_mins=None, out_mins=None):
    out = np.zeros(inp.shape if out_shape is None else out_shape, np.float32)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.nl_means(bi, patch, search, sigma, bo)
    bo.copy_to_host()
    return out


def close(got, want):
    assert np.isfinite(got).all()
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-3)
    assert err.max() <= RTOL, f"max rel err {err.max()} at {np.unravel_index(err.argmax(), err.shape)}"


@pytest.mark.parametrize("h,w", [(1, 1), (5, 9), (16, 32), (33, 47), (70, 101)])
def test_config4_parameters(hb, oracle, h, w):
    inp = f32_frame((3, h, w), h * 3 + w)
    close(run(hb, inp, 3, 7, 0.12), oracle.nl_means(inp, 3, 7, 0.12))


@pytest.mark.parametrize("patch,search,sigma", [(7, 7, 0.12), (1, 1, 0.5), (2, 4, 0.2), (5, 9, 0.3), (7, 13, 0.12)])
def test_parameter_sweep(hb, oracle, patch, search, sigma):
    inp = f32_frame((3, 40, 52), patch * 10 + search)
    close(run(hb, inp, patch, search, sigma), oracle.nl_means(inp, patch, search, sigma))


def test_smooth_content_and_offsets(hb, oracle):
    yy, xx = np.mgrid[0:50, 0:70].astype(np.float32)
    base = 0.5 + 0.4 * np.sin(xx / 9.0) * np.cos(yy / 7.0)
    inp = np.stack([base, base * 0.8, 1.0 - base]).astype(np.float32)
    inp += f32_frame(inp.shape, 1) * 0.05
    kw = dict(out_shape=(3, 30, 41), in_mins=(-4, 2, 0), out_mins=(1, 6, 0))
    close(run(hb, inp, 3, 7, 0.12, **kw), oracle.nl_means(inp, 3, 7, 0.12, **kw))


def test_output_channel_constraint(hb):
    from halide_b200 import HalideBuffer, HalideError, filters
    inp = f32_frame((3, 8, 8), 0)
    bi = HalideBuffer.from_numpy(inp)
    bo = HalideBuffer.from_numpy(np.zeros((2, 8, 8), np.float32))
    with pytest.raises(HalideError) as e:
        filters.nl_means(bi, 3, 7, 0.12, bo)
    assert e.value.code == -8  # non_local_means.dim(2).set_bounds(0, 3), generator :68


def test_constant_frame_4k_band(hb):
    """Config-4 frame width: a constant frame must be reproduced exactly (all weights equal 1)."""
    inp = np.full((3, 540, 3840), 0.25, np.float32)
    got = run(hb, inp, 3, 7, 0.12)
    assert np.allclose(got, 0.25, rtol=1e-6)


def test_4k_random_frame_regions(hb, oracle):
    """Config 4 size (3840 x 2160 x 3) on a sensitive frame: regions of the full-size result against the oracle on the
    crop that determines them (footprint = search/2 + patch/2 = 4 px; margin 16)."""
    h, w = 2160, 3840
    inp = sensitive_frame(3, h, w, 0.12, 33)
    got = run(hb, inp, 3, 7, 0.12)
    for (y0, x0) in [(0, 0), (h - 64, w - 64), (1000, 1900), (540 - 32, 3000)]:
        n, m = 64, 16
        ya, yb, xa, xb = max(0, y0 - m), min(h, y0 + n + m), max(0, x0 - m), min(w, x0 + n + m)
        crop = np.ascontiguousarray(inp[:, ya:yb, xa:xb])
        want = oracle.nl_means(crop, 3, 7, 0.12, in_mins=(xa, ya, 0), out_mins=(xa, ya, 0))
        close(got[:, y0:y0 + n, x0:x0 + n], want[:, y0 - ya:y0 - ya + n, x0 - xa:x0 - xa + n])


@pytest.mark.parametrize("variant", [1, 0])
def test_generic_and_window_kernels(hb, oracle, variant):
    """The generic kernel (variant 1, hook halide_b200_nl_means_variant) and the default, which takes the register-window
    kernel for patch 3 / 7 and search 7, against the oracle: ragged sizes, a crop with offsets, and a patch / search pair
    the window kernel does not cover (the default must fall back to the generic kernel by itself)."""
    l = hb.load_library()
    try:
        l.halide_b200_nl_means_variant(variant)
        for h, w in ((1, 1), (16, 32), (33, 47), (70, 101)):
            inp = sensitive_frame(3, h, w, 0.12, 11 * variant + h + w)
            close(run(hb, inp, 3, 7, 0.12), oracle.nl_means(inp, 3, 7, 0.12))
        inp = sensitive_frame(3, 40, 52, 0.12, 77)
        close(run(hb, inp, 7, 7, 0.12), oracle.nl_means(inp, 7, 7, 0.12))
        inp = sensitive_frame(3, 40, 52, 0.3, 77)
        close(run(hb, inp, 5, 9, 0.3), oracle.nl_means(inp, 5, 9, 0.3))
        kw = dict(out_shape=(3, 30, 41), in_mins=(-4, 2, 0), out_mins=(1, 6, 0))
        inp = sensitive_frame(3, 50, 70, 0.12, 5)
        close(run(hb, inp, 3, 7, 0.12, **kw), oracle.nl_means(inp, 3, 7, 0.12, **kw))
    finally:
        l.halide_b200_nl_means_variant(0)
