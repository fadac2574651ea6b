"""GPU parity tests for conv_layer through the C ABI (fixed shapes of the generator).  Float pipeline: 1e-4 relative."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
N, CI, CO, W, H = 5, 128, 128, 100, 80


def make(seed, scale):
    rng = np.random.default_rng(seed)
    inp = (rng.random((N, H + 2, W + 2, CI), dtype=np.float32) * scale).astype(np.float32)
    filt = (rng.random((CI, 3, 3, CO), dtype=np.float32) * scale).astype(np.float32)
    bias = (rng.random((CO,), dtype=np.float32) * scale).astype(np.float32)
    return inp, filt, bias


def run(hb, inp, filt, bias):
    out = np.zeros((N, H, W, CO), np.float32)
    bi, bf, bb = hb.HalideBuffer.from_numpy(inp), hb.HalideBuffer.from_numpy(filt), hb.HalideBuffer.from_numpy(bias)
    bo = hb.HalideBuffer.from_numpy(out, host_dirty=False)
    hb.filters.conv_layer(bi, bf, bb, bo)
    bo.copy_to_host()
    return out


# the harness fills with raw rand() up to 2^31
@pytest.mark.parametrize("seed,scale", [(0, 1.0), (1, 2147483648.0), (3, 1.0), (4, 2147483648.0)])
def test_matches_oracle(hb, oracle, seed, scale):
    inp, filt, bias = make(seed, scale)
    got = run(hb, inp, filt, bias)
    want = oracle.conv_layer(inp, filt, bias)
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
    assert np.isfinite(got).all() and err.max() <= 1e-4, err.max()


def test_signed_data_and_relu(hb, oracle):
    inp, filt, bias = make(2, 1.0)
    inp -= 0.5
    filt -= 0.5
    got = run(hb, inp, filt, bias)
    want = oracle.conv_layer(inp, filt, bias)
    assert (got >= 0).all() and (got == 0).any()
    # mixed signs cancel: compare against the magnitude of the accumulated terms, not of the result
    assert np.max(np.abs(got - want)) <= 1e-4 * 1152 * 0.25


def test_wrong_shape_is_a_constraint_violation(hb):
    from halide_b200 import HalideBuffer, HalideError, filters
    inp, filt, bias = make(0, 1.0)
    bi = HalideBuffer.from_numpy(inp[:, :, :-1, :].copy())
    bf, bb = HalideBuffer.from_numpy(filt), HalideBuffer.from_numpy(bias)
    bo = HalideBuffer.from_numpy(np.zeros((N, H, W, CO), np.float32))
    with pytest.raises(HalideError) as e:
        filters.conv_layer(bi, bf, bb, bo)
    assert e.value.code == -8
