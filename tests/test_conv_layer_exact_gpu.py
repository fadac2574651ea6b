"""conv_layer's 3xTF32 tensor-core contraction against a float64 reference (tests/conv_exact.py): bit for bit on data
where the split and the accumulation are exact, within a derived bound on harness-scale data, and across calls."""
import numpy as np
import pytest

from conv_exact import HARNESS_CASES, OUT_SHAPE, dense_exact, harness, harness_bound, one_hot, run

pytestmark = pytest.mark.gpu


def _mismatch(got, want):
    bad = ~(got == want)
    idx = tuple(int(i) for i in np.argwhere(bad)[0]) if bad.any() else None
    return f"{int(bad.sum())} of {bad.size} outputs differ; first at (n, y, x, co) = {idx}: got {got[idx] if idx else None}, " \
           f"want {want[idx] if idx else None}"


@pytest.mark.parametrize("part", [0, 1])
def test_one_hot_filters_sum_exactly_three_products(hb, part):
    """Every co reads one (ky, kx, ci): pins the tap / channel mapping of both operands and that the kernel sums
    hi*hi + hi*lo + lo*hi, not a*b and not fewer terms."""
    inp, filt, bias, want, _ = one_hot(part)
    got = run(hb, inp, filt, bias)
    assert np.array_equal(got, want), _mismatch(got, want)


@pytest.mark.parametrize("mirrored", [False, True], ids=["lo_in_input", "lo_in_filter"])
def test_dense_exact_data_bit_for_bit(hb, mirrored):
    """All 36 K steps into both accumulators, bias, relu, every tile and image, on data with exact partial sums."""
    inp, filt, bias, want = dense_exact(mirrored)
    got = run(hb, inp, filt, bias)
    assert np.array_equal(got, want), _mismatch(got, want)


@pytest.mark.parametrize("case", HARNESS_CASES)
def test_harness_scale_within_derived_bound(hb, case):
    """Every output within E * sum |a*b| + 2^-24 |result| of float64 (conv_exact.E_SPLIT_ACCUM).  The bound is derived:
    a ratio above 1 is a kernel error, not a reason to raise E."""
    inp, filt, bias = harness(case)
    want, bound = harness_bound(inp, filt, bias)
    got = run(hb, inp, filt, bias)
    assert np.isfinite(got).all()
    ratio = np.abs(got.astype(np.float64) - want) / bound
    worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    assert ratio.max() <= 1.0, f"max err / bound = {ratio.max():.3f} at (n, y, x, co) = {worst}"


def test_reused_buffers_take_new_data(hb):
    """Two calls on the same buffers with different data each equal a call on fresh buffers."""
    data = [harness("signed"), harness("channel_scales")]
    fresh = [run(hb, *d) for d in data]
    arrays = [a.copy() for a in data[0]]
    bufs = [hb.HalideBuffer.from_numpy(a) for a in arrays]
    out = np.full(OUT_SHAPE, np.nan, np.float32)
    bo = hb.HalideBuffer.from_numpy(out)
    hb.lib.check(hb.capi.halide_copy_to_device(None, bo.ptr, None))
    for d, want in zip(data, fresh):
        for a, b, new in zip(arrays, bufs, d):
            a[...] = new
            b.set_host_dirty(True)
        hb.filters.conv_layer(*bufs, bo)
        bo.copy_to_host()
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), _mismatch(out, want)


def test_repeated_call_is_bitwise_identical(hb):
    d = harness("channel_scales")
    a, b = run(hb, *d), run(hb, *d)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), _mismatch(a, b)


def test_device_resident_torch_tensors_match_host_buffers(hb):
    import torch
    d = harness("signed")
    want = run(hb, *d)
    ti, tf, tb = (torch.from_numpy(a).cuda() for a in d)
    to = torch.full(OUT_SHAPE, float("nan"), dtype=torch.float32, device="cuda")
    bo = hb.HalideBuffer.from_torch(to)
    hb.filters.conv_layer(hb.HalideBuffer.from_torch(ti), hb.HalideBuffer.from_torch(tf), hb.HalideBuffer.from_torch(tb), bo)
    bo.device_sync()
    torch.cuda.synchronize()
    got = to.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), _mismatch(got, want)
