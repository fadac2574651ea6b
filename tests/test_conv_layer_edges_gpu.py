"""conv_layer and halide_b200_conv_layer_any_shape byte for byte against tests/conv_edge.py's want (the oracle's result,
checked by test_conv_layer_edges.py): infinities and NaNs in every operand, sums and products that overflow, an exponent
sweep down to subnormal lo parts and products, and -0.0.  Bytes, not values: +0.0 is not -0.0 and inf is not a large
finite number.  relu never gives NaN, so the NaN pre-fill of conv_any_exact.run still marks an output not written."""
import numpy as np
import pytest

import conv_any_exact as cx
import conv_edge as ce
import conv_exact

pytestmark = pytest.mark.gpu
SHAPE_IDS = [str(s) for s in ce.SHAPES]


def _mismatch(got, want):
    bad = got.view(np.uint32) != want.view(np.uint32)
    idx = tuple(int(i) for i in np.argwhere(bad)[0]) if bad.any() else None
    return f"{int(bad.sum())} of {bad.size} outputs differ; first at (n, y, x, co) = {idx}: got {got[idx] if idx else None}, " \
           f"want {want[idx] if idx else None}"


def _same_bytes(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("dataset", ce.DATASET_IDS)
@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_equals_want_byte_for_byte(hb, shape, dataset):
    """At conv_layer's shape both entry points, which must also agree with each other."""
    inp, filt, bias, want = ce.datasets(shape)[dataset]()
    got = cx.run(hb, inp, filt, bias)
    assert _same_bytes(got, want), _mismatch(got, want)
    if shape == cx.FIXED:
        fixed = conv_exact.run(hb, inp, filt, bias)
        assert _same_bytes(fixed, want), _mismatch(fixed, want)


@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_non_finite_values_do_not_leak(hb, shape):
    """Harness-scale signed data with +-inf and NaNs planted in the input: the outputs they reach equal want byte for
    byte, every other output stays within the derived bound of the data without them."""
    inp, filt, bias, want, touched = ce.planted_harness(shape)
    entries = [None, hb.filters.conv_layer] if shape == cx.FIXED else [None]
    clean = [np.where(np.isfinite(a), a, np.float32(0)) for a in (inp, filt, bias)]
    ref, bound = cx.harness_bound(*clean)
    for entry in entries:
        got = cx.run(hb, inp, filt, bias, entry)
        assert _same_bytes(got[touched], want[touched]), _mismatch(np.where(touched, got, 0), np.where(touched, want, 0))
        err = np.abs(got.astype(np.float64) - ref)[~touched] / bound[~touched]
        assert np.isfinite(got[~touched]).all() and (err <= 1.0).all(), err.max()


@pytest.mark.parametrize("dataset", ["inf_w_lo-mirrored", "f_low_nan-direct", "b_inf-direct", "overflow_sum"])
def test_padded_device_views_take_the_scalar_split(hb, dataset):
    """Device-resident torch views with odd pitches (not multiples of four floats: the split's scalar path, no float2
    stores) give want byte for byte and leave the padding alone."""
    import torch
    shape = (1, 160, 136, 9, 5)
    n, ci, co, w, h = shape
    inp, filt, bias, want = ce.datasets(shape)[dataset]()
    ti_full = torch.zeros((n, h + 3, w + 3, ci + 1), device="cuda")
    ti = ti_full[:, :h + 2, :w + 2, :ci]
    ti.copy_(torch.from_numpy(inp))
    tf_full = torch.zeros((ci, 4, 3, co + 1), device="cuda")
    tf = tf_full[:, :3, :, :co]
    tf.copy_(torch.from_numpy(filt))
    to_full = torch.full((n, h + 1, w + 1, co + 1), float("nan"), device="cuda")
    to = to_full[:, :h, :w, :co]
    bufs = [hb.HalideBuffer.from_torch(t) for t in (ti, tf, torch.from_numpy(bias).cuda(), to)]
    hb.filters.conv_layer_any_shape(*bufs)
    torch.cuda.synchronize()
    got = to.cpu().numpy()
    assert _same_bytes(got, want), _mismatch(got, want)
    written = torch.zeros_like(to_full, dtype=torch.bool)
    written[:, :h, :w, :co] = True
    assert torch.isnan(to_full[~written]).all(), "the output's padding was written"


def test_kernels_launched(hb):
    """Non-finite sums are recomputed inside the GEMM kernels: no other kernel runs."""
    from util import kernels_run
    for shape, gemm in [((1, 160, 136, 9, 5), "conv_layer_tc_n128_fold"), ((1, 1024, 64, 6, 6), "conv_layer_tc_n64_fold"),
                        ((2, 32, 8, 1, 1), "conv_layer_tc_n64"),
                        ((3, 37, 75, 29, 17), "conv_layer_tc_n128"), (cx.FIXED, "conv_layer_tc_n128")]:
        d = ce.planted(shape, "inf_w_lo", False)[:3]
        with kernels_run(hb) as ran:
            cx.run(hb, *d)
        assert set(ran) == {"conv_split_input_any", "conv_prep_filter_any", gemm}, (shape, sorted(ran))
    with kernels_run(hb) as ran:
        conv_exact.run(hb, *d)
    assert set(ran) == {"conv_split_input", "conv_prep_filter", "conv_layer_tc"}, sorted(ran)
