"""halide_b200_conv_layer_any_shape on the GPU: against oracle/oracle_conv_layer.cpp (1e-4 relative, conv_layer's bar),
against a float64 reference within the bound conv_exact.py derives (the same constant at every CI), bit for bit on exact
data, byte for byte against conv_layer at its shape, and across buffer layouts.  Shapes are (N, CI, CO, W, H)."""
import numpy as np
import pytest

import conv_any_exact as cx
import conv_exact

pytestmark = pytest.mark.gpu
RTOL = 1e-4
# tools/conv_any_shape_bench.py's shapes (the larger ones at a smaller N, which keeps the CPU oracle quick) ...
SHAPES = [cx.FIXED, (1, 3, 64, 224, 224), (2, 64, 64, 56, 56), (3, 128, 128, 28, 28), (3, 256, 256, 14, 14), (5, 512, 512, 7, 7),
          (1, 1024, 1024, 14, 14), (3, 37, 75, 29, 17),
          # ... one pixel; CO below a fragment; an odd K-step count with a second CO tile of 8 channels; 288 K steps on the N = 64 tile
          (1, 1, 1, 1, 1), (2, 32, 8, 1, 1), (1, 160, 136, 9, 5), (1, 1024, 64, 6, 6)]
SMALL = [s for s in SHAPES if 2 * 9 * s[0] * s[1] * s[2] * s[3] * s[4] < 2e9]  # for the generators that loop in Python
# the exact-data tests must reach a shape that folds on each N tile
assert any(cx.folds(s[1]) > 0 and cx.n_tile(s[2]) == 128 for s in SMALL) and any(cx.folds(s[1]) > 0 and cx.n_tile(s[2]) == 64 for s in SMALL)


def _mismatch(got, want):
    bad = ~(got == want)
    idx = tuple(int(i) for i in np.argwhere(bad)[0]) if bad.any() else None
    return f"{int(bad.sum())} of {bad.size} outputs differ; first at (n, y, x, co) = {idx}: got {got[idx] if idx else None}, " \
           f"want {want[idx] if idx else None}"


def _same_bytes(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_matches_oracle(hb, oracle, shape):
    inp, filt, bias = cx.harness("rand", shape)
    got, want = cx.run(hb, inp, filt, bias), oracle.conv_layer(inp, filt, bias)
    assert np.isfinite(got).all(), f"{int((~np.isfinite(got)).sum())} outputs not written"
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-6)
    assert err.max() <= RTOL, f"max rel err {err.max()} at {np.unravel_index(err.argmax(), err.shape)}"


@pytest.mark.parametrize("case", ["signed", "channel_scales"])
@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_within_derived_bound_at_every_ci(hb, shape, case):
    """E_SPLIT_ACCUM is derived for 216 chained additions per accumulator; the folds keep it valid at CI = 1024."""
    inp, filt, bias = cx.harness(case, shape)
    got = cx.run(hb, inp, filt, bias)
    assert np.isfinite(got).all()
    ratio = cx.worst_ratio(got, inp, filt, bias)
    assert ratio <= 1.0, f"max err / bound = {ratio:.3f} ({cx.folds(shape[1])} folds)"


@pytest.mark.parametrize("shape", SMALL, ids=str)
def test_one_hot_filters_bit_for_bit(hb, shape):
    inp, filt, bias, want = cx.one_hot(shape)
    got = cx.run(hb, inp, filt, bias)
    assert np.array_equal(got, want), _mismatch(got, want)


@pytest.mark.parametrize("mirrored", [False, True], ids=["lo_in_input", "lo_in_filter"])
@pytest.mark.parametrize("shape", SMALL, ids=str)
def test_dense_exact_data_bit_for_bit(hb, shape, mirrored):
    """Includes shapes that fold (CI = 160, 256, 512, 1024) and shapes on the N = 64 tile (CO = 1, 8, 64)."""
    inp, filt, bias, want = cx.dense_exact(shape, mirrored)
    got = cx.run(hb, inp, filt, bias)
    assert np.array_equal(got, want), _mismatch(got, want)


@pytest.mark.parametrize("case", conv_exact.HARNESS_CASES)
def test_fixed_shape_equals_conv_layer_byte_for_byte(hb, case):
    d = conv_exact.harness(case)
    got, want = cx.run(hb, *d), conv_exact.run(hb, *d)
    assert _same_bytes(got, want), _mismatch(got, want)


def test_kernels_launched(hb):
    """The N tile follows CO and the folding form K steps > 36; conv_layer keeps its own kernels."""
    from util import kernels_run
    for shape, gemm in [((1, 128, 128, 5, 3), "conv_layer_tc_n128"), ((1, 129, 65, 5, 3), "conv_layer_tc_n128_fold"),
                        ((1, 128, 64, 5, 3), "conv_layer_tc_n64"), ((1, 129, 64, 5, 3), "conv_layer_tc_n64_fold")]:
        with kernels_run(hb) as ran:
            cx.run(hb, *cx.harness("rand", shape))
        assert set(ran) == {"conv_split_input_any", "conv_prep_filter_any", gemm}, (shape, sorted(ran))
    with kernels_run(hb) as ran:
        conv_exact.run(hb, *conv_exact.harness("rand"))
    assert set(ran) == {"conv_split_input", "conv_prep_filter", "conv_layer_tc"}, sorted(ran)


# ---- layouts: device-resident torch views, so that memory outside relu's region can be inspected ----------------------

def _torch_call(hb, ti, tf, tb, to, mins=(None, None, None, None)):
    bufs = [hb.HalideBuffer.from_torch(t, m) for t, m in zip((ti, tf, tb, to), mins)]
    hb.filters.conv_layer_any_shape(*bufs)
    import torch
    torch.cuda.synchronize()


@pytest.mark.parametrize("shape", [(3, 37, 75, 29, 17), (2, 160, 64, 12, 9)], ids=str)
def test_padded_strides_equal_the_dense_call(hb, shape):
    """Row- and image-padded input and output (odd pitches: no float2 stores; even ones: float2 stores) and a filter with
    padded strides give the dense call's bytes, and the output's padding keeps its NaN pre-fill."""
    import torch
    n, ci, co, w, h = shape
    inp, filt, bias = cx.harness("signed", shape)
    want = cx.run(hb, inp, filt, bias)
    for pad in (1, 2):
        ti_full = torch.zeros((n, h + 2 + pad, w + 2 + pad, ci + pad), device="cuda")
        ti = ti_full[:, :h + 2, :w + 2, :ci]
        ti.copy_(torch.from_numpy(inp))
        tf_full = torch.zeros((ci, 3 + pad, 3, co + pad), device="cuda")
        tf = tf_full[:, :3, :, :co]
        tf.copy_(torch.from_numpy(filt))
        to_full = torch.full((n, h + pad, w + pad, co + pad), float("nan"), device="cuda")
        to = to_full[:, :h, :w, :co]
        _torch_call(hb, ti, tf, torch.from_numpy(bias).cuda(), to)
        got = to.cpu().numpy()
        assert _same_bytes(got, want), (pad, _mismatch(got, want))
        written = torch.zeros_like(to_full, dtype=torch.bool)
        written[:, :h, :w, :co] = True
        assert torch.isnan(to_full[~written]).all(), "the output's padding was written"


@pytest.mark.parametrize("shape", [(2, 37, 75, 13, 7), (2, 64, 40, 8, 8)], ids=str)
def test_crop_of_larger_tensors_with_nonzero_mins(hb, shape):
    """relu is a crop of a larger tensor with nonzero mins in all four dimensions; input, filter and bias are the larger
    tensors themselves, with their own mins.  Equals the dense call on the matching crops; nothing outside the crop is
    written."""
    import torch
    n, ci, co, w, h = shape
    c0, x0, y0, n0 = 5, 3, 2, 1  # the crop's offsets inside the larger tensors
    big = (n + 2, ci, co + 9, w + 7, h + 4)
    inp, filt, bias = cx.harness("signed", big)
    want = cx.run(hb, np.ascontiguousarray(inp[n0:n0 + n, y0:y0 + h + 2, x0:x0 + w + 2, :]),
                  np.ascontiguousarray(filt[..., c0:c0 + co]), np.ascontiguousarray(bias[c0:c0 + co]))
    ti, tf, tb = (torch.from_numpy(a).cuda() for a in (inp, filt, bias))
    to_full = torch.full((big[0], big[4], big[3], big[2]), float("nan"), device="cuda")
    to = to_full[n0:n0 + n, y0:y0 + h, x0:x0 + w, c0:c0 + co]
    # buffer coordinates: the larger tensors start at (100, -20, 7, -3) (co, x, y, n); the filter's taps and ci at 0
    o_c, o_x, o_y, o_n = 100, -20, 7, -3
    _torch_call(hb, ti, tf, tb, to, mins=((0, o_x, o_y, o_n), (o_c, 0, 0, 0), (o_c,), (o_c + c0, o_x + x0, o_y + y0, o_n + n0)))
    got = to.cpu().numpy()
    assert _same_bytes(got, want), _mismatch(got, want)
    written = torch.zeros_like(to_full, dtype=torch.bool)
    written[n0:n0 + n, y0:y0 + h, x0:x0 + w, c0:c0 + co] = True
    assert torch.isnan(to_full[~written]).all(), "elements outside the crop were written"


def test_calls_at_other_shapes_in_between_do_not_change_a_result(hb):
    """Scratch and tensor maps are per call: A, B, conv_layer, A again gives A's first result."""
    a, b = (3, 37, 75, 29, 17), (1, 160, 136, 9, 5)
    da, db = cx.harness("signed", a), cx.harness("channel_scales", b)
    first_a, first_b = cx.run(hb, *da), cx.run(hb, *db)
    conv_exact.run(hb, *conv_exact.harness("signed"))
    again_a, again_b = cx.run(hb, *da), cx.run(hb, *db)
    assert _same_bytes(first_a, again_a), _mismatch(first_a, again_a)
    assert _same_bytes(first_b, again_b), _mismatch(first_b, again_b)
