"""The premises of test_conv_layer_edges_gpu.py (CPU only): tests/conv_edge.py's data reach every class of result it is
built for at every shape, the overflow and sweep data keep their margins, and the oracle computes want byte for byte on
every dataset, so the GPU test can compare with want and never run the oracle."""
import numpy as np
import pytest

import conv_any_exact as cx
import conv_edge as ce

SHAPE_IDS = [str(s) for s in ce.SHAPES]


@pytest.mark.parametrize("mirrored", [False, True], ids=["direct", "mirrored"])
@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_every_planted_class_occurs(shape, mirrored):
    """At one target at least, each plant gives its class: +inf alone (against a weight exact in TF32 and one with
    lo != 0, in the input and the filter), +inf with -inf, inf against a zero, NaNs, and an infinite bias."""
    for name, (_, _, _, want_class) in ce.PLANTS.items():
        inp, filt, bias, want = ce.planted(shape, name, mirrored)
        cls = ce.classes(ce.pre_relu(inp, filt, bias))
        at = [cls[n, y, x, co] for n, y, x, co, *_ in ce.targets(shape)]
        assert want_class in at, (name, at)
        if want_class == "+inf":
            assert np.isposinf(want).any()
        assert not np.isnan(want).any() and not np.signbit(want).any()


@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_overflow_margins(shape):
    for kind in ce.OVERFLOWS:
        inp, filt, bias, want = ce.overflow(shape, kind)
        pre = cx.ref64(inp, filt, bias)
        terms = cx.ref64(np.abs(inp), np.abs(filt), np.zeros_like(bias))
        assert np.array_equal(np.abs(cx.ref64(inp, filt, 0 * bias)), terms), "every term of one sign"
        assert np.abs(bias).max() < 4
        assert ((np.abs(pre) <= 2.0 ** 127 + 4) | (np.abs(pre) >= 2.0 ** 128 - 4)).all(), "no sum near FLT_MAX"
        at = np.array([pre[n, y, x, co] for n, y, x, co, *_ in ce.targets(shape)])
        assert (np.abs(at) >= (2.0 ** 140 if kind == "product" else 2.0 ** 129)).all()
        assert (np.isinf(want) == (pre >= ce.OVER)).all() and np.isposinf(want).any() == (kind != "neg_sum")
        finite_big = np.isfinite(want) & (np.abs(pre) >= 2.0 ** 120)
        if min(shape[3], shape[4]) >= 3 and kind != "product":  # room for a neighbour through other corner taps
            assert finite_big.any(), "a neighbour of 2^127 must stay finite"


@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_sweep_reaches_both_ends(shape):
    """The generators assert exactness and the 2^-149 grid; here: the top scale has sums above 2^115, the bottom ones
    subnormal lo parts and subnormal sums."""
    tops, lows, lo_sub, sub_products = [], [], False, False
    for kind, scales, mirrored in ce.SWEEP:
        inp, filt, bias, _ = ce.sweep(shape, kind, scales, mirrored)
        pre = cx.ref64(inp, filt, bias)
        nz = pre[pre != 0]
        if nz.size:
            tops.append(np.abs(nz).max())
            lows.append(np.abs(nz).min())
        for a in (inp, filt):
            lo = np.abs(ce.split(a)[1])
            lo_sub |= bool(((lo > 0) & (lo < 2.0 ** -126)).any())
        sub_products |= bool(((np.abs(nz) > 0) & (np.abs(nz) < 2.0 ** -126)).any())
    assert max(tops) >= 2.0 ** 115 and min(lows) < 2.0 ** -126
    assert lo_sub and sub_products


@pytest.mark.parametrize("dataset", [d for d in ce.DATASET_IDS if "one_hot" not in d])
@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_oracle_equals_want(oracle, shape, dataset):
    """one_hot's want is the kernel's three products, not the generator's sum, and is left out."""
    inp, filt, bias, want = ce.datasets(shape)[dataset]()
    got = oracle.conv_layer(inp, filt, bias)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got.view(np.uint32) != want.view(np.uint32)).sum())


@pytest.mark.parametrize("shape", ce.SHAPES, ids=SHAPE_IDS)
def test_planted_harness_reaches_few_outputs(oracle, shape):
    inp, filt, bias, want, touched = ce.planted_harness(shape)
    assert touched.any() and (not touched.all() or min(shape[3], shape[4]) < 3)
    got = oracle.conv_layer(inp, filt, bias)
    assert np.array_equal(got[touched].view(np.uint32), want[touched].view(np.uint32))
