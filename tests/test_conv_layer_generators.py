"""The conv_layer generators of tests/conv_exact.py hold the invariants that make test_conv_layer_exact_gpu.py's
bit-for-bit comparisons sound (CPU only)."""
import numpy as np
import pytest

from conv_exact import CI, CO, GRID, K_STEP, abs_terms, dense_exact, one_hot, ref64, split


@pytest.mark.parametrize("part", [0, 1])
def test_one_hot_operands_are_twelve_bit_and_three_terms_differ_from_the_product(part):
    inp, filt, bias, want, taps = one_hot(part)
    for x in (inp, filt[filt != 0]):
        assert not (x.view(np.uint32) & np.uint32(0xFFF)).any(), "more than 12 significant bits"
        hi, lo = split(x)
        assert np.array_equal(np.abs(lo), np.ldexp(np.float32(1.0), np.frexp(x)[1] - 12).astype(np.float32)), \
            "lo is not the single 12th significant bit"
    assert (filt != 0).sum(axis=(0, 1, 2)).tolist() == [1] * CO and not bias.any()
    product = np.maximum(ref64(inp, filt, bias), 0.0)
    assert (want == 0).mean() < 0.4
    assert (want != product).mean() > 0.5, "the 3-term sum must differ from a*b on most outputs"


def test_one_hot_parts_reach_every_wgmma_slice():
    slots = set()
    for part in (0, 1):
        for ky, kx, ci in one_hot(part)[4]:
            slots.add((((ky * 3 + kx) * (CI // K_STEP) + ci // K_STEP) * 4 + (ci % K_STEP) // 8))
    assert slots == set(range(9 * (CI // K_STEP) * 4))


@pytest.mark.parametrize("mirrored", [False, True])
def test_dense_exact_data_is_exact_and_the_oracle_agrees(oracle, mirrored):
    inp, filt, bias, want = dense_exact(mirrored)
    grid_side, ternary_side = (filt, inp) if mirrored else (inp, filt)
    assert np.array_equal(grid_side / GRID, np.round(grid_side / GRID)) and np.abs(grid_side / GRID).max() < 2 ** 12
    assert set(np.unique(ternary_side).tolist()) == {-1.0, 0.0, 1.0}
    assert 0.4 < (split(grid_side)[1] != 0).mean() < 0.6, "lo should be nonzero on about half the grid values"
    assert (abs_terms(inp, filt) + np.abs(bias.astype(np.float64))).max() <= 2.0 ** 21 * GRID
    assert 0.3 < (want == 0).mean() < 0.7, "a good share of outputs must be negative before relu"
    assert np.array_equal(oracle.conv_layer(inp, filt, bias), want)
