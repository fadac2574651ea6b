"""camera_pipe's per-call tables in the oracle against a float64 evaluation of the generator's formulas.

The GPU tests compare the kernel with the oracle bit for bit, and both restate apps/camera_pipe/camera_pipe_generator.cpp
(:263-271 matrix, :297-332 tone curve, :372 sharpen strength).  A misreading the two share would pass every one of them;
this checks the oracle's tables against the formulas themselves, in float64 with exact pow, from the same float32
inputs.  The float32 pipeline with halide_pow is within one u8 step of that everywhere (the curve is continuous at
g = 0.5), and within one Q8.8 step for the matrix."""
import numpy as np
import pytest

from util import CP_EXTREMES, CP_M3200, CP_M7000, cp_matrix_q88, cp_param_id, cp_params


def curve_f64(gamma, contrast, black, white):
    """Tone curve entries for x in (black, white] (the others are the guards' 0 and 255), evaluated in float64."""
    x = np.arange(1024, dtype=np.float64)
    g32 = np.float64(np.float32(gamma))
    b = 2.0 - 2.0 ** (np.float64(np.float32(contrast)) / 100.0)
    a = 2.0 - 2.0 * b
    out = np.where(x <= black, 0.0, 255.0)
    live = (x > black) & (x <= white)
    xf = np.clip((x[live] - black) / (white - black), 0.0, 1.0)
    g = xf ** (1.0 / g32)
    z = np.where(g > 0.5, 1.0 - (a * (1.0 - g) * (1.0 - g) + b * (1.0 - g)), a * g * g + b * g)
    out[live] = np.trunc(np.clip(z * 255.0 + 0.5, 0.0, 255.0))
    return out, live


@pytest.mark.parametrize("overrides", CP_EXTREMES, ids=cp_param_id)
def test_oracle_tables_follow_the_formulas(oracle, overrides):
    color_temp, gamma, contrast, sharpen, black, white = cp_params(overrides)
    matrix, curve, s32 = oracle.camera_pipe_tables(CP_M3200, CP_M7000, color_temp, gamma, contrast, sharpen, black, white)

    # matrix: within one Q8.8 step of trunc(float64 val * 256), and exactly what the tests' float32 restatement gives
    ct = np.float64(np.float32(color_temp))
    alpha = (1.0 / ct - 1.0 / 3200.0) / (1.0 / 7000.0 - 1.0 / 3200.0)
    val = CP_M3200.astype(np.float64) * alpha + CP_M7000.astype(np.float64) * (1.0 - alpha)
    assert np.abs(matrix.astype(np.int64) - np.trunc(val * 256.0)).max() <= 1
    assert np.array_equal(matrix, cp_matrix_q88(CP_M3200, CP_M7000, color_temp))

    # curve: the guards exactly, the rest within one step
    want, live = curve_f64(gamma, contrast, black, white)
    assert np.array_equal(curve[~live], want[~live])
    assert np.abs(curve[live].astype(np.float64) - want[live]).max(initial=0) <= 1

    # sharpen_strength_x32 = u8_sat(sharpen * 32): exact (the product is exact in float32)
    assert s32 == int(min(255.0, max(0.0, np.trunc(np.float64(np.float32(sharpen)) * 32.0))))


def test_extremes_reach_the_table_branches(oracle):
    """The parameter sets above reach what random frames with the harness's parameters do not: curves that are all
    guard (black >= white), a curve with no 255 guard (white > 1023), z outside [0, 1] before the clamp (contrast 200),
    extrapolated alpha, and sharpen_strength_x32 = 0, 1, 255 exactly and saturated."""
    def tables(**o):
        return oracle.camera_pipe_tables(CP_M3200, CP_M7000, *cp_params(o))

    for b, w in ((500, 500), (600, 400)):
        _, curve, _ = tables(black=b, white=w)
        assert np.array_equal(curve, np.where(np.arange(1024) <= b, 0, 255))
    _, curve, _ = tables(black=25, white=4000)
    assert curve.max() < 255
    x = np.arange(1024, dtype=np.float64)
    g = ((x - 25) / 998).clip(0, 1) ** 0.5
    b = 2.0 - 2.0 ** 2.0
    z = np.where(g > 0.5, 1 - ((2 - 2 * b) * (1 - g) ** 2 + b * (1 - g)), (2 - 2 * b) * g * g + b * g)
    assert z.min() < 0 and z.max() > 1
    for t in (1000.0, 2000.0, 20000.0, 1e5):
        alpha = (1 / t - 1 / 3200) / (1 / 7000 - 1 / 3200)
        assert not 0 <= alpha <= 1
    assert [tables(sharpen=s)[2] for s in (-1.0, 0.03, 1 / 32, 7.96875, 100.0)] == [0, 0, 1, 255, 255]
