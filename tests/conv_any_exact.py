"""conv_exact.py's generators and float64 reference over any shape (N, CI, CO, W, H), for
halide_b200_conv_layer_any_shape.  Arrays are numpy outermost-first as there: inp [N, H+2, W+2, CI], filt [CI, ky, kx, CO],
bias [CO], out [N, H, W, CO].

What changes with the shape in the kernel (halide_b200/csrc/conv_layer_tc.cu): input channels are padded with zeros to a
multiple of 32 (K steps = 9 * ceil(CI / 32)), output channels to the N tile (64 for CO <= 64, else 128), and with more
than 36 K steps the two accumulators are folded into a running fp32 sum every 36 steps, so each accumulator still takes
at most 216 truncating additions and conv_exact.E_SPLIT_ACCUM holds at every CI."""
import numpy as np

from conv_exact import E_SPLIT_ACCUM, GRID, K_STEP, _grid, _signs, _twelve_bit, split

FIXED = (5, 128, 128, 100, 80)
FOLD_STEPS = 36


def shapes_of(shape):
    n, ci, co, w, h = shape
    return (n, h + 2, w + 2, ci), (ci, 3, 3, co), (co,), (n, h, w, co)


def k_steps(ci):
    return 9 * max(1, -(-ci // K_STEP))


def folds(ci):
    """How many times the kernel adds its accumulators into the running sum before the final addition."""
    return -(-k_steps(ci) // FOLD_STEPS) - 1


def n_tile(co):
    return 64 if co <= 64 else 128


def ref64(inp, filt, bias):
    """bias + sum_{ky,kx,ci} inp[n, y+ky, x+kx, ci] * filt[ci, ky, kx, co] in float64, before relu."""
    x, f = np.asarray(inp, np.float64), np.asarray(filt, np.float64)
    n, hp, wp, ci = x.shape
    h, w, co = hp - 2, wp - 2, f.shape[3]
    acc = np.empty((n * h * w, co))
    acc[:] = np.asarray(bias, np.float64)
    for ky in range(3):
        for kx in range(3):
            acc += x[:, ky:ky + h, kx:kx + w, :].reshape(-1, ci) @ f[:, ky, kx, :]
    return acc.reshape(n, h, w, co)


def abs_terms(inp, filt):
    return ref64(np.abs(inp), np.abs(filt), np.zeros(filt.shape[3]))


def one_hot(shape, seed=11):
    """Each output channel reads one (ky, kx, ci) with a nonzero 12-bit weight, bias 0: want = max(0, a*b - lo(a)*lo(b))
    exactly.  The channels walk a seeded permutation of all 9 * CI (tap, ci) pairs, so CO >= 9 * CI reaches every one."""
    n, ci, co, w, h = shape
    in_shape, f_shape, _, out_shape = shapes_of(shape)
    rng = np.random.default_rng([seed, *shape])
    pairs = rng.permutation(9 * ci)
    inp = _twelve_bit(rng, in_shape, 0.8)
    filt = np.zeros(f_shape, np.float32)
    wts = _twelve_bit(rng, (co,), 0.8)
    w_lo = split(wts)[1].astype(np.float64)
    want = np.empty(out_shape, np.float64)
    for c in range(co):
        tap, k = divmod(int(pairs[c % (9 * ci)]), ci)
        ky, kx = divmod(tap, 3)
        filt[k, ky, kx, c] = wts[c]
        a = inp[:, ky:ky + h, kx:kx + w, k]
        want[..., c] = np.maximum(a.astype(np.float64) * float(wts[c]) - split(a)[1].astype(np.float64) * w_lo[c], 0.0)
    assert np.array_equal(want.astype(np.float32).astype(np.float64), want), "a*b - lo(a)*lo(b) must be exact in fp32"
    return inp, filt, np.zeros(co, np.float32), want.astype(np.float32)


def dense_exact(shape, mirrored, seed=21):
    """Grid values (multiples of 2^-10 below 4) against {-1, 0, 1}, mirrored: the other way round; bias on the grid.  The
    ternary side is nonzero in about min(1/4, 288 / (9 CI)) of its entries, which keeps every partial sum below 2^21 grid
    units at any CI: exact in fp32 in any order, through the folds too, so want = relu of the float64 result."""
    n, ci, co, w, h = shape
    in_shape, f_shape, b_shape, _ = shapes_of(shape)
    rng = np.random.default_rng([seed, int(mirrored), *shape])
    p = min(0.125, 144.0 / (9 * ci))

    def ternary(s):
        return rng.choice(np.array([-1.0, 0.0, 1.0], np.float32), size=s, p=[p, 1.0 - 2.0 * p, p])

    if mirrored:
        inp, filt = ternary(in_shape), _grid(rng, f_shape)
    else:
        inp, filt = _grid(rng, in_shape), ternary(f_shape)
    bias = _grid(rng, b_shape)
    bound = (abs_terms(inp, filt) + np.abs(bias.astype(np.float64))).max()
    assert bound <= 2.0 ** 21 * GRID, bound / GRID
    want = np.maximum(ref64(inp, filt, bias), 0.0)
    assert np.array_equal(want.astype(np.float32).astype(np.float64), want)
    return inp, filt, bias, want.astype(np.float32)


CASES = ("rand", "signed", "channel_scales")


def harness(case, shape, seed=31):
    """conv_exact.harness at any shape: rand() in [0, 1), the same minus 0.5, and that with input channels scaled by 2^s,
    s uniform in [-24, 24]."""
    in_shape, f_shape, b_shape, _ = shapes_of(shape)
    rng = np.random.default_rng([seed, CASES.index(case), *shape])
    inp, filt, bias = (rng.random(s, dtype=np.float32) for s in (in_shape, f_shape, b_shape))
    if case != "rand":
        inp, filt, bias = (a - np.float32(0.5) for a in (inp, filt, bias))
        if case == "channel_scales":
            inp *= np.ldexp(np.float32(1.0), rng.integers(-24, 25, shape[1])).astype(np.float32)
    return inp, filt, bias


def harness_bound(inp, filt, bias):
    """(relu(float64 result), allowed error per output): E_SPLIT_ACCUM * sum |a*b| for the split and the accumulators'
    chains, the same constant at every CI, plus 2^-24 of the result for each fp32 addition into the running sum and the
    bias (folds + 1 of them)."""
    r = ref64(inp, filt, bias)
    return np.maximum(r, 0.0), E_SPLIT_ACCUM * abs_terms(inp, filt) + 2.0 ** -24 * np.abs(r) * (folds(inp.shape[3]) + 1)


def worst_ratio(got, inp, filt, bias):
    want, bound = harness_bound(inp, filt, bias)
    return float((np.abs(got.astype(np.float64) - want) / np.maximum(bound, 1e-300)).max())


def run(hb, inp, filt, bias, entry=None):
    """halide_b200_conv_layer_any_shape (or `entry`) through the C ABI on host arrays; the output's device allocation is
    filled with NaN first, so an output the kernel does not write reads back as NaN."""
    n, hp, wp, _ = inp.shape
    out = np.full((n, hp - 2, wp - 2, bias.shape[0]), np.nan, np.float32)
    bi, bf, bb = hb.HalideBuffer.from_numpy(inp), hb.HalideBuffer.from_numpy(filt), hb.HalideBuffer.from_numpy(bias)
    bo = hb.HalideBuffer.from_numpy(out)
    hb.lib.check(hb.capi.halide_copy_to_device(None, bo.ptr, None))
    (entry or hb.filters.conv_layer_any_shape)(bi, bf, bb, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out
