"""Input generators and a float64 reference for conv_layer (fixed shapes: N5 CI128 CO128 100x80, numpy outermost-first:
inp [N, H+2, W+2, CI], filt [CI, ky, kx, CO], bias [CO], out [N, H, W, CO]).

The kernel (halide_b200/csrc/conv_layer_tc.cu) splits each fp32 operand into hi = x & 0xFFFFE000 (11 significant bits,
exact in TF32) and lo = x - hi, and accumulates hi*hi + hi*lo + lo*hi on the tensor cores.  The generators here make
data on which that sum is exact, so the kernel's output is known bit for bit:
  one_hot      one weight per output channel, 12-bit operands: out = max(0, a*b - lo(a)*lo(b)) exactly
  dense_exact  integer multiples of 2^-10 against {-1, 0, 1}: every partial sum is exact in fp32
and data at the harness's scales, for which harness_bound() gives the error the split and the accumulation allow."""
import numpy as np

N, CI, CO, W, H = 5, 128, 128, 100, 80
IN_SHAPE, FILT_SHAPE, OUT_SHAPE = (N, H + 2, W + 2, CI), (CI, 3, 3, CO), (N, H, W, CO)
K_STEP = 32  # input channels per K step of the kernel (one TMA box), 8 per wgmma
GRID = 2.0 ** -10  # the dense_exact grid unit

# Error per output allowed on harness-scale data, as a multiple of sum |a*b| (harness_bound).  Each of the two
# accumulators takes 216 wgmma additions (18 K steps x 4 x 3), each truncating by at most one ulp, 2^-23 of a partial
# sum no larger than sum |a*b|: 216 * 2^-23 = 2^-15.24.  The split loses lo*lo and reads lo with 11 significant bits,
# at most 3 * 2^-20 = 2^-18.4 of |a*b| per product.  Together 2.86e-5, under 2^-15 = 3.05e-5.
E_SPLIT_ACCUM = 2.0 ** -15


def split(x):
    """The kernel's operand split: hi keeps the top 11 significant bits, lo = x - hi (exact in fp32)."""
    x = np.asarray(x, np.float32)
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, x - hi


def ref64(inp, filt, bias):
    """bias + sum_{ky,kx,ci} inp[n, y+ky, x+kx, ci] * filt[ci, ky, kx, co] in float64, before relu: 9 GEMMs, one per tap."""
    x, f = np.asarray(inp, np.float64), np.asarray(filt, np.float64)
    acc = np.empty((N * H * W, CO))
    acc[:] = np.asarray(bias, np.float64)
    for ky in range(3):
        for kx in range(3):
            acc += x[:, ky:ky + H, kx:kx + W, :].reshape(-1, CI) @ f[:, ky, kx, :]
    return acc.reshape(OUT_SHAPE)


def abs_terms(inp, filt):
    """sum |a*b| over the 1152 products of each output (float64)."""
    return ref64(np.abs(inp), np.abs(filt), np.zeros(CO))


def _signs(rng, shape, p_pos):
    return np.where(rng.random(shape) < p_pos, 1.0, -1.0)


def _twelve_bit(rng, shape, p_pos):
    """Odd 12-bit significands (so lo is exactly the last significant bit, never 0) times 2^e, |x| in [2^e, 2^(e+1)),
    e uniform in [-20, 20]."""
    m = 2 * rng.integers(1 << 10, 1 << 11, shape) + 1
    e = rng.integers(-20, 21, shape)
    return (_signs(rng, shape, p_pos) * np.ldexp(m.astype(np.float64), e - 11)).astype(np.float32)


def one_hot(part, seed=11):
    """Each output channel co reads one (ky, kx, ci) with a nonzero weight; bias 0.  Returns (inp, filt, bias, want, taps)
    with taps[co] = (ky, kx, ci) and want = max(0, a*b - lo(a)*lo(b)) exactly.

    The 36 K steps x 4 wgmma slices (8 channels each) are 144 slots; a seeded permutation deals them to the 128 channels,
    part 0 taking slots 0..127 and part 1 slots 128..143 and 0..111, so the two parts reach every slot.  Signs are
    positive with probability 0.8 on both operands, so about two thirds of the products survive relu."""
    rng = np.random.default_rng(seed)
    slots = rng.permutation(144)
    rng = np.random.default_rng([seed, part])
    inp = _twelve_bit(rng, IN_SHAPE, 0.8)
    filt = np.zeros(FILT_SHAPE, np.float32)
    w = _twelve_bit(rng, (CO,), 0.8)
    taps = []
    want = np.empty(OUT_SHAPE, np.float64)
    w_lo = split(w)[1].astype(np.float64)
    for co in range(CO):
        slot = int(slots[(part * CO + co) % 144])
        step, sub = divmod(slot, 4)
        tap, kc = divmod(step, CI // K_STEP)
        ky, kx = divmod(tap, 3)
        ci = kc * K_STEP + 8 * sub + int(rng.integers(0, 8))
        filt[ci, ky, kx, co] = w[co]
        taps.append((ky, kx, ci))
        a = inp[:, ky:ky + H, kx:kx + W, ci]
        three = a.astype(np.float64) * float(w[co]) - split(a)[1].astype(np.float64) * w_lo[co]
        want[..., co] = np.maximum(three, 0.0)
    assert len(set(taps)) == CO
    assert np.array_equal(want.astype(np.float32).astype(np.float64), want), "a*b - lo(a)*lo(b) must be exact in fp32"
    return inp, filt, np.zeros(CO, np.float32), want.astype(np.float32), taps


def _grid(rng, shape):
    """i * 2^-10 with 2^11 <= |i| < 2^12 and a random sign: 12 significant bits, lo nonzero exactly when i is odd."""
    i = rng.integers(1 << 11, 1 << 12, shape) * _signs(rng, shape, 0.5)
    return (i * GRID).astype(np.float32)


def _ternary(rng, shape):
    """{-1, 0, 1} with P(+-1) = 1/8 each."""
    return rng.choice(np.array([-1.0, 0.0, 1.0], np.float32), size=shape, p=[0.125, 0.75, 0.125])


def dense_exact(mirrored, seed=21):
    """Grid values in the input and {-1, 0, 1} in the filter (mirrored: the other way round, so lo is nonzero in the B
    operand instead of the A operand); bias on the grid.  Every product and partial sum is a multiple of 2^-10 no
    larger than 2^21 of them, exact in fp32 in any order, so want = relu of the float64 result.  Signs are symmetric:
    about half the outputs are negative before relu.  Returns (inp, filt, bias, want)."""
    rng = np.random.default_rng([seed, int(mirrored)])
    if mirrored:
        inp, filt = _ternary(rng, IN_SHAPE), _grid(rng, FILT_SHAPE)
    else:
        inp, filt = _grid(rng, IN_SHAPE), _ternary(rng, FILT_SHAPE)
    bias = _grid(rng, (CO,))
    bound = (abs_terms(inp, filt) + np.abs(bias.astype(np.float64))).max()
    assert bound <= 2.0 ** 21 * GRID, bound / GRID
    want = np.maximum(ref64(inp, filt, bias), 0.0)
    assert np.array_equal(want.astype(np.float32).astype(np.float64), want)
    return inp, filt, bias, want.astype(np.float32)


HARNESS_CASES = ("rand", "rand_2^31", "signed", "channel_scales")


def harness(case, seed=31):
    """Data at the scales the reference's harness uses (rand() in [0, 1) and raw rand() up to 2^31), signed data, and
    signed data whose input channels are scaled by 2^s, s uniform in [-24, 24].  Returns (inp, filt, bias)."""
    rng = np.random.default_rng([seed, HARNESS_CASES.index(case)])
    inp, filt, bias = (rng.random(s, dtype=np.float32) for s in (IN_SHAPE, FILT_SHAPE, (CO,)))
    if case == "rand_2^31":
        inp, filt, bias = (a * np.float32(2.0 ** 31) for a in (inp, filt, bias))
    elif case in ("signed", "channel_scales"):
        inp, filt, bias = (a - np.float32(0.5) for a in (inp, filt, bias))
        if case == "channel_scales":
            inp *= np.ldexp(np.float32(1.0), rng.integers(-24, 25, CI)).astype(np.float32)
    return inp, filt, bias


def harness_bound(inp, filt, bias):
    """(relu(float64 result), allowed error per output): E * sum |a*b| for the split and the accumulation plus 2^-24 of
    the result for the fp32 additions of the two accumulators' sum and the bias."""
    r = ref64(inp, filt, bias)
    return np.maximum(r, 0.0), E_SPLIT_ACCUM * abs_terms(inp, filt) + 2.0 ** -24 * np.abs(r)


def run(hb, inp, filt, bias):
    """conv_layer through the C ABI on host buffers.  The output's device allocation is filled with NaN first, so an
    output the kernel does not write reads back as NaN."""
    out = np.full(OUT_SHAPE, np.nan, np.float32)
    bi, bf, bb = hb.HalideBuffer.from_numpy(inp), hb.HalideBuffer.from_numpy(filt), hb.HalideBuffer.from_numpy(bias)
    bo = hb.HalideBuffer.from_numpy(out)
    hb.lib.check(hb.capi.halide_copy_to_device(None, bo.ptr, None))
    hb.filters.conv_layer(bi, bf, bb, bo)
    bo.copy_to_host()
    return out
