"""conv_layer data at the edges of fp32, for any shape (N, CI, CO, W, H), with the generator's result known byte for byte.
Arrays as in conv_any_exact.py: inp [N, H+2, W+2, CI], filt [CI, ky, kx, CO], bias [CO], out [N, H, W, CO].  Every
generator returns (inp, filt, bias, want); want is relu as the generator lowers it, select(conv > 0, conv, 0):
+inf stays +inf, -inf, NaN and -0.0 become +0.0.

  planted    +-inf, a quiet NaN and a NaN whose payload is only in the low 13 bits (which the split's mask turns into
             +inf) in the input, the filter or the bias of dense_exact data, at three targets: the input's top-left
             corner in the first image, its bottom-right corner (x = W+1, y = H+1) in the last image through tap (2, 2)
             and the last channel (in a partial K chunk when CI is not a multiple of 32, in a fold segment after the
             first when CI > 128), and the middle
  overflow   finite powers of two whose products or sums pass FLT_MAX with every term of one sign
  sweep      dense_exact and one_hot scaled by powers of two, from partial sums of 2^127 down to products of 2^-149
  neg_zero   -0.0 in the input, the filter and the bias

want is derived without BLAS wherever a value is not finite (matmul is not reliable on inf * 0): ref64 of the data with
the non-finite values replaced by zeros, plus, for every output a non-finite value reaches, its terms as elementwise
float64 products, whose sum is +inf (+inf terms only), -inf (-inf terms only) or NaN (a NaN operand, inf * 0, or
both signs of inf)."""
import numpy as np

import conv_any_exact as cx
from conv_exact import split

SHAPES = [cx.FIXED, (1, 1, 1, 1, 1), (2, 32, 8, 1, 1), (3, 37, 75, 29, 17), (1, 160, 136, 9, 5), (1, 1024, 64, 6, 6)]

QNAN = np.array(0x7FC00000, np.uint32).view(np.float32)
LOW_NAN = np.array(0x7F800001, np.uint32).view(np.float32)  # hi = x & 0xFFFFE000 is +inf
INF = np.float32(np.inf)
W_EXACT = np.float32(0.75)                # exact in TF32: lo = 0
W_LO = np.float32(0.75 + 2.0 ** -14)      # lo = 2^-14
assert split(W_EXACT)[1] == 0 and split(W_LO)[1] != 0

# name: (where the value goes, the value, its partner at the target (the other operand of its term), the class of the
# target's sum before relu)
PLANTS = {
    "inf_w_exact": ("input", INF, W_EXACT, "+inf"),
    "inf_w_lo": ("input", INF, W_LO, "+inf"),
    "inf_w_zero": ("input", INF, 0.0, "nan"),
    "inf_and_neg_inf": ("input", INF, W_EXACT, "nan"),  # and -inf at another tap of the same output
    "neg_inf": ("input", -INF, W_EXACT, "-inf"),
    "qnan": ("input", QNAN, W_EXACT, "nan"),
    "low_nan": ("input", LOW_NAN, W_EXACT, "nan"),
    "f_inf_x_exact": ("filter", INF, W_EXACT, "+inf"),
    "f_inf_x_lo": ("filter", INF, W_LO, "+inf"),
    "f_inf_x_zero": ("filter", INF, 0.0, "nan"),
    "f_neg_inf": ("filter", -INF, W_EXACT, "-inf"),
    "f_qnan": ("filter", QNAN, W_EXACT, "nan"),
    "f_low_nan": ("filter", LOW_NAN, W_EXACT, "nan"),
    "b_inf": ("bias", INF, None, "+inf"),
    "b_neg_inf": ("bias", -INF, None, "-inf"),
    "b_qnan": ("bias", QNAN, None, "nan"),
    "b_low_nan": ("bias", LOW_NAN, None, "nan"),
}


def targets(shape):
    """[(n, y, x, co, ky, kx, ci)]: an output and the tap and input channel of the term planted for it."""
    n, ci, co, w, h = shape
    return [(0, 0, 0, 0, 0, 0, 0), (n - 1, h - 1, w - 1, co - 1, 2, 2, ci - 1), (n // 2, h // 2, w // 2, co // 2, 1, 1, ci // 2)]


def relu(pre):
    """select(v > 0, v, 0) on float64, to float32 (+0.0 for NaN, -inf and -0.0)."""
    with np.errstate(invalid="ignore"):
        return np.where(pre > 0, pre, 0.0).astype(np.float32)


def pre_relu(inp, filt, bias):
    """The generator's sum before relu (float64), exact on exact data, with the class of every sum a non-finite value
    reaches."""
    nf_in, nf_f, nf_b = (~np.isfinite(a) for a in (inp, filt, bias))
    pre = cx.ref64(np.where(nf_in, 0, inp), np.where(nf_f, 0, filt), np.where(nf_b, 0, bias))
    _, hp, wp, _ = inp.shape
    h, w = hp - 2, wp - 2
    with np.errstate(invalid="ignore", over="ignore"):
        f64 = filt.astype(np.float64)
        for n, yy, xx, c in np.argwhere(nf_in):
            for ky in range(3):
                for kx in range(3):
                    y, x = yy - ky, xx - kx
                    if 0 <= y < h and 0 <= x < w:
                        pre[n, y, x, :] += np.float64(inp[n, yy, xx, c]) * f64[c, ky, kx, :]
        for c, ky, kx, co in np.argwhere(nf_f):
            t = inp[:, ky:ky + h, kx:kx + w, c].astype(np.float64) * f64[c, ky, kx, co]
            t[nf_in[:, ky:ky + h, kx:kx + w, c]] = 0.0  # counted with the input above
            pre[..., co] += t
        pre[..., nf_b] += bias[nf_b].astype(np.float64)
    return pre


def classes(pre):
    """'+inf', '-inf', 'nan' or 'finite' per element."""
    c = np.full(pre.shape, "finite", object)
    c[np.isposinf(pre)], c[np.isneginf(pre)], c[np.isnan(pre)] = "+inf", "-inf", "nan"
    return c


def plant(inp, filt, bias, shape, name):
    """PLANTS[name] at every target, in place.  The planted input channel (filter row, for a value in the filter) is
    zeroed first, so that a partner with lo != 0 meets nothing finite but zeros and every finite sum stays exact."""
    site, value, partner, _ = PLANTS[name]
    for _, _, _, _, _, _, ci in targets(shape):
        if site == "input":
            inp[..., ci] = 0
        elif site == "filter":
            filt[ci] = 0
    for n, y, x, co, ky, kx, ci in targets(shape):
        if site == "bias":
            bias[co] = value
            continue
        if site == "input":
            inp[n, y + ky, x + kx, ci], filt[ci, ky, kx, co] = value, partner
        else:
            filt[ci, ky, kx, co], inp[n, y + ky, x + kx, ci] = value, partner
        if name == "inf_and_neg_inf":
            ky2, kx2 = (0, 0) if (ky, kx) == (1, 1) else (2 - ky, 2 - kx)
            inp[n, y + ky2, x + kx2, ci], filt[ci, ky2, kx2, co] = -INF, W_EXACT


def planted(shape, name, mirrored):
    """PLANTS[name] at the targets of dense_exact data."""
    inp, filt, bias, _ = cx.dense_exact(shape, mirrored)
    plant(inp, filt, bias, shape, name)
    return inp, filt, bias, relu(pre_relu(inp, filt, bias))


def planted_harness(shape):
    """+inf, -inf and both NaNs in the input at the targets of harness-scale signed data, with their partners, and the
    mask of the outputs they reach."""
    inp, filt, bias = cx.harness("signed", shape)
    for t, name in zip(targets(shape), ("inf_w_lo", "qnan", "low_nan")):
        n, y, x, co, ky, kx, ci = t
        inp[n, y + ky, x + kx, ci], filt[ci, ky, kx, co] = PLANTS[name][1], PLANTS[name][2]
    n, y, x, co, ky, kx, ci = targets(shape)[0]
    inp[n, y + 2, x + 1, ci] = -INF
    pre = pre_relu(inp, filt, bias)
    return inp, filt, bias, relu(pre), ~np.isfinite(pre)


# ---- overflow ----------------------------------------------------------------------------------------------------------
OVERFLOWS = ("sum", "neg_sum", "product")
OVER = 2.0 ** 128 - 2.0 ** 103  # FLT_MAX + half an ulp: an exact sum at or above it rounds to inf


def overflow(shape, kind):
    """Zero input and filter, grid bias, and powers of two at the targets: 'sum' and 'neg_sum' give a target four terms
    of +-2^127 (2^64 x 2^63) at the corner taps, 2^129 in all; 'product' one term 2^100 x 2^40.  Every term has the same
    sign and is a power of two, and the bias is below 4: an output holding one term of 2^127 (a neighbour through
    another pair of corner taps) rounds to 2^127 in every order, and one holding two or more terms totals at least
    2^128 - 4 and overflows in every order."""
    in_shape, f_shape, b_shape, _ = cx.shapes_of(shape)
    rng = np.random.default_rng([41, OVERFLOWS.index(kind), *shape])
    inp, filt = np.zeros(in_shape, np.float32), np.zeros(f_shape, np.float32)
    bias = cx._grid(rng, b_shape)
    for n, y, x, co, _, _, ci in targets(shape):
        if kind == "product":
            inp[n, y + 1, x + 1, ci], filt[ci, 1, 1, co] = 2.0 ** 100, 2.0 ** 40
            continue
        for ky, kx in ((0, 0), (0, 2), (2, 0), (2, 2)):
            inp[n, y + ky, x + kx, ci], filt[ci, ky, kx, co] = 2.0 ** 64, (-1 if kind == "neg_sum" else 1) * 2.0 ** 63
    pre = cx.ref64(inp, filt, bias)
    big = np.abs(pre) >= OVER
    pre = np.where(big, np.copysign(np.inf, pre), pre)
    return inp, filt, bias, relu(pre)


# ---- exponent sweep ----------------------------------------------------------------------------------------------------
# (scale of the grid side, scale of the {-1, 0, 1} side) of dense_exact: from partial sums up to 2^127 (2^11 * 2^116)
# down to products of 2^-149 (grid unit 2^-10 * 2^-139), through lo parts (the grid's last bit, 2^(g - 10)) that are
# subnormal from g = -116 on.  No operand goes below 2^-136: the tensor cores read an operand's top 19 bits, which keep
# a subnormal down to 2^-136 and drop the rest.
DENSE_SCALES = [(105, 11), (60, 56), (-60, -60), (-100, -30), (-116, -10), (-126, 0), (-126, -13), (-3, -136)]
# (input scale, filter scale) of one_hot (12-bit operands of 2^-20 .. 2^21): products up to 2^127, down to 2^-149
# (the kernel's result, a*b - lo(a)*lo(b), not the generator's: the oracle does not compute it)
ONE_HOT_SCALES = [(60, 25), (-45, -42)]
SWEEP = [("dense", s, m) for s in DENSE_SCALES for m in (False, True)] + [("one_hot", s, False) for s in ONE_HOT_SCALES]


def _assert_on_grid(*arrays):
    """Finite, and multiples of 2^-149: representable in float32 with nothing lost to the subnormal range."""
    for a in arrays:
        a64 = np.asarray(a, np.float64)
        assert np.isfinite(a64).all()
        assert np.array_equal(np.ldexp(a64, 149), np.round(np.ldexp(a64, 149)))


def sweep(shape, kind, scales, mirrored):
    g, t = scales
    if kind == "dense":
        inp, filt, bias, _ = cx.dense_exact(shape, mirrored)
        si, sf = (t, g) if mirrored else (g, t)
        inp, filt, bias = np.ldexp(inp, si), np.ldexp(filt, sf), np.ldexp(bias, si + sf)
        pre = cx.ref64(inp, filt, bias)
    else:
        inp, filt, bias, _ = cx.one_hot(shape)
        inp, filt = np.ldexp(inp, g), np.ldexp(filt, t)
        # the kernel's sum of one weight's three products: a*b - lo(a)*lo(b)
        pre = cx.ref64(inp, filt, bias) - cx.ref64(split(inp)[1], split(filt)[1], bias * 0)
    inp, filt, bias = (a.astype(np.float32) for a in (inp, filt, bias))
    want = relu(pre)
    assert np.array_equal(want.astype(np.float64), np.where(pre > 0, pre, 0.0)), "the result must be exact in float32"
    assert np.abs(pre).max() <= 2.0 ** 127
    _assert_on_grid(inp, filt, bias, want)
    for a in (inp, filt):
        assert np.array_equal(np.ldexp(a.astype(np.float64), 136), np.round(np.ldexp(a.astype(np.float64), 136)))
    return inp, filt, bias, want


# ---- -0.0 --------------------------------------------------------------------------------------------------------------
def neg_zero(shape, mirrored):
    """dense_exact with half its zeros in the input and the filter made -0.0, output channel 0's filter all -0.0 and
    the bias -0.0 on every other channel: channel 0 sums +-0.0 terms from a -0.0 bias."""
    inp, filt, bias, _ = cx.dense_exact(shape, mirrored)
    rng = np.random.default_rng([51, int(mirrored), *shape])
    for a in (inp, filt):
        a[(a == 0) & (rng.random(a.shape) < 0.5)] = -0.0
    filt[..., 0] = -0.0
    bias[::2] = -0.0
    return inp, filt, bias, relu(cx.ref64(inp, filt, bias))


def datasets(shape):
    """{id: generator call} of every dataset at one shape."""
    d = {f"{name}-{'mirrored' if m else 'direct'}": (lambda name=name, m=m: planted(shape, name, m)) for name in PLANTS for m in (False, True)}
    d.update({f"overflow_{k}": (lambda k=k: overflow(shape, k)) for k in OVERFLOWS})
    d.update({f"sweep_{k}_{s[0]}_{s[1]}{'-mirrored' if m else ''}": (lambda k=k, s=s, m=m: sweep(shape, k, s, m)) for k, s, m in SWEEP})
    d.update({f"neg_zero-{'mirrored' if m else 'direct'}": (lambda m=m: neg_zero(shape, m)) for m in (False, True)})
    return d


DATASET_IDS = list(datasets(cx.FIXED))
