"""Second, independently structured restatement of the pipelines in numpy — TEST INFRASTRUCTURE ONLY.

oracle/*.cpp evaluates the generators pixel by pixel through memoised recursive lambdas; this file evaluates the same
Func definitions as whole-array float32 numpy expressions over explicitly inferred index ranges (the way Halide's
bounds inference would size them).  Neither is the reference (which cannot be built here, SURVEY.md §8c), but two
restatements written differently that agree bit for bit make a mis-transcribed formula, tap or rounding order in the
oracle much less likely.  tests/test_oracle_crosscheck.py compares them.

Follows: apps/local_laplacian/local_laplacian_generator.cpp:19-87 (algorithm), :262-282 (downsample / upsample);
src/IROperator.cpp:921-966 + :33-62 (halide_exp, evaluate_polynomial); src/Lerp.cpp:126-128 (lerp);
apps/stencil_chain/stencil_chain_generator.cpp:17-30; the other generators are cited at their functions.  Halide semantics used: Euclidean integer / and %, float
x / const -> x * fold(1/const), no FMA contraction, lerp(z, o, w) = z*(1-w) + o*w, clamp = max(min(a, hi), lo).
"""
import numpy as np

F = np.float32


class Field:
    """A Func realised on the box x in [x0, x0+nx), y in [y0, y0+ny): arr[y - y0, x - x0(, k)]."""

    def __init__(self, arr, x0, y0):
        self.arr, self.x0, self.y0 = arr, x0, y0

    def at(self, xs, ys):
        xi, yi = np.asarray(xs) - self.x0, np.asarray(ys) - self.y0
        assert xi.min() >= 0 and yi.min() >= 0 and xi.max() < self.arr.shape[1] and yi.max() < self.arr.shape[0], "read outside the realised box"
        return self.arr[yi[:, None], xi[None, :]]


def halide_exp(x_full):
    x_full = x_full.astype(F)
    ln2_part1, ln2_part2 = F(0.6931457519), F(1.4286067653e-6)
    one_over_ln2 = F(1.0) / np.log(F(2.0), dtype=F)
    scaled = x_full * one_over_ln2
    k_real = np.floor(scaled)
    k = k_real.astype(np.int32)
    x = x_full - k_real * ln2_part1
    x = x - k_real * ln2_part2
    c = [F(v) for v in (0.00031965933071842413, 0.00119156835564003744, 0.00848988645943932717, 0.04160188091348320655,
                        0.16667983794100929562, 0.49999899033463041098, 1.0, 1.0)]
    x2 = x * x
    even, odd = c[0], c[1]
    for i in range(2, 8):
        if i & 1:
            odd = odd * x2 + c[i]
        else:
            even = even * x2 + c[i]
    result = even * x + odd
    biased = k + 127
    two_to_the_n = (np.clip(biased, 0, 255).astype(np.uint32) << np.uint32(23)).view(F)
    result = result * two_to_the_n
    result = np.where(biased < 255, result, F(np.inf))
    return np.where(biased > 0, result, F(0)).astype(F)


def _down(f, xlo, xhi, ylo, yhi):
    """downsample(f) on [xlo, xhi] x [ylo, yhi]: 1-3-3-1 in y, then in x (generator :266-272)."""
    xs_wide = np.arange(2 * xlo - 1, 2 * xhi + 3)
    ys = np.arange(ylo, yhi + 1)
    downy = _down4(f.at(xs_wide, 2 * ys - 1), f.at(xs_wide, 2 * ys), f.at(xs_wide, 2 * ys + 1), f.at(xs_wide, 2 * ys + 2))
    dy = Field(downy, 2 * xlo - 1, ylo)
    xs = np.arange(xlo, xhi + 1)
    downx = _down4(dy.at(2 * xs - 1, ys), dy.at(2 * xs, ys), dy.at(2 * xs + 1, ys), dy.at(2 * xs + 2, ys))
    return Field(downx.astype(F), xlo, ylo)


def _down4(a, b, c, d):
    """(f(2x-1) + 3 * (f(2x) + f(2x+1)) + f(2x+2)) / 8, summed left to right; / 8 folds to * 0.125."""
    return (a + F(3.0) * (b + c) + d) * F(0.125)


def _lerp(zero, one, w):
    return zero * (F(1.0) - w) + one * w


def _up(f, xlo, xhi, ylo, yhi):
    """upsample(f) on [xlo, xhi] x [ylo, yhi]: bilinear, x then y (generator :275-282); integer / and % are Euclidean."""
    xs, ys = np.arange(xlo, xhi + 1), np.arange(ylo, yhi + 1)
    cy = np.arange((ylo - 1) >> 1, ((yhi + 1) >> 1) + 1)  # coarse rows upy reads
    wx = (((xs & 1) * 2 + 1).astype(F) * F(0.25))
    wx = wx[None, :] if f.arr.ndim == 2 else wx[None, :, None]
    upx = Field(_lerp(f.at((xs + 1) >> 1, cy), f.at((xs - 1) >> 1, cy), wx).astype(F), xlo, cy[0])
    wy = (((ys & 1) * 2 + 1).astype(F) * F(0.25))
    wy = wy[:, None] if f.arr.ndim == 2 else wy[:, None, None]
    upy = _lerp(upx.at(xs, (ys + 1) >> 1), upx.at(xs, (ys - 1) >> 1), wy)
    return Field(upy.astype(F), xlo, ylo)


def local_laplacian(inp, levels, alpha, beta, out_shape=None, in_mins=(0, 0, 0), out_mins=(0, 0, 0), J=8):
    """inp: uint16 [c, h, w] whose element [0, 0, 0] sits at coordinates in_mins = (x, y, c); alpha as the filter
    receives it (already divided by levels - 1).  Returns uint16 [C, H, W] at out_mins."""
    return clamp_u16(local_laplacian_color(inp, levels, alpha, beta, out_shape, in_mins, out_mins, J))


def clamp_u16(color):
    """u16(clamp(color, 0, 65535)) (generator :87).  Halide's min and max select on a comparison, which is false for NaN:
    min(NaN, 65535) = 65535, then max(65535, 0) = 65535.  (np.minimum / np.maximum would pass the NaN on to the cast.)"""
    m = np.where(color < F(65535.0), color, F(65535.0))
    return np.where(m > F(0.0), m, F(0.0)).astype(np.uint16)


def local_laplacian_color(inp, levels, alpha, beta, out_shape=None, in_mins=(0, 0, 0), out_mins=(0, 0, 0), J=8):
    """local_laplacian's colour before the final clamp and cast: float32 [C, H, W].  Every float alpha and beta is
    accepted; large ones overflow the pyramid's sums to infinities and NaN, as they do in Halide."""
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        return _color(inp, levels, F(alpha), F(beta), out_shape, in_mins, out_mins, J)


def _color(inp, levels, alpha, beta, out_shape, in_mins, out_mins, J):
    ic, ih, iw = inp.shape
    if out_shape is None:
        out_shape = inp.shape
    C, H, W = out_shape
    ix0, iy0, ic0 = in_mins
    ox0, oy0, oc0 = out_mins
    # --- bounds: O_j = box of outGPyramid[j] / lPyramid[j]; G_j = box of gPyramid[j] / inGPyramid[j] -------------------
    O = [(ox0, ox0 + W - 1, oy0, oy0 + H - 1)]
    for j in range(1, J):
        xl, xh, yl, yh = O[j - 1]
        O.append(((xl - 1) >> 1, (xh + 1) >> 1, (yl - 1) >> 1, (yh + 1) >> 1))
    G = [None] * J
    G[J - 1] = O[J - 1]
    for j in range(J - 2, -1, -1):
        xl, xh, yl, yh = G[j + 1]
        d = (2 * xl - 1, 2 * xh + 2, 2 * yl - 1, 2 * yh + 2)
        G[j] = (min(O[j][0], d[0]), max(O[j][1], d[1]), min(O[j][2], d[2]), max(O[j][3], d[3]))
    # --- remap LUT on every index it can be asked for ----------------------------------------------------------------
    lm1 = levels - 1
    lut_x = np.arange(-256 * lm1, 256 * lm1 + 1)
    fx = lut_x.astype(F) * F(1.0 / 256.0)
    lut = (alpha * fx) * halide_exp((-fx * fx) * F(0.5))
    # --- gray on G_0 from the edge-clamped input -----------------------------------------------------------------------
    gx = np.arange(G[0][0], G[0][1] + 1)
    gy = np.arange(G[0][2], G[0][3] + 1)
    cx = np.clip(gx, ix0, ix0 + iw - 1) - ix0
    cy = np.clip(gy, iy0, iy0 + ih - 1) - iy0
    inv65535 = F(1.0 / 65535.0)

    def floating(c):
        cc = min(max(c, ic0), ic0 + ic - 1) - ic0
        return inp[cc][cy[:, None], cx[None, :]].astype(F) * inv65535

    gray = F(0.299) * floating(0) + F(0.587) * floating(1) + F(0.114) * floating(2)
    # --- gPyramid[0] on G_0 ------------------------------------------------------------------------------------------------
    flm1 = F(lm1)
    inv_lm1 = F(1.0) / flm1
    idx = np.clip(((gray * flm1) * F(256.0)).astype(np.int32), 0, lm1 * 256)
    ks = np.arange(levels)
    level = ks.astype(F) * inv_lm1
    g0 = beta * (gray[:, :, None] - level[None, None, :]) + level[None, None, :]
    g0 = g0 + lut[(idx[:, :, None] - 256 * ks[None, None, :]) + 256 * lm1]
    gP = [Field(g0.astype(F), G[0][0], G[0][2])]
    inG = [Field(gray.astype(F), G[0][0], G[0][2])]
    for j in range(1, J):
        gP.append(_down(gP[j - 1], *G[j]))
        inG.append(_down(inG[j - 1], *G[j]))
    # --- Laplacian pyramid of the processed stack, output pyramids ---------------------------------------------------------
    outG = [None] * J
    for j in range(J - 1, -1, -1):
        xl, xh, yl, yh = O[j]
        xs, ys = np.arange(xl, xh + 1), np.arange(yl, yh + 1)
        lP = gP[j].at(xs, ys) if j == J - 1 else gP[j].at(xs, ys) - _up(gP[j + 1], xl, xh, yl, yh).arr
        lev = inG[j].at(xs, ys) * flm1
        li = np.clip(lev.astype(np.int32), 0, levels - 2)
        lf = lev - li.astype(F)
        yy, xx = np.meshgrid(np.arange(len(ys)), np.arange(len(xs)), indexing="ij")
        outL = (F(1.0) - lf) * lP[yy, xx, li] + lf * lP[yy, xx, li + 1]
        if j == J - 1:
            outG[j] = Field(outL.astype(F), xl, yl)
        else:
            outG[j] = Field((_up(outG[j + 1], xl, xh, yl, yh).arr + outL).astype(F), xl, yl)
    # --- colour ---------------------------------------------------------------------------------------------------------------
    eps = F(0.01)
    xs, ys = np.arange(ox0, ox0 + W), np.arange(oy0, oy0 + H)
    g_out = inG[0].at(xs, ys)
    num = outG[0].arr + eps
    den = g_out + eps
    out = np.empty((C, H, W), F)
    for c in range(C):
        ch = inp[oc0 + c - ic0][(ys - iy0)[:, None], (xs - ix0)[None, :]].astype(F)  # unclamped read: must be inside the input
        out[c] = (ch * num) / den
    return out


def stencil_chain(inp, out_shape=None, in_mins=(0, 0), out_mins=(0, 0), stencils=32):
    """inp: uint16 [h, w] at in_mins = (x, y).  32 chained 5x5 stencils, weight (i+3)(j+3), all in uint16 (wraps);
    only the input is edge-clamped, every stage is evaluated on the region the next one reads."""
    ih, iw = inp.shape
    if out_shape is None:
        out_shape = inp.shape
    H, W = out_shape
    ix0, iy0 = in_mins
    ox0, oy0 = out_mins
    r = 2 * stencils
    xs = np.arange(ox0 - r, ox0 + W + r)
    ys = np.arange(oy0 - r, oy0 + H + r)
    cur = inp[(np.clip(ys, iy0, iy0 + ih - 1) - iy0)[:, None], (np.clip(xs, ix0, ix0 + iw - 1) - ix0)[None, :]].astype(np.uint16)
    for _ in range(stencils):
        h, w = cur.shape
        acc = np.zeros((h - 4, w - 4), np.uint16)
        for i in range(-2, 3):        # x offset, outer
            for j in range(-2, 3):    # y offset, inner
                acc = acc + np.uint16((i + 3) * (j + 3)) * cur[2 + j:h - 2 + j, 2 + i:w - 2 + i]
        cur = acc
    return cur


def _clamped2(inp, mins, xs, ys):
    """repeat_edge(input)(xs, ys) for a 2-D array at mins = (x, y): outer product of row / column index vectors."""
    h, w = inp.shape
    return inp[(np.clip(ys, mins[1], mins[1] + h - 1) - mins[1])[:, None], (np.clip(xs, mins[0], mins[0] + w - 1) - mins[0])[None, :]]


def bilateral_grid(inp, r_sigma, out_shape=None, in_mins=(0, 0), out_mins=(0, 0), s_sigma=8):
    """apps/bilateral_grid/bilateral_grid_generator.cpp:17-67.  inp: float32 [h, w] at in_mins = (x, y)."""
    inp = inp.astype(F)
    if out_shape is None:
        out_shape = inp.shape
    H, W = out_shape
    ox0, oy0 = out_mins
    s = s_sigma
    inv_r = F(1.0) / F(r_sigma)
    xs, ys = np.arange(ox0, ox0 + W), np.arange(oy0, oy0 + H)
    # cells read by the slice: xi .. xi+1, yi .. yi+1; the blurs widen that by 2 cells per axis
    cx_lo, cx_hi = (ox0 // s) - 2, ((ox0 + W - 1) // s) + 1 + 2
    cy_lo, cy_hi = (oy0 // s) - 2, ((oy0 + H - 1) // s) + 1 + 2
    z_lo, z_hi = -4, int(np.floor(float(inv_r))) + 6  # generous: bins that are never hit stay 0
    ncx, ncy, nz = cx_hi - cx_lo + 1, cy_hi - cy_lo + 1, z_hi - z_lo + 1
    hist = np.zeros((ncy, ncx, nz, 2), F)
    cys, cxs = np.arange(cy_lo, cy_hi + 1), np.arange(cx_lo, cx_hi + 1)
    yy, xx = np.meshgrid(np.arange(ncy), np.arange(ncx), indexing="ij")
    for ry in range(s):          # RDom r(0, s, 0, s): r.x is the inner loop
        for rx in range(s):
            val = _clamped2(inp, in_mins, cxs * s + rx - s // 2, cys * s + ry - s // 2)
            val = np.maximum(np.minimum(val, F(1.0)), F(0.0))
            zi = (val * inv_r + F(0.5)).astype(np.int32)
            hist[yy, xx, zi - z_lo, 0] += val
            hist[yy, xx, zi - z_lo, 1] += F(1.0)

    def blur5(a, axis):
        n = a.shape[axis]

        def sl(o):
            idx = [slice(None)] * a.ndim
            idx[axis] = slice(2 + o, n - 2 + o)
            return a[tuple(idx)]
        return (((sl(-2) + sl(-1) * F(4)) + sl(0) * F(6)) + sl(1) * F(4)) + sl(2)

    blurz = blur5(hist, 2)        # z range shrinks by 2 at each end
    blurx = blur5(blurz, 1)
    blury = blur5(blurx, 0)       # now cells [cx_lo+2, cx_hi-2] x [cy_lo+2, cy_hi-2], z [z_lo+2, z_hi-2]
    bx0, by0, bz0 = cx_lo + 2, cy_lo + 2, z_lo + 2
    val = inp[(ys - in_mins[1])[:, None], (xs - in_mins[0])[None, :]]  # unclamped read: must lie inside the input
    val = np.maximum(np.minimum(val, F(1.0)), F(0.0))
    zv = val * inv_r
    zi = zv.astype(np.int32)
    zf = zv - zi.astype(F)
    xf = ((xs % s).astype(F) * F(1.0 / s))[None, :]
    yf = ((ys % s).astype(F) * F(1.0 / s))[:, None]
    xi = (xs // s - bx0)[None, :] + np.zeros((H, 1), np.int64)
    yi = (ys // s - by0)[:, None] + np.zeros((1, W), np.int64)

    def g(dx, dy, dz, c):
        return blury[yi + dy, xi + dx, zi - bz0 + dz, c]

    def interp(c):
        return _lerp(_lerp(_lerp(g(0, 0, 0, c), g(1, 0, 0, c), xf), _lerp(g(0, 1, 0, c), g(1, 1, 0, c), xf), yf),
                     _lerp(_lerp(g(0, 0, 1, c), g(1, 0, 1, c), xf), _lerp(g(0, 1, 1, c), g(1, 1, 1, c), xf), yf), zf)

    return (interp(0) / interp(1)).astype(F)


def fast_exp(x_full):
    """src/IROperator.cpp:1616-1643."""
    x_full = x_full.astype(F)
    ln2 = np.log(F(2.0), dtype=F)                 # logf(2.0)
    scaled = x_full * F(1.0 / float(ln2))         # x / const -> x * fold(1 / const), folded in double
    k_real = np.floor(scaled)
    k = k_real.astype(np.int32)
    x = x_full - k_real * ln2
    c = [F(v) for v in (0.01314350012789660196, 0.03668965196652099192, 0.16873890085469545053, 0.49970514590562437052, 1.0, 1.0)]
    x2 = x * x
    even, odd = c[0], c[1]
    for i in range(2, 6):
        if i & 1:
            odd = odd * x2 + c[i]
        else:
            even = even * x2 + c[i]
    result = even * x + odd
    biased = np.clip(k + 127, 0, 255)
    return (result * (biased.astype(np.uint32) << np.uint32(23)).view(F)).astype(F)


def nl_means(inp, patch_size, search_area, sigma, out_shape=None, in_mins=(0, 0, 0), out_mins=(0, 0, 0)):
    """apps/nl_means/nl_means_generator.cpp:17-63.  inp: float32 [c, h, w] at in_mins = (x, y, c); output has 3 channels."""
    inp = inp.astype(F)
    ic, ih, iw = inp.shape
    if out_shape is None:
        out_shape = (3, ih, iw)
    _, H, W = out_shape
    ix0, iy0, ic0 = in_mins
    ox0, oy0, _ = out_mins
    sg, p, sa = F(sigma), patch_size, search_area
    inv_sigma_sq = F(-1.0) / (((sg * sg) * F(p)) * F(p))
    hp = p // 2

    def clamped(c, xs, ys):
        cc = min(max(c, ic0), ic0 + ic - 1) - ic0
        return _clamped2(inp[cc], (ix0, iy0), xs, ys)

    xs, ys = np.arange(ox0, ox0 + W), np.arange(oy0, oy0 + H)
    xs_w = np.arange(ox0 - hp, ox0 + W - hp + p - 1 + 1)     # x range blur_d reads of blur_d_y
    ys_w = np.arange(oy0 - hp, oy0 + H - hp + p - 1 + 1)     # y range blur_d_y reads of d
    acc = np.zeros((4, H, W), F)
    for sy in range(-(sa // 2), -(sa // 2) + sa):             # s_dom.y outer, s_dom.x inner
        for sx in range(-(sa // 2), -(sa // 2) + sa):
            d = np.zeros((len(ys_w), len(xs_w)), F)
            for c in range(3):
                t = clamped(c, xs_w, ys_w) - clamped(c, xs_w + sx, ys_w + sy)
                d = d + t * t
            blur_d_y = np.zeros((H, len(xs_w)), F)
            for r in range(p):
                blur_d_y = blur_d_y + d[r:r + H, :]
            blur_d = np.zeros((H, W), F)
            for r in range(p):
                blur_d = blur_d + blur_d_y[:, r:r + W]
            w = fast_exp(blur_d * inv_sigma_sq)
            for c in range(3):
                acc[c] = acc[c] + w * clamped(c, xs + sx, ys + sy)
            acc[3] = acc[3] + w * F(1.0)
    out = acc[:3] / acc[3][None]
    return np.maximum(np.minimum(out, F(1.0)), F(0.0)).astype(F)


# ---- camera_pipe (apps/camera_pipe/camera_pipe_generator.cpp:16-35, 37-152, 240-425) -------------------------------------
# Every Func is a Python function of integer index grids (X, Y broadcast to one shape), evaluated by plain recursion
# with no memoisation — slow, but there is no region bookkeeping to get wrong; small frames only.

def halide_log(x_full):
    """src/IROperator.cpp:845-919."""
    x_full = np.asarray(x_full, F)
    use_nan, use_neg_inf = x_full < 0, x_full == 0
    patched = np.where(use_nan | use_neg_inf, F(1.0), x_full).astype(F)
    iv = patched.view(np.int32)
    no_exp = iv & np.int32(-2139095041)          # 0x807fffff
    new_e = no_exp >> 22
    new_biased = 127 - new_e
    exponent = (iv >> 23) - new_biased
    reduced = (no_exp | (new_biased << 23)).astype(np.int32).view(F)
    c = [F(v) for v in (0.05111976432738144643, -0.11793923497136414580, 0.14971993724699017569, -0.16862004708254804686,
                        0.19980668101718729313, -0.24991211576292837737, 0.33333435275479328386, -0.50000106292873236491,
                        1.0, 0.0)]
    x1 = reduced - F(1.0)
    x2 = x1 * x1
    even, odd = c[0], c[1]
    for i in range(2, 10):
        if i & 1:
            odd = odd * x2 if c[i] == 0 else odd * x2 + c[i]
        else:
            even = even * x2 if c[i] == 0 else even * x2 + c[i]
    result = even * x1 + odd
    result = result + exponent.astype(F) * np.log(F(2.0), dtype=F)
    return np.where(use_nan, F(np.nan), np.where(use_neg_inf, F(-np.inf), result)).astype(F)


def halide_pow(x, y):
    """pow_f32 lowering, src/CodeGen_LLVM.cpp:3925-3942 (only the branches x >= 0 can reach here)."""
    x, y = np.asarray(x, F), np.asarray(y, F)
    with np.errstate(all="ignore"):
        p = halide_exp(halide_log(np.abs(x)) * y)
    return np.where(x > 0, p, np.where(y == 0, F(1.0), F(0.0))).astype(F)


def camera_pipe(raw, m3200, m7000, color_temp, gamma, contrast, sharpen_strength, black, white, out_shape, in_mins=(0, 0),
                out_mins=(0, 0, 0)):
    """raw: uint16 [h, w] at in_mins = (x, y); returns uint8 [3, H, W] at out_mins = (x, y, c)."""
    u16, i16, i32, u32, u8 = np.uint16, np.int16, np.int32, np.uint32, np.uint8
    C, H, W = out_shape

    def inp(X, Y):  # unclamped: the caller supplies the region the pipeline reads
        xi, yi = X - in_mins[0], Y - in_mins[1]
        assert xi.min() >= 0 and yi.min() >= 0 and xi.max() < raw.shape[1] and yi.max() < raw.shape[0], "raw read out of bounds"
        return raw[yi, xi]

    def shifted(X, Y):
        return inp(X + 16, Y + 12)

    def denoised(X, Y):
        a = np.maximum(np.maximum(shifted(X - 2, Y), shifted(X + 2, Y)), np.maximum(shifted(X, Y - 2), shifted(X, Y + 2)))
        return np.maximum(np.minimum(shifted(X, Y), a), u16(0))

    def deint(X, Y, c):
        return denoised(2 * X + (c & 1), 2 * Y + (c >> 1))

    def avg(a, b):  # (widen(a) + b + 1) / 2, narrowed back
        wide = {u16: u32, u8: u16}[a.dtype.type]
        return ((a.astype(wide) + b.astype(wide) + wide(1)) // wide(2)).astype(a.dtype)

    def absd(a, b):
        return np.where(a > b, a - b, b - a).astype(a.dtype)

    g_gr = lambda X, Y: deint(X, Y, 0)
    r_r = lambda X, Y: deint(X, Y, 1)
    b_b = lambda X, Y: deint(X, Y, 2)
    g_gb = lambda X, Y: deint(X, Y, 3)

    def g_r(X, Y):
        gv, gvd = avg(g_gb(X, Y - 1), g_gb(X, Y)), absd(g_gb(X, Y - 1), g_gb(X, Y))
        gh, ghd = avg(g_gr(X + 1, Y), g_gr(X, Y)), absd(g_gr(X + 1, Y), g_gr(X, Y))
        return np.where(ghd < gvd, gh, gv)

    def g_b(X, Y):
        gv, gvd = avg(g_gr(X, Y + 1), g_gr(X, Y)), absd(g_gr(X, Y + 1), g_gr(X, Y))
        gh, ghd = avg(g_gb(X - 1, Y), g_gb(X, Y)), absd(g_gb(X - 1, Y), g_gb(X, Y))
        return np.where(ghd < gvd, gh, gv)

    # uint16 arithmetic wraps (numpy does the same for same-typed arrays)
    def r_gr(X, Y):
        return (g_gr(X, Y) - avg(g_r(X, Y), g_r(X - 1, Y))) + avg(r_r(X - 1, Y), r_r(X, Y))

    def b_gr(X, Y):
        return (g_gr(X, Y) - avg(g_b(X, Y), g_b(X, Y - 1))) + avg(b_b(X, Y), b_b(X, Y - 1))

    def r_gb(X, Y):
        return (g_gb(X, Y) - avg(g_r(X, Y), g_r(X, Y + 1))) + avg(r_r(X, Y), r_r(X, Y + 1))

    def b_gb(X, Y):
        return (g_gb(X, Y) - avg(g_b(X, Y), g_b(X + 1, Y))) + avg(b_b(X, Y), b_b(X + 1, Y))

    def r_b(X, Y):
        rp = (g_b(X, Y) - avg(g_r(X, Y), g_r(X - 1, Y + 1))) + avg(r_r(X, Y), r_r(X - 1, Y + 1))
        rpd = absd(r_r(X, Y), r_r(X - 1, Y + 1))
        rn = (g_b(X, Y) - avg(g_r(X - 1, Y), g_r(X, Y + 1))) + avg(r_r(X - 1, Y), r_r(X, Y + 1))
        rnd = absd(r_r(X - 1, Y), r_r(X, Y + 1))
        return np.where(rpd < rnd, rp, rn)

    def b_r(X, Y):
        bp = (g_r(X, Y) - avg(g_b(X, Y), g_b(X + 1, Y - 1))) + avg(b_b(X, Y), b_b(X + 1, Y - 1))
        bpd = absd(b_b(X, Y), b_b(X + 1, Y - 1))
        bn = (g_r(X, Y) - avg(g_b(X + 1, Y), g_b(X, Y - 1))) + avg(b_b(X + 1, Y), b_b(X, Y - 1))
        bnd = absd(b_b(X + 1, Y), b_b(X, Y - 1))
        return np.where(bpd < bnd, bp, bn)

    def interleave(f00, f10, f01, f11):  # interleave_y(interleave_x(f00, f10), interleave_x(f01, f11)); Euclidean / and %
        def out(X, Y):
            hx, hy = X >> 1, Y >> 1
            top = np.where((X & 1) == 0, f00(hx, hy), f10(hx, hy))
            bot = np.where((X & 1) == 0, f01(hx, hy), f11(hx, hy))
            return np.where((Y & 1) == 0, top, bot)
        return out

    demosaiced = [interleave(r_gr, r_r, r_b, r_gb), interleave(g_gr, g_r, g_b, g_gb), interleave(b_gr, b_r, b_b, b_gb)]

    # colour matrix, Q8.8
    kelvin = F(color_temp)
    alpha = (F(1.0) / kelvin - F(1.0) / F(3200)) / (F(1.0) / F(7000) - F(1.0) / F(3200))
    val = m3200.astype(F) * alpha + m7000.astype(F) * (F(1.0) - alpha)
    matrix = (val * F(256.0)).astype(i16)        # [row y][col x]; matrix(x, y) in the generator

    def corrected(X, Y, c):
        ir, ig, ib = (demosaiced[k](X, Y).astype(u16).view(i16).astype(i32) for k in range(3))
        m = matrix.astype(i32)
        v = m[c, 3] + m[c, 0] * ir + m[c, 1] * ig + m[c, 2] * ib
        return (v >> 8).astype(i16)              # Euclidean / 256, then wrap to int16

    # tone curve LUT on [0, 1023]
    xs = np.arange(1024, dtype=i32)
    min_raw, max_raw = i32(black), i32(white)
    inv_range = F(1.0) / F(max_raw - min_raw)
    bq = F(2.0) - halide_pow(F(2.0), F(contrast) * F(0.01))
    aq = F(2.0) - F(2.0) * bq
    xf = np.maximum(np.minimum((xs - min_raw).astype(F) * inv_range, F(1.0)), F(0.0))
    g = halide_pow(xf, F(1.0) / F(gamma))
    omg = F(1.0) - g
    z = np.where(g > F(0.5), F(1.0) - ((aq * omg) * omg + bq * omg), (aq * g) * g + bq * g).astype(F)
    cval = np.maximum(np.minimum(z * F(255.0) + F(0.5), F(255.0)), F(0.0)).astype(u8)
    curve = np.where(xs <= min_raw, u8(0), np.where(xs > max_raw, u8(255), cval)).astype(u8)

    def curved(X, Y, c):
        return curve[np.clip(corrected(X, Y, c), 0, 1023)]

    sv = F(sharpen_strength) * F(32)
    strength = u8(255) if sv >= F(255.0) else u8(max(sv, F(0.0)))      # u8_sat of a float

    def blur121(a, b, c):
        return avg(avg(a, c), b)

    def unsharp_y(X, Y, c):
        return blur121(curved(X, Y - 1, c), curved(X, Y, c), curved(X, Y + 1, c))

    def unsharp(X, Y, c):
        return blur121(unsharp_y(X - 1, Y, c), unsharp_y(X, Y, c), unsharp_y(X + 1, Y, c))

    def sharpened(X, Y, c):
        cur = curved(X, Y, c)
        mask = cur.astype(i16) - unsharp(X, Y, c).astype(i16)
        t = (mask * i16(strength)) >> 5          # int16 product wraps; Euclidean / 32
        return np.clip(cur.astype(i16) + t, 0, 255).astype(u8)

    Y, X = np.meshgrid(np.arange(out_mins[1], out_mins[1] + H), np.arange(out_mins[0], out_mins[0] + W), indexing="ij")
    return np.stack([sharpened(X, Y, out_mins[2] + c) for c in range(C)])


def conv_layer(inp, filt, bias):
    """apps/conv_layer/conv_layer_generator.cpp:18-25: conv = bias; conv += filter(c, r.y, r.z, r.x) * input(r.x, x + r.y,
    y + r.z, n) over RDom r(ci, kx, ky) with ci innermost, then relu.  Arrays are outermost-first: inp [N, H+2, W+2, CI],
    filt [CI, ky, kx, CO] (Halide filter(c, kx, ky, ci)), bias [CO]."""
    n, hp, wp, ci = inp.shape
    co = bias.shape[0]
    H, W = hp - 2, wp - 2
    acc = np.broadcast_to(bias.astype(F), (n, H, W, co)).copy()
    for ky in range(3):
        for kx in range(3):
            for c in range(ci):
                acc = acc + filt[c, ky, kx, :].astype(F)[None, None, None, :] * inp[:, ky:ky + H, kx:kx + W, c].astype(F)[..., None]
    return np.maximum(acc, F(0.0))
