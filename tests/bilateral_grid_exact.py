"""Content, a float64 reference and the case table for the bit-exact bilateral_grid tests (test_bilateral_grid_exact.py
on the CPU, test_bilateral_grid_exact_gpu.py on the GPU).

The any-S kernels (bg_hist_blurz_s, bg_blur_xy, bg_slice_s) perform the oracle's float operations in the oracle's order,
so they give its bits on any input.  bilateral_grid's own histogram kernel (bg_hist_blurz, s_sigma = 8) adds each bin as
two 4-column partial sums, which gives the oracle's bits wherever every partial sum is exact: on a frame of multiples of
2^-16 (a uint16 frame / 65536) a bin holds at most 64 such values and every partial sum fits in 22 bits.  So every case
at s_sigma = 8 uses that "dyadic" content, and every case is compared bit for bit."""
from collections import namedtuple

import numpy as np

from halide_b200 import dist
from util import f32_frame, u16_frame

KERNELS_8 = frozenset({"bg_hist_blurz", "bg_blur_xy", "bg_slice"})
KERNELS_S = frozenset({"bg_hist_blurz_s", "bg_blur_xy", "bg_slice_s"})


def kernels(s):
    """The kernels a call with cell size s must run: bilateral_grid's own at s = 8, the any-S kernels otherwise."""
    return KERNELS_8 if s == 8 else KERNELS_S


# Largest relative difference (|a - b| / max(|b|, FLOOR)) between the oracle and bilateral_grid64 allowed on a case of
# CASES.  The oracle sums each bin of up to s^2 pixels in float32, one rounding per term, so its error grows with s^2; the
# blurs and the slice add a few roundings more, and all terms are non-negative, so nothing cancels.  Measured on CASES
# (the largest over each s): 3.3e-7 at s <= 5, 4.4e-7 at 7, 3.0e-7 at 8, 9.6e-7 at 9, 2.0e-6 at 16, 7.8e-6 at 31, 2.9e-5
# at 64, 9.5e-5 at 100, 9.0e-5 at 127 and 1.57e-4 at 128 (r_sigma 1 / 199: 200 bins).
FLOOR = 1e-6


def oracle_bound(s):
    return 1e-6 + 1.5e-8 * s * s


# ---- content -------------------------------------------------------------------------------------------------------

def noise(shape, seed, spread=False):
    """Uniform float32 noise in [0, 1), or spread over [-0.25, 1.25) so the input clamp acts on both sides."""
    f = f32_frame(shape, seed)
    return (f * np.float32(1.5) - np.float32(0.25)).astype(np.float32) if spread else f


def dyadic(shape, seed, spread=False):
    """float32 multiples of 2^-16: u16_frame / 65536 in [0, 1), or in [-0.25, 1.25) when spread."""
    if not spread:
        return (u16_frame(shape, seed).astype(np.float64) / 65536).astype(np.float32)
    u = np.random.default_rng(seed).integers(-16384, 65536 + 16384, shape)
    return (u / 65536).astype(np.float32)


DENORMAL = np.nextafter(np.float32(0), np.float32(1))


def special_values(s, r_sigma):
    """NaN, +-inf, -0.0, 0, 1, the smallest denormal (except at s = 8: it is no multiple of 2^-16) and every value on
    a histogram bin boundary, where val * inv_r + 0.5 is exactly an integer (exact for r_sigma a power of two)."""
    inv_r = 1.0 / r_sigma
    assert inv_r == np.float32(1) / np.float32(r_sigma) and inv_r == int(inv_r), r_sigma
    vals = [np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0] + ([] if s == 8 else [DENORMAL])
    vals += [(k - 0.5) / inv_r for k in range(1, int(inv_r) + 1)]
    return np.array(vals, np.float32)


def special_positions(s, h, w):
    """(y, x) pixels: the frame's corners and edge midpoints, and along each axis a histogram cell's first and last
    pixel (cells start at n * s - s / 2), a slice cell's first pixel (n * s) and a cell interior, in every third cell."""
    def axis(n):
        at = {0, n - 1, n // 2}
        for c in range(0, n // s + 2, 3):
            at |= {c * s - s // 2, c * s - s // 2 + s - 1, c * s, c * s + s // 3}
        return sorted(i for i in at if 0 <= i < n)
    ys, xs = axis(h), axis(w)
    edges = [(y, x) for y in (0, h // 2, h - 1) for x in (0, w // 2, w - 1)]
    return list(dict.fromkeys(edges + [(y, x) for y in ys for x in xs]))


def with_specials(frame, s, r_sigma, seed):
    """frame with the special values cycled over special_positions, in a seeded order."""
    out = frame.copy()
    vals = special_values(s, r_sigma)
    pos = special_positions(s, *frame.shape)
    order = np.random.default_rng(seed).permutation(len(pos))
    for k, i in enumerate(order):
        out[pos[i]] = vals[k % len(vals)]
    return out


# ---- float64 reference ---------------------------------------------------------------------------------------------

def clamp01(v):
    """clamp(v, 0, 1) as Halide's min / max select it: min(v, 1) is v < 1 ? v : 1 and max(m, 0) is m > 0 ? m : 0, so
    NaN gives 1 and -0.0 gives 0.  (np.clip and np.minimum propagate NaN.)"""
    m = np.where(v < 1, v, 1.0)
    return np.where(m > 0, m, 0.0)


def params(r_sigma):
    """The filter's float32 parameters: inv_r = 1 / r_sigma and the largest bin zmax = int(1 * inv_r + 0.5)."""
    f = np.float32
    inv_r = f(1) / f(r_sigma)
    return inv_r, int(f(f(1) * inv_r) + f(0.5))


def cells(inp, s, r_sigma, out_shape=None, in_mins=None, out_mins=None):
    """The histogram cells of the grid a call computes, cell rows gy0 .. gy1 and columns gx0 .. gx1 (the slice's cells
    grown by 2 for each blur): (clamped pixel values float64 [GH, GW, s, s], their bins [GH, GW, s, s], (gx0, gy0)).
    Cell (gx, gy) holds the pixels (gx * s + rx - s / 2, gy * s + ry - s / 2) at [ry, rx], read at coordinates clamped
    to the input.  The bin is the generator's float32 expression int(val * inv_r + 0.5)."""
    h, w = inp.shape
    ix, iy = in_mins or (0, 0)
    H, W = out_shape or inp.shape
    ox, oy = out_mins or (0, 0)
    gx0, gx1 = ox // s - 2, (ox + W - 1) // s + 3
    gy0, gy1 = oy // s - 2, (oy + H - 1) // s + 3
    GW, GH = gx1 - gx0 + 1, gy1 - gy0 + 1
    xs = np.clip(np.arange(gx0 * s - s // 2, (gx1 + 1) * s - s // 2) - ix, 0, w - 1)
    ys = np.clip(np.arange(gy0 * s - s // 2, (gy1 + 1) * s - s // 2) - iy, 0, h - 1)
    raw = inp[ys][:, xs]
    val32 = clamp01(raw).astype(np.float32)
    inv_r, _ = params(r_sigma)
    zi = (val32 * inv_r + np.float32(0.5)).astype(np.int64)
    split = lambda a: a.reshape(GH, s, GW, s).transpose(0, 2, 1, 3)  # noqa: E731
    return split(val32.astype(np.float64)), split(zi), (gx0, gy0)


def blur5(a, axis):
    """1 4 6 4 1 along axis, valid part (length n - 4)."""
    n = a.shape[axis]
    t = lambda o: np.take(a, range(o, n - 4 + o), axis=axis)  # noqa: E731
    return t(0) + 4 * t(1) + 6 * t(2) + 4 * t(3) + t(4)


def lerp(a, b, w):
    return a * (1 - w) + b * w


def bilateral_grid64(inp, s, r_sigma, out_shape=None, in_mins=None, out_mins=None):
    """bilateral_grid in float64 (float64 [H, W]): the histogram of each cell's (value, 1) over its bins, the 1 4 6 4 1
    blurs along z, x and y, the trilinear slice at (x / s, y / s, val * inv_r) and value / weight.  Only the bin index
    is taken in float32, where the generator defines it."""
    H, W = out_shape or inp.shape
    ix, iy = in_mins or (0, 0)
    ox, oy = out_mins or (0, 0)
    vals, zi, (gx0, gy0) = cells(inp, s, r_sigma, out_shape, in_mins, out_mins)
    inv_r, zmax = params(r_sigma)
    GH, GW = vals.shape[:2]
    nb = zmax + 1
    cell = np.arange(GH * GW).reshape(GH, GW, 1, 1)
    idx = (cell * nb + zi).ravel()
    hist = np.zeros((GH, GW, nb + 5, 2))  # bins -2 .. zmax + 2, zero outside [0, zmax]
    hist[:, :, 2:2 + nb, 0] = np.bincount(idx, vals.ravel(), GH * GW * nb).reshape(GH, GW, nb)
    hist[:, :, 2:2 + nb, 1] = np.bincount(idx, minlength=GH * GW * nb).reshape(GH, GW, nb)
    grid = blur5(blur5(blur5(hist, 2), 1), 0)  # planes 0 .. zmax + 1, cells gx0 + 2 .. and gy0 + 2 ..
    x = np.arange(ox, ox + W)
    y = np.arange(oy, oy + H)[:, None]
    val = clamp01(inp[y - iy, x - ix].astype(np.float64))
    zv = val * float(inv_r)
    z = np.floor(zv).astype(np.int64)
    zf = zv - z
    xi, xf = x // s - gx0 - 2, (x % s) / s
    yi, yf = y // s - gy0 - 2, (y % s) / s

    def at(dx, dy, dz):
        return grid[yi + dy, xi + dx, z + dz]

    def plane(dz):
        return lerp(lerp(at(0, 0, dz), at(1, 0, dz), xf[..., None]), lerp(at(0, 1, dz), at(1, 1, dz), xf[..., None]),
                    yf[..., None])

    out = lerp(plane(0), plane(1), zf[..., None])
    return out[..., 0] / out[..., 1]


def rel(a, b):
    """Largest |a - b| relative to max(|b|, FLOOR)."""
    return float((np.abs(np.asarray(a, np.float64) - b) / np.maximum(np.abs(b), FLOOR)).max())


# ---- the cases -----------------------------------------------------------------------------------------------------
# content: kind ("noise" or "dyadic"), spread (over [-0.25, 1.25)), specials (with_specials).  kw: in_mins, out_shape,
# out_mins, or crop (y0, y1, x0, x1) of the frame for the config-3 regions.
Case = namedtuple("Case", "id group s r_sigma shape seed content kw kernels")
S_SIZES = (1, 2, 3, 4, 5, 7, 9, 12, 16, 31, 32, 64, 100, 128, 8, 33, 127)  # test_bilateral_grid_s_sigma_gpu's S, 8, 33, 127
S_BINS = (1, 8, 16, 128)
S_CROPS = (3, 5, 8, 12, 33)
S_SPECIALS = (1, 3, 8, 16, 128)
S_CONFIG3 = (3, 8, 16, 64)
H8K, W8K = 4320, 7680
REGION = 96
REGIONS_8K = [(0, 0), (0, W8K - REGION), (H8K - REGION, 0), (H8K - REGION, W8K - REGION), (2001, 3333),
              (4096 - 45, 4096 - 51), (2160 - 4, 3840 - 61)]


def r_sigma_for(zmax):
    """An r_sigma whose largest bin is zmax."""
    r = float(np.float32(1.0) / np.float32(zmax))
    assert params(r)[1] == zmax
    return r


def case(id, group, s, r_sigma, shape, seed, spread=False, specials=False, kw=None):
    content = dict(kind="dyadic" if s == 8 else "noise", spread=spread, specials=specials)
    return Case(id, group, s, r_sigma, shape, seed, content, kw or {}, kernels(s))


def _cases():
    out = []
    for s in S_SIZES:
        for h, w in [(1, 1), (max(1, s - 1), s + 1), (61, 107), (240, 519)]:
            out.append(case(f"size_s{s}_{h}x{w}", "sizes", s, 0.1, (h, w), 1000 * s + h + w, spread=(h * w) % 2 == 1))
    crops = {  # (input shape, input mins, output shape, output mins), (x, y) mins
        "negative": ((130, 170), (-29, -21), (70, 101), (-19, -11)),
        "mismatched": ((130, 170), (-13, 5), (45, 61), (-6, 23)),
        "same_mins": ((97, 131), (-7, -3), (97, 131), (-7, -3)),
        "one_px": ((60, 80), (3, 4), (1, 1), (40, 37)),
    }
    for s in S_CROPS:
        mid = ((130, 170), (0, 0), (45, 61), (2 * s + s // 2 + 1, 2 * s - 1))  # the output starts inside a cell
        for name, (shape, imins, oshape, omins) in dict(crops, mid_cell=mid).items():
            kw = dict(in_mins=imins, out_shape=oshape, out_mins=omins)
            out.append(case(f"crop_{name}_s{s}", "crops", s, 0.25 if name == "mismatched" else 0.1, shape,
                            len(out), spread=name != "same_mins", kw=kw))
    rs = [0.05, 0.1, 0.25, 1.0] + [r_sigma_for(z) for z in (47, 48, 126, 127, 199)] + [float("inf")]
    for s in S_BINS:
        for k, r in enumerate(rs):
            out.append(case(f"bins_s{s}_r{r:.6g}", "bins", s, r, (61, 107), 2000 + 10 * s + k, spread=k % 2 == 1))
    for s in S_SPECIALS:
        shape = (max(61, 2 * s + 37), max(107, 3 * s + 11))
        for r in (0.125, 0.0625):
            out.append(case(f"specials_s{s}_r{r:g}", "specials", s, r, shape, 3000 + s, spread=True, specials=True))
    for s in S_CONFIG3:
        m = 5 * s
        for y0, x0 in REGIONS_8K:
            ya, yb, xa, xb = max(0, y0 - m), min(H8K, y0 + REGION + m), max(0, x0 - m), min(W8K, x0 + REGION + m)
            out.append(case(f"8k_s{s}_{y0}_{x0}", "config3", s, 0.1, (H8K, W8K), 21 + s,
                            kw=dict(crop=(ya, yb, xa, xb), in_mins=(xa, ya), out_mins=(xa, ya))))
    return out


CASES = _cases()
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASES)
assert all(c.content["kind"] == "dyadic" for c in CASES if c.s == 8)  # bg_hist_blurz's bits need exact bin sums


def group(name):
    return [c for c in CASES if c.group == name]


def content(c):
    """The whole frame of case c (float32 [h, w])."""
    gen = dyadic if c.content["kind"] == "dyadic" else noise
    f = gen(c.shape, c.seed, c.content["spread"])
    return with_specials(f, c.s, c.r_sigma, c.seed) if c.content["specials"] else f


_frames = {}


def frame(c):
    """(input, keyword arguments for bilateral_grid64 / the oracle / the filter) of a case.  Config-3 cases give the
    crop of the whole frame that determines their region (the blurs reach 2 cells and the slice 1: margin 5 s)."""
    key = (c.shape, c.seed, tuple(sorted(c.content.items())), c.s, c.r_sigma)
    if key not in _frames:
        if c.group == "config3":  # keep one 130 MB frame at a time
            _frames.clear()
        _frames[key] = content(c)
    inp, kw = _frames[key], dict(c.kw)
    if "crop" in kw:
        ya, yb, xa, xb = kw.pop("crop")
        inp = np.ascontiguousarray(inp[ya:yb, xa:xb])
        kw["out_shape"] = inp.shape
    return inp, kw


def region(c):
    """(y0, x0) of a config-3 case's REGION x REGION output within the frame."""
    return tuple(int(t) for t in c.id.split("_")[2:])


# ---- row bands -----------------------------------------------------------------------------------------------------

def halo_derived(s):
    """(rows above, rows below) an output row y reads: grid cells yi - 2 .. yi + 3 (yi = floor(y / s): the slice reads
    yi and yi + 1, blury 2 more on each side), cell gy holding rows gy * s - s / 2 .. gy * s - s / 2 + s - 1.  The most
    above is at y mod s = s - 1, the most below at y mod s = 0.  That last row below is read but weighs nothing: at
    y mod s = 0 the slice's fraction yf is 0, and lerp(a, b, 0) = a * 1 + b * 0 is a, bit for bit, so the output
    depends on no row past 4 s - 2 - s / 2 below (reached at y mod s = 1; at s = 1 too, where every yf is 0)."""
    return 3 * s - 1 + s // 2, 4 * s - 1 - s // 2


BAND_WORLDS = (2, 3, 4, 8)


def band_height(s, start=600):
    """The least frame height from start on whose band_rows boundaries, over BAND_WORLDS, include a band starting at a
    row = s - 1 (mod s) and a band ending at a row = 1 (mod s): the rows whose output depends on the farthest halo row
    above, and the farthest one that carries weight below."""
    h = start
    while True:
        los = {dist.band_rows(r, w, h)[0] for w in BAND_WORLDS for r in range(1, w)}
        if any(lo % s == s - 1 for lo in los) and any((lo - 1) % s == 1 % s for lo in los):
            return h
        h += 1
