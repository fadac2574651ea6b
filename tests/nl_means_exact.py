"""Content, a float64 reference and the case table for the bit-exact nl_means tests (test_nl_means_exact.py on the CPU,
test_nl_means_exact_gpu.py on the GPU).

On uniform noise in [0, 1) at sigma 0.12 every off-centre patch distance is large, its weight is about exp(-35), and the
filter returns its input: a kernel that reads the wrong neighbour at any off-centre offset still passes.  The content
here is a base plus noise of amplitude about 1.4 sigma, on which every search offset carries weight.  test_nl_means_exact
asserts, for every case of CASES, that the kernel mistakes worth catching (an offset left out, a neighbour one column off,
the patch window one row off) move the float64 result far beyond the oracle's own rounding, and the GPU tests compare
both kernels with the oracle bit for bit on exactly these cases."""
from collections import namedtuple

import numpy as np

from util import f32_frame

# Largest relative difference between the oracle and nl_means64 allowed on a case of CASES: the oracle computes in
# float32 and uses Halide's fast_exp, a degree-5 polynomial, where the reference uses exp.  Measured on CASES: 1.1e-6 at
# search 7 and 8, 2.5e-6 at 13, 3.9e-6 at 17 and 18, 1.05e-5 at 31 and 4.9e-5 at 63 (patch 1; weights vary most there).
# Relative to max(|out|, 0.1), the scale of the terms summed, since the rounding follows that scale even where terms of
# both signs (the clamp cases) give a result near 0.
def oracle_bound(search):
    return 2e-6 * max(1.0, (search / 9.0) ** 2)


# Each mutation must move the float64 output by at least MIN_EFFECT (same measure): ten times the 1e-4 tolerance the
# float pipelines were once held to, so even that tolerance would see it.  With search 31 or 63 one offset is one of 961
# or 3969 carrying similar weights, and with patch 15 or 31 one patch row is a fifteenth or less of every distance, so
# no content with every offset in play gets there.  Those cases, and all others, need the effect to be at least twice
# the oracle's own distance from float64 on the same case: then the mutated result cannot round to the oracle's bits,
# which is all a bit-exact comparison needs.
MIN_EFFECT = 1e-3
FLOOR = 0.1


def sensitive_frame(c, h, w, sigma, seed, lo=0.3, outside=False, amp=None):
    """float32 [c, h, w]: lo plus uniform noise of amplitude 1.4 |sigma| (at most 0.6, so the frame stays in [0, 1] for
    the default lo; amp overrides it).  outside=True adds a slow wave that takes the frame over [-0.5, 1.5], so the
    final clamp to [0, 1] acts on both sides while neighbouring patches stay alike."""
    amp = min(1.4 * abs(sigma), 0.6) if amp is None else amp
    noise = amp * f32_frame((c, h, w), seed)
    if not outside:
        return (lo + noise).astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    wave = np.stack([np.sin(2 * np.pi * (xx + 11 * k) / 48.0) * np.cos(2 * np.pi * yy / 64.0) for k in range(c)])
    return np.clip(0.5 - amp / 2 + (1.0 - amp / 2) * wave + noise, -0.5, 1.5).astype(np.float32)


def offsets(search):
    """Search offsets (dx, dy) in the oracle's order: dy outer, dx inner, both ascending from -(search / 2)."""
    lo = -(search // 2)
    return [(dx, dy) for dy in range(lo, lo + search) for dx in range(lo, lo + search)]


def probe_offsets(search):
    """The offsets the mutations act on: the four corners and (+-1, 0), (0, +-1), where the window has them."""
    lo = -(search // 2)
    hi = lo + search - 1
    cand = [(lo, lo), (hi, lo), (lo, hi), (hi, hi), (-1, 0), (1, 0), (0, -1), (0, 1)]
    return [o for o in dict.fromkeys(cand) if o != (0, 0) and lo <= min(o) and max(o) <= hi]


def _box(a, p, axis):
    """Sums of p consecutive entries along axis (length n - p + 1), by cumulative sum in float64."""
    cs = np.cumsum(a, axis=axis)
    cs = np.concatenate([np.zeros_like(np.take(cs, [0], axis=axis)), cs], axis=axis)
    n = a.shape[axis]
    return np.take(cs, range(p, n + 1), axis=axis) - np.take(cs, range(0, n - p + 1), axis=axis)


def nl_means_terms(inp, patch, search, sigma, out_shape=None, in_mins=None, out_mins=None, patch_row=0):
    """Per search offset (offsets(search) order): the weight [H, W] and the neighbour [3, H, W] it multiplies, in
    float64 with np.exp, plus a function giving the neighbour at another offset.  Coordinates clamp to the input's
    extent in x, y and channel, as the filter's do.  patch_row moves every patch window down by that many rows (a
    mutation)."""
    inp = np.asarray(inp)
    in_c, h, w = inp.shape
    ix, iy, ic = in_mins or (0, 0, 0)
    H, W = (out_shape or inp.shape)[1:]
    ox, oy = (out_mins or (0, 0, 0))[:2]
    r = patch + search + 2
    xi = np.clip(np.arange(ox - r, ox + W + r) - ix, 0, w - 1)
    yi = np.clip(np.arange(oy - r, oy + H + r) - iy, 0, h - 1)
    ci = np.clip(np.arange(3), ic, ic + in_c - 1) - ic
    f = inp.astype(np.float64)[ci][:, yi][:, :, xi]

    def at(dx, dy, hh=H, ww=W):  # [3, hh, ww] of the clamped frame from (ox + dx, oy + dy)
        return f[:, r + dy:r + dy + hh, r + dx:r + dx + ww]

    inv = -1.0 / (float(sigma) ** 2 * patch * patch)
    p_lo = -(patch // 2)
    centre = at(p_lo, p_lo + patch_row, H + patch - 1, W + patch - 1)
    weights, neighbours = [], []
    for dx, dy in offsets(search):
        d = ((centre - at(p_lo + dx, p_lo + patch_row + dy, H + patch - 1, W + patch - 1)) ** 2).sum(0)
        bd = _box(_box(d, patch, 0), patch, 1)
        weights.append(np.exp(bd * inv))
        neighbours.append(at(dx, dy))
    return weights, neighbours, at


def nl_means64(inp, patch, search, sigma, **kw):
    """nl_means in float64 with np.exp: clamp(sum w * neighbour / sum w, 0, 1), float64 [3, H, W]."""
    weights, neighbours, _ = nl_means_terms(inp, patch, search, sigma, **kw)
    return np.clip(sum(wt * nb for wt, nb in zip(weights, neighbours)) / sum(weights), 0.0, 1.0)


def rel(a, b):
    """Largest |a - b| relative to max(|b|, FLOOR)."""
    return float((np.abs(np.asarray(a, np.float64) - b) / np.maximum(np.abs(b), FLOOR)).max())


def mutation_effects(inp, patch, search, sigma, **kw):
    """{mutation: rel(mutated float64 result, float64 result)} for the mistakes a kernel could make: each probe offset
    left out of the sum ("drop"), its neighbour read one column to the right ("shift"), and every patch window one row
    down ("patch_row")."""
    weights, neighbours, at = nl_means_terms(inp, patch, search, sigma, **kw)
    num, den = sum(wt * nb for wt, nb in zip(weights, neighbours)), sum(weights)
    ref = np.clip(num / den, 0.0, 1.0)
    index = {o: i for i, o in enumerate(offsets(search))}
    out = {}
    for dx, dy in probe_offsets(search):
        k = index[(dx, dy)]
        wt, nb = weights[k], neighbours[k]
        out[f"drop({dx},{dy})"] = rel(np.clip((num - wt * nb) / (den - wt), 0.0, 1.0), ref)
        out[f"shift({dx},{dy})"] = rel(np.clip((num + wt * (at(dx + 1, dy) - nb)) / den, 0.0, 1.0), ref)
    out["patch_row"] = rel(nl_means64(inp, patch, search, sigma, patch_row=1, **kw), ref)
    return out


# ---- the cases -------------------------------------------------------------------------------------------------------
# Every case the GPU file runs.  need: the least mutation effect test_nl_means_exact asserts, or None with the reason
# the content cannot show one (then the case still runs bit for bit on the GPU).
Case = namedtuple("Case", "id group patch search sigma shape seed content kw need why")
PATCHES = (1, 2, 3, 4, 5, 7, 9, 15, 31)
SEARCHES = (1, 2, 3, 4, 7, 8, 13, 31, 63)
ORACLE_BUDGET = 4e7  # search^2 * patch^2 * output pixels per oracle call: about a second
H4K, W4K = 2160, 3840
REGION = 64  # config-4 regions: REGION x REGION outputs, cropped from the frame with a 16-pixel margin
REGIONS_4K = [(0, 0), (0, W4K - REGION), (H4K - REGION, 0), (H4K - REGION, W4K - REGION), (1000, 1900),
              (540 - 32, 3000), (1080 - 8, 1920 - 16), (2000, 77)]


def _need(patch, search):
    return MIN_EFFECT if search <= 13 and patch <= 9 else 0.0


def case(id, group, patch, search, sigma, shape, seed, content=None, kw=None, why=None, need=None):
    need = _need(patch, search) if need is None else need
    return Case(id, group, patch, search, sigma, shape, seed, content or {}, kw or {}, None if why else need, why)


def interior(patch, search, h, w, seed, sigma=0.12):
    """A frame with an output window whose every read, shifted one column more, stays inside the input (so no offset
    clamps onto another); the window is the whole frame where the oracle budget allows."""
    m = search // 2 + patch // 2 + 2
    while h > 1 and w > 1 and search ** 2 * patch ** 2 * h * w > ORACLE_BUDGET:
        h, w = (h + 1) // 2, (w + 1) // 2
    shape = (3, h + 2 * m, w + 2 * m)
    if search ** 2 * patch ** 2 * shape[1] * shape[2] <= ORACLE_BUDGET:
        return dict(shape=shape, seed=seed)
    return dict(shape=shape, seed=seed, kw=dict(out_shape=(3, h, w), out_mins=(m, m, 0)))


def _cases():
    out = []
    # tile seams and ragged frames at config 4's parameters
    for w in (1, 2, 31, 32, 33, 63, 65, 97):
        for h in (1, 15, 16, 17, 33):
            why = "a frame 1 or 2 pixels across: most offsets clamp onto the same pixels" if min(h, w) <= 2 else None
            out.append(case(f"seam{h}x{w}", "seams", 3, 7, 0.12, (3, h, w), 100 * h + w, why=why))
    mins = {  # (input shape, input mins, output shape, output mins)
        "out_inside": ((3, 50, 70), (-4, 2, 0), (3, 30, 41), (1, 6, 0)),
        "out_left_top": ((3, 40, 70), (5, 3, 0), (3, 33, 65), (-3, -2, 0)),
        "out_right_bottom": ((3, 40, 70), (5, 3, 0), (3, 33, 65), (30, 20, 0)),
        "negative_mins": ((3, 40, 70), (-100, -37, 0), (3, 33, 65), (-93, -33, 0)),
        "out_larger": ((3, 20, 30), (0, 0, 0), (3, 40, 70), (-10, -9, 0)),
        "in_smaller_than_apron": ((3, 3, 2), (4, -6, 0), (3, 17, 33), (-8, -12, 0)),
    }
    for name, (shape, imins, oshape, omins) in mins.items():
        why = "a 2 x 3 input: most offsets clamp onto the same pixels" if shape[1] * shape[2] < 10 else None
        out.append(case(name, "mins", 3, 7, 0.12, shape, len(out), kw=dict(in_mins=imins, out_shape=oshape,
                                                                            out_mins=omins), why=why))
    # patch x search grid
    for p in PATCHES:
        for s in SEARCHES:
            why = "search 1: the centre is the only offset" if s == 1 else None
            out.append(case(f"p{p}s{s}", "grid", p, s, 0.12, why=why, **interior(p, s, 17, 33, 1000 + 100 * p + s)))
    # dx batches of the generic kernel, each side of each threshold (test_nl_means_exact_gpu asserts the sides)
    for p, s in ((3, 7), (3, 8), (3, 17), (3, 18), (7, 14), (7, 15), (15, 9), (15, 10), (15, 11), (31, 4), (31, 5),
                 (9, 31)):
        out.append(case(f"dx_p{p}s{s}", "dx", p, s, 0.12, **interior(p, s, 17, 33, 2000 + 100 * p + s)))
    # the final clamp
    for p in (3, 7, 5):
        # a third of the pixels clamp, where no mistake shows: only twice the oracle's deviation is asked
        out.append(case(f"clamp_p{p}", "clamp", p, 7, 0.12, (3, 64, 96), 3000 + p, dict(outside=True), need=0.0))
    # sigma
    for sigma in (1e-20, 1e-4, 0.12, -0.12, 1.0, 1e4, float("inf")):
        content = dict(amp=0.2) if abs(sigma) < 0.01 else {}
        why = "every off-centre weight is 0 (or NaN)" if abs(sigma) < 0.01 else None
        out.append(case(f"sigma{sigma:g}", "sigma", 3, 7, sigma, (3, 33, 65), 4000, content, why=why))
    # input channels
    for in_c, c0 in ((1, 0), (2, 0), (4, 0), (3, 1)):
        out.append(case(f"channels{in_c}_min{c0}", "channels", 3, 7, 0.12, (in_c, 37, 53), 5000 + 10 * in_c + c0,
                        kw=dict(in_mins=(0, 0, c0))))
    # config 4: regions of the 3840 x 2160 frame, as the crops that determine them
    for y0, x0 in REGIONS_4K:
        ya, yb, xa, xb = max(0, y0 - 16), min(H4K, y0 + REGION + 16), max(0, x0 - 16), min(W4K, x0 + REGION + 16)
        out.append(case(f"4k_{y0}_{x0}", "config4", 3, 7, 0.12, (3, H4K, W4K), 4,
                        kw=dict(crop=(ya, yb, xa, xb), in_mins=(xa, ya, 0), out_mins=(xa, ya, 0))))
    return out


CASES = _cases()
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASES)


def group(name):
    return [c for c in CASES if c.group == name]


_frames = {}


def frame(c):
    """(input, keyword arguments for nl_means64 / the oracle / run) of a case.  Config-4 cases give the crop of the
    whole frame that determines their region."""
    key = (c.shape, c.seed, c.sigma, tuple(sorted(c.content.items())))
    if key not in _frames:
        if c.group == "config4":  # keep one 100 MB frame at a time
            _frames.clear()
        _frames[key] = sensitive_frame(*c.shape, c.sigma, c.seed, **c.content)
    inp, kw = _frames[key], dict(c.kw)
    if "crop" in kw:
        ya, yb, xa, xb = kw.pop("crop")
        inp = np.ascontiguousarray(inp[:, ya:yb, xa:xb])
        kw["out_shape"] = inp.shape
    kw.setdefault("out_shape", (3,) + inp.shape[1:])
    return inp, kw
