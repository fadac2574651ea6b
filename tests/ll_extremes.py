"""Content and the case table for the local_laplacian tests at extreme and non-finite alpha and beta (test_ll_extremes.py
on the CPU, test_ll_extremes_gpu.py on the GPU).

The generator takes any float for both scalars.  Past about 1e37 the remap table's values (up to 0.61 alpha) and the
pyramid's 1-3-3-1 sums overflow, and inf - inf makes NaN colours.  Halide's clamp selects on a comparison, so a NaN
colour is 65535 (255 for the 8-bit entry points); a float-to-integer conversion would give 0.  Every case here compares
bit for bit.  The NaN-mixed cases sit where some colours are NaN and some are +-inf or finite: the value depends on the
frame and on `levels`, so test_ll_extremes asserts their shares of each kind, and a change of content that moves them
fails there rather than silently testing something else."""
from collections import namedtuple

import numpy as np

from util import smooth_u16_frame

F = np.float32
# Neither dimension a multiple of a tile (32 x 16 in the final kernel, 28-column strips in level 1); an even width, so the
# final kernel's aligned and TMA paths can take the frame.
SHAPE = (3, 45, 78)
SEED = 11
MIXED_SHARE = 0.05  # least share of NaN, of positive and of negative colours in a NaN-mixed case


def frame(shape=SHAPE, seed=SEED):
    """Smooth content plus noise (util.smooth_u16_frame) with a black block, a 65535 block and a flat mid-grey block.  The
    black block makes 0 * inf = NaN colours and the remap table's ends (gray 0 and 1) are read at the other two."""
    img = smooth_u16_frame(shape, seed)
    _, h, w = shape
    img[:, 5:15, 6:18] = 0
    img[:, h // 2:h // 2 + 8, w // 2:w // 2 + 12] = 65535
    img[:, h - 14:h - 5, w - 19:w - 7] = 32768
    return img


def f32(v):
    """v as the filter receives it: a float32, returned as the Python float of the same value."""
    return float(F(v))


MAX = f32(np.finfo(F).max)
INF, NAN = float("inf"), float("nan")

# The NaN-mixed values of SHAPE / SEED, per `levels`: (alpha at beta 1 and 0.6, beta at alpha 1/7 and 0).  With two
# levels a fine scan of alpha and beta found none: the colours go from no NaN to all NaN at once, below 1e38.
MIXED = {8: (5.4e37, 4.77e37), 32: (1.25e37, 4.77e37), 2: (None, None)}

# Cases whose every colour lies beyond [0, 65535] and none is NaN, so the output is 0 or 65535 by the colour's sign: no
# content can make a rounding mistake or a NaN clamp show there (the three mutations of test_ll_extremes change nothing),
# so test_ll_extremes asserts that they saturate, with both signs present, and a sign mistake still fails them.  Below
# about 5e37 the pyramid's sums stay finite (no NaN), while alpha or beta beyond about 1e12 already take every colour
# out of range.  At 32 levels 4e37 is past the NaN threshold.
SATURATED = {levels: {(1e20, b) for b in (1.0, 0.6)} | {(1e36, b) for b in (1.0, 0.6)} | {(a, 3e37) for a in (1.0 / 7.0, 0.0)}
             for levels in (8, 2, 32)}
for _levels in (8, 2):
    SATURATED[_levels] |= {(4e37, 1.0), (4e37, 0.6), (3e37, -3e37)}

Case = namedtuple("Case", "id levels alpha beta mixed saturated")


def _cases():
    out = []
    for levels in (8, 2, 32):
        mixed_alpha, mixed_beta = MIXED[levels]
        alphas = [0.0, -0.0, 1e-45, 1e-38, 1.0 / 7.0, 1.0, -1.0, 7.0, 1e3, -1e3, 1e20, 1e36, 4e37, 1e38, MAX, -MAX, INF,
                  -INF, NAN]
        betas = [0.0, -0.0, 1e-45, -1.0, 2.0, 1e3, 3e37, 1e38, MAX, INF, -INF, NAN]
        table = [(a, b, False) for b in (1.0, 0.6) for a in alphas]
        table += [(a, b, False) for a in (1.0 / 7.0, 0.0) for b in betas]
        table += [(3e37, -3e37, False), (NAN, NAN, False), (INF, -INF, False)]
        if mixed_alpha is not None:
            table += [(mixed_alpha, b, True) for b in (1.0, 0.6)] + [(a, mixed_beta, True) for a in (1.0 / 7.0, 0.0)]
        saturated = {(f32(a), f32(b)) for a, b in SATURATED[levels]}
        for a, b, mixed in table:
            a, b = f32(a), f32(b)
            out.append(Case(f"L{levels}_a{a:g}_b{b:g}" + ("_mixed" if mixed else ""), levels, a, b, mixed,
                            (a, b) in saturated))
    return out


CASES = _cases()
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASES), "two cases share an id"


def group(levels):
    return [c for c in CASES if c.levels == levels]


def mixed():
    return [c for c in CASES if c.mixed]
