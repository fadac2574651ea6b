"""Every filter family on device-resident frames whose elements lie 2^31 or more elements or bytes apart.

check_shapes limits each dimension to extent * |stride| <= 2^31 - 1 elements, but not their sum, and not bytes: a legal
(x, y, c[, n]) buffer can hold elements up to about dimensions x 2^31 elements from its first one.  The kernels pick
their index width on purpose (local_laplacian's level-1 kernel takes 32-bit element offsets only when `idx32` holds, its
final kernel an aligned form only when `final_form`'s spans are below 2^31; the other filters widen to 64 bits at each
use), so every case here puts a small frame (at most 256 x 256 per frame) on one side of one of those lines, or past
2^31 elements or bytes, through its row, channel, pixel or frame strides.

- One device arena per case, filled with a sentinel byte; the input and output are strided views of it (HalideBuffer
  wrapping the device pointer: no host copy of a huge-pitch buffer is ever made).
- The output, read back compactly, against each filter's oracle rule; the input must be unchanged, and every arena byte
  the output does not describe must still hold the sentinel (the whole arena is scanned).
- local_laplacian frames whose own samples (planar and interleaved, input and output) lie past 2^31 elements from the
  frame's first, on the 64-bit side of idx32 and of both spans, at every final-kernel mask.
- test_cases_sit_where_they_claim (no GPU): restates idx32, final_form (spans, word alignment, masks and the TMA frame
  tile's rules) and check_shapes' limits in Python and checks every case against the side and the final-kernel form its
  description claims, and that its views are disjoint and fit the arena.

Not covered: host buffers with such pitches (the runtime's host <-> device copies), local_laplacian's tone kernel's
row-band split (it starts at 2^34 pixels) and the row-sharded local_laplacian."""
import ctypes
import gc
import importlib
from dataclasses import dataclass

import numpy as np
import pytest

from bilateral_grid_exact import KERNELS_8, KERNELS_S, dyadic, noise
from conv_any_exact import harness, worst_ratio
from halide_b200.image_io import convert
from test_camera_pipe_edges_gpu import raw_frame
from util import CP_M3200, CP_M7000, cp_params, f32_frame, kernels_run, nl_means_variant, u16_frame

G = 1 << 31
ARENA_CAP = 12 << 30  # bytes: the most one case may allocate
SENTINEL = 0xA5
FRAME_CAP = 256 * 256 * 4  # elements of one compact frame
LL_ALPHA, LL_LEVELS = 1.0 / 7.0, 8
CP = cp_params({})


# ---- views and cases ------------------------------------------------------------------------------------------------

@dataclass
class View:
    """A strided buffer inside the arena: logical shape and element strides outermost first (torch / numpy order),
    the byte offset of its first element (all indices 0), Halide mins and whether it is pixel-interleaved (the logical
    channel axis is then the one of stride 1)."""
    dtype: object
    shape: tuple
    strides: tuple
    at: int
    mins: tuple = None
    il: bool = False

    @property
    def isz(self):
        return np.dtype(self.dtype).itemsize

    def reach(self):
        """(lowest, highest) element offset from the first element."""
        lo = sum((e - 1) * s for e, s in zip(self.shape, self.strides) if s < 0)
        hi = sum((e - 1) * s for e, s in zip(self.shape, self.strides) if s > 0)
        return lo, hi

    def halide(self):
        """[(extent, stride)] in Halide order (x first)."""
        return list(zip(reversed(self.shape), reversed(self.strides)))

    def byte_set(self):
        """Every byte address the view's elements occupy (the frames are small)."""
        idx = np.zeros((), np.int64)
        for e, s in zip(self.shape, self.strides):
            idx = idx[..., None] + np.arange(e, dtype=np.int64) * s
        first = self.at + idx.ravel() * self.isz
        return (first[:, None] + np.arange(self.isz)).ravel()


@dataclass
class Case:
    """A call on strided views.  `call(hb, ins, out)` runs it on HalideBuffers; `want(oracle, xs)` gives the logical
    output from the compact inputs, or `check(hb, oracle, got, xs)` judges it; `claims` {rule: side} and `why`, the description
    of where the case sits; `kernels`: launches the call must make; `force`: the local_laplacian path mask."""
    id: str
    ins: list
    out: View
    data: object
    call: object
    why: str
    claims: dict
    want: object = None
    check: object = None
    kernels: frozenset = frozenset()
    force: int = 0
    variant: int = 0
    ll: bool = False


def max_offset(v):
    lo, hi = v.reach()
    return max(-lo, hi)


def frame_dims(v, clip):
    """The Halide (extent, stride) of one frame: all dimensions but a clip's last."""
    d = v.halide()
    return d[:-1] if clip else d


def ll_idx32(v, clip):
    """local_laplacian.cu, launch_level12_kernel: the level-1 kernel's 32-bit element offsets."""
    d = frame_dims(v, clip)
    (w, sx), (h, sy), (c, sc) = d[:3]
    px = sx if v.il else 0
    return sy > 0 and sc > 0 and h * sy + c * sc + w * px < G


def ll_span(v, clip):
    """local_laplacian.cu, final_form: in_span / out_span = extent_y * stride_y + 3 * stride_c, below 2^31."""
    d = frame_dims(v, clip)
    return d[1][0] * d[1][1] + 3 * d[2][1] < G


def frame_reach(v, clip, channels=None):
    """The farthest element of one frame a local_laplacian call touches, in elements from the frame's first: over its
    first `channels` channels (the input's first three are the ones read)."""
    d = frame_dims(v, clip)
    c = d[2][0] if channels is None else min(channels, d[2][0])
    return (d[0][0] - 1) * abs(d[0][1]) + (d[1][0] - 1) * abs(d[1][1]) + (c - 1) * abs(d[2][1])


ARENA_ALIGN = 256  # the arena's base address is a multiple of this (the GPU test asserts it)


def ll_final_form(case):
    """local_laplacian.cu: final_form (the span rule, the word-alignment rule and the masks) and frame_tile_map's
    16-byte TMA rules, for a case at mins 0 whose batch runs as one group: the final kernel's form."""
    i, o = case.ins[0], case.out
    clip = len(o.shape) == 4
    di, do = i.halide(), o.halide()
    eb = i.isz
    wb = 2 * eb
    (W, opx), (_, osy), (C, osc) = do[:3]
    (_, ipx), (_, isy), (ic, isc) = di[:3]
    N = do[3][0] if clip else 1
    fs_in, fs_out = (di[3][1], do[3][1]) if N > 1 else (0, 0)
    general, tile_tma = bool(case.force & 16), not case.force & 64

    def mult(n, *vals):
        return all(x % n == 0 for x in vals)
    assert ARENA_ALIGN % 16 == 0
    if i.il:
        pairs = W % 2 == 0 and osy > 0 and mult(wb, o.at, osy * eb, fs_out * eb)
        rgb = C == 3 and ic == ipx and (ipx, opx) in ((3, 3), (4, 3), (4, 4))
        if not (pairs and not general and tile_tma and rgb):
            return "GeneralIL"
        form = "Rgb" if ipx == 3 else "RgbaToRgb" if opx == 3 else "Rgba"
    else:
        aligned = (C == 3 and ic >= 3 and isy > 0 and isc > 0 and osy > 0 and osc > 0 and ll_span(i, clip) and
                   ll_span(o, clip) and mult(wb, W * eb, i.at, o.at, isy * eb, isc * eb, osy * eb, osc * eb,
                                             fs_in * eb, fs_out * eb))
        if not aligned or general:
            return "General"
        if not tile_tma:
            return "Aligned"
        form = "AlignedTma"
    # frame_tile_map: a 16-byte aligned base and positive strides below 2^40 that are multiples of 16 bytes
    strides = [isy * eb] + ([] if i.il else [isc * eb]) + ([fs_in * eb] if N > 1 else [])
    if i.at % 16 == 0 and all(0 < st < 1 << 40 and st % 16 == 0 for st in strides):
        return form
    return "Aligned" if form == "AlignedTma" else "GeneralIL"


def facts(case):
    """Each rule a case can claim a side of, computed from its views."""
    i, o = case.ins[0], case.out
    clip = len(o.shape) == 4 and case.ll
    f = {"in_elems_past": max_offset(i) >= G, "in_bytes_past": max_offset(i) * i.isz >= G,
         "out_elems_past": max_offset(o) >= G, "out_bytes_past": max_offset(o) * o.isz >= G}
    if len(case.ins) > 1:  # conv_layer_any_shape's filter
        f["filter_elems_past"] = max_offset(case.ins[1]) >= G
        f["filter_bytes_past"] = max_offset(case.ins[1]) * case.ins[1].isz >= G
    if case.ll:
        f["idx32"] = ll_idx32(i, clip)
        d = frame_dims(i, clip)
        f["idx32_sum"] = d[1][0] * d[1][1] + d[2][0] * d[2][1] + (d[0][0] * d[0][1] if i.il else 0)
        f["in_frame_elems_past"] = frame_reach(i, clip, 3) >= G
        f["out_frame_elems_past"] = frame_reach(o, clip) >= G
        f["final_form"] = ll_final_form(case)
        if not i.il:
            f["in_span_below"] = ll_span(i, clip)
            f["out_span_below"] = ll_span(o, clip)
    return f


def check_shapes_ok(v):
    """hb_runtime.cu, check_shapes: each dimension's extent * |stride| and the product of extents at most 2^31 - 1."""
    return all(e * abs(s) < G for e, s in v.halide()) and int(np.prod(v.shape)) < G


def arena_bytes(case):
    views = case.ins + [case.out]
    for v in views:
        assert v.at + v.reach()[0] * v.isz >= 0, (case.id, "a view starts before the arena")
    return -(-max(v.at + (v.reach()[1] + 1) * v.isz for v in views) // 256) * 256


# ---- local_laplacian ------------------------------------------------------------------------------------------------

def ll_entry(u8, il, batch, J):
    """The entry point of a layout: the pyramid_levels forms when J != 8."""
    if J == 8:
        name = "local_laplacian" + ("_u8" if u8 else "") + ("_interleaved" if il else "") + ("_batch" if batch else "")
        fn = getattr(importlib.import_module("halide_b200.filters"), name)
        return lambda hb, ins, out: fn(ins[0], LL_LEVELS, LL_ALPHA, 1.0, out)
    name = ("local_laplacian_pyramid_levels" + ("_u8" if u8 else "") + ("_interleaved" if il else "") +
            ("_batch" if batch else ""))
    mod = "halide_b200.filters" if name == "local_laplacian_pyramid_levels" else "halide_b200.local_laplacian_depth"
    fn = getattr(importlib.import_module(mod), name)
    return lambda hb, ins, out: fn(ins[0], J, LL_LEVELS, LL_ALPHA, 1.0, out)


def ll_want(u8, J):
    """The oracle on each frame's first three channels (an input's fourth is never read), at depth J; 8-bit frames
    through to_u16 and to_u8."""
    def one(o, f):
        f = np.ascontiguousarray(f[:3])
        if u8:
            return convert(o.local_laplacian(convert(f, np.uint16), LL_LEVELS, LL_ALPHA, 1.0, pyramid_levels=J), np.uint8)
        return o.local_laplacian(f, LL_LEVELS, LL_ALPHA, 1.0, pyramid_levels=J)
    return lambda o, xs: np.stack([one(o, f) for f in xs[0]]) if xs[0].ndim == 4 else one(o, xs[0])


def ll_case(id, why, claims, vin, vout, form, J=8, force=0, seed=0):
    """A local_laplacian case; `form`: the final kernel's form it claims (ll_final_form)."""
    u8 = vin.dtype == np.uint8
    batch = len(vin.shape) == 4
    shape = vin.shape
    data = (lambda: [np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)]) if u8 else \
        (lambda: [u16_frame(shape, seed)])
    claims = dict(claims, final_form=form)
    return Case(id, [vin], vout, data, ll_entry(u8, vin.il, batch, J), why, claims, want=ll_want(u8, J),
                kernels=frozenset({"ll_level1", "ll_final2"}), force=force, ll=True)


def il_pitch(target, h, w, sy0):
    """(row stride, pixel pitch) of an interleaved 3-channel frame whose idx32 sum h * sy + 3 + w * px is exactly
    `target`, with the row stride the least from sy0 on that makes it so."""
    for sy in range(sy0, sy0 + 4 * w):
        r = target - 3 - h * sy
        if r % w == 0:
            return sy, r // w
    raise AssertionError("no pitch")


def ll_cases():
    cases = []
    H, W = 64, 96
    # Planar frames stored row-block by row-block: memory [y][c][x], a row stride near 2^31 / 64 and a small channel
    # stride, so the idx32 sum and final_form's spans land where each case needs them and the frame's last rows lie
    # close to 2^31 elements from its first.
    for dt, tag in ((np.uint16, "u16"), (np.uint8, "u8")):
        isz = np.dtype(dt).itemsize
        # idx32 sum exactly 2^31 - 1 (odd: an odd channel stride, so no aligned form)
        S, sc = 33554425, 149
        assert 64 * S + 3 * sc == G - 1
        cases.append(ll_case(f"{tag}_idx32_max", "idx32 sum 2^31 - 1: the level-1 kernel's 32-bit offsets, at the last "
                             "sum that takes them; unaligned strides: the general final kernel",
                             {"idx32": True, "idx32_sum": G - 1, "in_span_below": True},
                             View(dt, (3, H, W), (sc, S, 1), 0), View(dt, (3, H, W), (sc, S, 1), 512 * isz), "General",
                             seed=1))
        # idx32 false, final_form's input span below: a fourth input channel makes the difference
        S, sc = 33554416, 256
        assert 64 * S + 4 * sc == G and 64 * S + 3 * sc < G
        for force in (0, 64, 16):
            cases.append(ll_case(f"{tag}_idx32_off_span_below_f{force}",
                                 "idx32 sum exactly 2^31 (four channels): the level-1 kernel's 64-bit path; in_span and "
                                 "out_span 2^31 - 256, aligned: the final kernel's TMA (mask 0), non-TMA aligned "
                                 "(mask 64, its int products) and general (mask 16) forms",
                                 {"idx32": False, "idx32_sum": G, "in_span_below": True, "out_span_below": True},
                                 View(dt, (4, H, W), (sc, S, 1), 0), View(dt, (3, H, W), (sc, S, 1), 1024 * isz),
                                 {0: "AlignedTma", 64: "Aligned", 16: "General"}[force], force=force, seed=2))
        # out_span exactly 2^31 while the input's is below (and idx32 holds)
        So = 33554426
        assert 64 * So + 3 * 128 == G and 64 * S + 3 * sc < G
        for force in (0, 64):
            cases.append(ll_case(f"{tag}_out_span_at_f{force}", "out_span exactly 2^31, in_span below and idx32 holds: "
                                 "the general final kernel, whatever the mask",
                                 {"idx32": True, "in_span_below": True, "out_span_below": False},
                                 View(dt, (3, H, W), (sc, S, 1), 0), View(dt, (3, H, W), (128, So, 1), 1024 * isz),
                                 "General", force=force, seed=3))
    # uint16 only: the input span exactly 2^31 with an output below, and J = 5
    S, sc = 33554426, 128
    assert 64 * S + 3 * sc == G and 64 * (S - 2) + 3 * sc < G
    for force in (0, 64):
        cases.append(ll_case(f"u16_in_span_at_f{force}", "idx32 sum and in_span exactly 2^31 (even strides): the "
                             "level-1 kernel's 64-bit path and the general final kernel; out_span below",
                             {"idx32": False, "idx32_sum": G, "in_span_below": False, "out_span_below": True},
                             View(np.uint16, (3, H, W), (sc, S, 1), 0), View(np.uint16, (3, H, W), (sc, S - 2, 1), 1024),
                             "General", force=force, seed=4))
    S, sc = 33554416, 256
    for force in (0, 64):
        cases.append(ll_case(f"u16_J5_span_below_f{force}", "J = 5: idx32 holds (sum 2^31 - 256), both spans below "
                             "and aligned: the aligned final forms with offsets up to 2^31 - 2^25",
                             {"idx32": True, "in_span_below": True, "out_span_below": True},
                             View(np.uint16, (3, H, W), (sc, S, 1), 0), View(np.uint16, (3, H, W), (sc, S, 1), 2048),
                             {0: "AlignedTma", 64: "Aligned"}[force], J=5, force=force, seed=5))
    # Interleaved frames, memory [x][y][c]: a pixel pitch near 2^31 / W decides idx32 through in_w * px_in
    Wi = 95
    for target, side in ((G - 1, True), (G, False)):
        sy, px = il_pitch(target, H, Wi, 4)
        for dt, tag in ((np.uint16, "u16"), (np.uint8, "u8")):
            cases.append(ll_case(f"{tag}_il_idx32_{'max' if side else 'at'}",
                                 f"interleaved, idx32 sum {target - G:+d} from 2^31, in_w * px_in = {Wi * px}: the "
                                 f"level-1 kernel's {'32' if side else '64'}-bit path; the general interleaved final "
                                 "kernel (pitch > 4)", {"idx32": side, "idx32_sum": target},
                                 View(dt, (3, H, Wi), (1, sy, px), 0, il=True),
                                 View(dt, (3, H, Wi), (1, sy, px), (H * sy + 64) * np.dtype(dt).itemsize, il=True),
                                 "GeneralIL", seed=6 + side))
    # An interleaved batch (J = 5): frames 64 rows apart inside each pixel's column block, past 2^31 through the pitch
    # (frame 1's pixels halfway between frame 0's, the output's a quarter of the pitch after the input's)
    sy, px = il_pitch(G - 1, H, Wi, 4)
    sn = 44 * px + px // 2
    cases.append(ll_case("u16_il_batch_J5", "interleaved batch: idx32 holds per frame (sum 2^31 - 1), the second "
                         "frame's samples past 2^31 elements", {"idx32": True, "idx32_sum": G - 1, "in_elems_past": True,
                                                                 "out_elems_past": True},
                         View(np.uint16, (2, 3, H, Wi), (sn, 1, sy, px), 0, il=True),
                         View(np.uint16, (2, 3, H, Wi), (sn, 1, sy, px), (px // 4) * 2, il=True), "GeneralIL", J=5,
                         seed=8))
    # Planar batches: the channel planes 7e8 apart and the frames 1e9, so the last frame ends past 2^31 elements
    sy, sc, sn = 128, 700_000_000, 1_000_000_000
    for dt, tag, J, neg in ((np.uint16, "u16", 8, False), (np.uint8, "u8", 8, False), (np.uint16, "u16", 5, True),
                            (np.uint8, "u8", 10, True)):
        isz = np.dtype(dt).itemsize
        s = -sn if neg else sn
        at = sn * isz if neg else 0
        cases.append(ll_case(f"{tag}_batch_J{J}{'_reversed' if neg else ''}",
                             f"batch of 2, frame stride {s}: idx32 and both spans hold per frame, the "
                             f"{'first' if neg else 'last'} frame's elements past 2^31 from the buffer's first",
                             {"idx32": True, "in_span_below": True, "out_span_below": True, "in_elems_past": not neg,
                              "out_elems_past": not neg},
                             View(dt, (2, 3, H, W), (s, sc, sy, 1), at),
                             View(dt, (2, 3, H, W), (s, sc, sy, 1), at + 2 * H * sy * isz),
                             "Aligned" if neg else "AlignedTma", J=J, seed=9 + J))
    # Frames whose own elements pass 2^31: channel planes 7e8 + 1000 and rows 2e7 apart (plane c's rows fall 1000 c
    # elements after rows of plane 0), so a frame's last touched sample lies 2.66e9 elements from its first.  idx32 and
    # both spans are false: the level-1 kernel's 64-bit path and the general final kernel, whatever the mask.
    sy, sc = 20_000_000, 700_001_000
    for dt, tag in ((np.uint16, "u16"), (np.uint8, "u8")):
        isz = np.dtype(dt).itemsize
        for force in (0, 64, 16):
            cases.append(ll_case(f"{tag}_frame_past_f{force}", "input and output frames whose last samples lie 2.66e9 "
                                 "elements from their first: idx32 and both spans false, the 64-bit level-1 path and the "
                                 "general final kernel's 64-bit loads and stores",
                                 {"idx32": False, "in_span_below": False, "out_span_below": False,
                                  "in_frame_elems_past": True, "out_frame_elems_past": True},
                                 View(dt, (3, H, W), (sc, sy, 1), 0), View(dt, (3, H, W), (sc, sy, 1), 256 * isz),
                                 "General", force=force, seed=20 + force))
    # only one side past 2^31 within the frame; the other a dense frame 1e6 elements into the arena
    dense = (H * W, W, 1)
    cases.append(ll_case("u16_frame_past_in_only", "an input frame past 2^31 elements (idx32 and in_span false) into a "
                         "dense output (out_span below): the general final kernel's 64-bit loads",
                         {"idx32": False, "in_span_below": False, "out_span_below": True, "in_frame_elems_past": True,
                          "out_frame_elems_past": False},
                         View(np.uint16, (3, H, W), (sc, sy, 1), 0), View(np.uint16, (3, H, W), dense, 2_000_000),
                         "General", seed=30))
    for force in (0, 64):
        cases.append(ll_case(f"u16_frame_past_out_only_f{force}", "a dense input (idx32 and in_span hold) into an output "
                             "frame past 2^31 elements (out_span false): the level-1 kernel's 32-bit path and the "
                             "general final kernel's 64-bit stores",
                             {"idx32": True, "in_span_below": True, "out_span_below": False,
                              "in_frame_elems_past": False, "out_frame_elems_past": True},
                             View(np.uint16, (3, H, W), dense, 2_000_000), View(np.uint16, (3, H, W), (sc, sy, 1), 0),
                             "General", force=force, seed=31))
    # interleaved frames past 2^31 within the frame: pixels 2e7 and rows 2e7 + 8 apart (pixel (x, y) shares its block of
    # 2e7 with the pixels of x + y, 8 y elements in), the output 4 elements after the input
    for dt, tag in ((np.uint16, "u16"), (np.uint8, "u8")):
        isz = np.dtype(dt).itemsize
        cases.append(ll_case(f"{tag}_il_frame_past", "interleaved frames whose last samples lie 3.14e9 elements from "
                             "their first: idx32 false, the level-1 kernel's 64-bit path and the general interleaved "
                             "final kernel's 64-bit loads and stores",
                             {"idx32": False, "in_frame_elems_past": True, "out_frame_elems_past": True},
                             View(dt, (3, H, Wi), (1, 20_000_008, 20_000_000), 0, il=True),
                             View(dt, (3, H, Wi), (1, 20_000_008, 20_000_000), 4 * isz, il=True), "GeneralIL", seed=32))
    return cases


# ---- blur and stencil_chain -----------------------------------------------------------------------------------------

def clip_call(module, name, *scalars):
    fn = getattr(importlib.import_module(f"halide_b200.{module}"), name)
    return lambda hb, ins, out: fn(ins[0], *scalars, out)


def per_frame(one, nd):
    """want() of a clip or of one frame of nd axes: one(oracle, frame) over a clip's leading axis."""
    return lambda o, xs: np.stack([one(o, f) for f in xs[0]]) if xs[0].ndim > nd else one(o, xs[0])


def blur_route(vin, vout):
    """blur.cu: both bases 4-byte aligned and every row and frame stride even take the pair kernel."""
    pair = all(v.at % 4 == 0 and all(st % 2 == 0 for st in v.strides[:-1]) for v in (vin, vout))
    return frozenset({"blur3x3_u16_quad" if pair else "blur3x3_u16"})


def u16_cases():
    cases = []
    h, w = 48, 80
    # (frames 35 rows and 1000 elements apart: frame k + 1's rows fall between frame k's)
    sy, sn = 20_000_000, 700_001_000
    filters = [("blur", lambda o, f: o.blur(f), 2, "blur_video", "blur_batch", (), "halide_blur"),
               ("stencil_chain", lambda o, f: o.stencil_chain(f), 0, "stencil_chain_video", "stencil_chain_batch", (),
                "stencil_chain"),
               ("stencils7", lambda o, f: o.stencil_chain(f, stencils=7), 0, "stencil_chain_video",
                "stencil_chain_stencils_batch", (7,), "stencil_chain_stencils")]
    for k, (tag, one, grow, module, batch, scalars, single) in enumerate(filters):
        ish = (3, h + grow, w + grow)
        for name, s, at in (("even", sn, 0), ("odd", sn + 1, 0), ("reversed", -sn, 2 * sn * 2)):
            vin, vout = View(np.uint16, ish, (s, sy, 1), at), View(np.uint16, (3, h, w), (s, sy, 1), at + 256 * 2)
            kern = blur_route(vin, vout) if tag == "blur" else frozenset({"stencil_chain_window"})
            cases.append(Case(f"{tag}_batch_{name}", [vin], vout,
                              lambda ish=ish, k=k: [u16_frame(ish, 100 + k)], clip_call(module, batch, *scalars),
                              f"3 frames, row stride {sy}, {name} frame stride {s}: the allocation spans past 2^31 "
                              "elements, frames 2 and 3 (1 and 2 reversed) lie past 2^31 bytes",
                              {"in_elems_past": not name == "reversed", "in_bytes_past": True,
                               "out_elems_past": not name == "reversed"}, want=per_frame(one, 2), kernels=kern))
        # one frame, rows past 2^31 bytes (a single dimension cannot pass 2^31 elements)
        ish1 = (h + grow, w + grow)
        fn = getattr(importlib.import_module("halide_b200.filters"), single)
        vin, vout = View(np.uint16, ish1, (30_000_000, 1), 0), View(np.uint16, (h, w), (30_000_000, 1), 256 * 2)
        cases.append(Case(f"{tag}_rows_past_bytes", [vin], vout,
                          lambda ish1=ish1, k=k: [u16_frame(ish1, 110 + k)],
                          lambda hb, ins, out, fn=fn, scalars=scalars: fn(ins[0], *scalars, out),
                          "one frame, row stride 3e7: its last rows lie past 2^31 bytes",
                          {"in_bytes_past": True, "out_bytes_past": True}, want=per_frame(one, 2),
                          kernels=blur_route(vin, vout) if tag == "blur" else frozenset({"stencil_chain_window"})))
    return cases


# ---- bilateral_grid -------------------------------------------------------------------------------------------------

def bg_cases():
    from halide_b200 import filters
    cases = []
    h, w = 48, 80
    sy, sn = 20_000_000, 700_001_000
    cases.append(Case("bg_rows_past_bytes", [View(np.float32, (h, w), (sy, 1), 0)],
                      View(np.float32, (h, w), (sy, 1), 256 * 4), lambda: [dyadic((h, w), 120)],
                      lambda hb, ins, out: filters.bilateral_grid(ins[0], 0.1, out),
                      "float frame, row stride 2e7: rows past 2^31 bytes", {"in_bytes_past": True, "out_bytes_past": True},
                      want=lambda o, xs: o.bilateral_grid(xs[0], 0.1), kernels=KERNELS_8))
    cases.append(Case("bg_s5_rows_past_bytes", [View(np.float32, (h, w), (sy, 1), 0)],
                      View(np.float32, (h, w), (sy, 1), 256 * 4), lambda: [noise((h, w), 121)],
                      lambda hb, ins, out: filters.bilateral_grid_s_sigma(ins[0], 5, 0.1, out),
                      "float frame at S = 5, row stride 2e7: rows past 2^31 bytes",
                      {"in_bytes_past": True, "out_bytes_past": True},
                      want=lambda o, xs: o.bilateral_grid(xs[0], 0.1, s_sigma=5), kernels=KERNELS_S))
    for tag, gen, entry, scalars, one, kern in (
            ("float", lambda s, k: np.stack([dyadic(s[1:], k + i) for i in range(s[0])]), "bilateral_grid_batch", (0.1,),
             lambda o, f: o.bilateral_grid(f, 0.1), KERNELS_8),
            ("s5", lambda s, k: noise(s, k), "bilateral_grid_s_sigma_batch", (5, 0.1),
             lambda o, f: o.bilateral_grid(f, 0.1, s_sigma=5), KERNELS_S),
            ("u8", lambda s, k: np.random.default_rng(k).integers(0, 256, s, dtype=np.uint8), "bilateral_grid_u8_batch",
             (0.1,), None, KERNELS_8)):
        dt = np.uint8 if tag == "u8" else np.float32
        isz = np.dtype(dt).itemsize
        for rev in (False, True):
            s = -sn if rev else sn
            at = 2 * sn * isz if rev else 0
            cases.append(Case(f"bg_{tag}_batch{'_reversed' if rev else ''}", [View(dt, (3, h, w), (s, sy, 1), at)],
                              View(dt, (3, h, w), (s, sy, 1), at + 256 * isz),
                              lambda gen=gen, k=130 + len(cases): [gen((3, h, w), k)],
                              clip_call("bilateral_grid_video", entry, *scalars),
                              f"3 frames, frame stride {s}, row stride 2e7: "
                              f"{'frames 1 and 2 below the first, 1.4e9 elements away' if rev else 'elements past 2^31'}",
                              {"in_elems_past": not rev, "in_bytes_past": isz > 1 or not rev,
                               "out_elems_past": not rev},
                              want=per_frame(one, 2) if one else None, check=None if one else bg_u8_check,
                              kernels=kern))
    return cases


def bg_u8_check(hb, oracle, got, xs):
    """The 8-bit rule of test_bg_nl_u8_gpu.py and test_concurrent_callers_gpu.check_bg_u8, per frame: byte for byte
    to_u8 of the float filter on to_f32 of a dense copy of the frame; and the oracle's composition wherever the two float
    results agree, never more than 1 away elsewhere (bg_hist_blurz's re-association is exact only where every partial
    bin sum is, which v / 255 does not guarantee)."""
    from test_bg_nl_u8_gpu import float_path
    for k, x in enumerate(xs[0]):
        f = float_path(hb, "bg", x, (0.1,), x.shape)
        assert np.array_equal(got[k], convert(f, np.uint8)), f"frame {k}: differs from to_u8(bilateral_grid(to_f32(x)))"
        want_f = oracle.bilateral_grid(convert(x, np.float32), 0.1)
        want = convert(want_f, np.uint8)
        agree = f == want_f
        assert np.array_equal(got[k][agree], want[agree]), f"frame {k}: differs from the oracle where the floats agree"
        assert np.abs(got[k].astype(np.int16) - want).max() <= 1, f"frame {k}: more than 1 from the oracle"


# ---- nl_means -------------------------------------------------------------------------------------------------------

def nl_cases():
    from test_clip_entry_points_gpu import nl_u8
    cases = []
    h, w = 40, 56
    sy, sc, sn = 1_000_000, 600_000_000, 1_000_000_000
    for variant in (0, 1):
        vk = {"nl_means_window" if variant == 0 else "nl_means"}
        for tag, dt in (("f32", np.float32), ("u8", np.uint8)):
            isz = np.dtype(dt).itemsize
            gen = (lambda s, k: f32_frame(s, k)) if dt == np.float32 else \
                (lambda s, k: np.random.default_rng(k).integers(0, 256, s, dtype=np.uint8))
            one = (lambda o, f: o.nl_means(f, 3, 7, 0.12)) if dt == np.float32 else (lambda o, f: nl_u8(o, f, 3, 7, 0.12))
            entry = "nl_means_batch" if dt == np.float32 else "nl_means_u8_batch"
            cases.append(Case(f"nl_{tag}_batch_v{variant}", [View(dt, (2, 3, h, w), (sn, sc, sy, 1), 0)],
                              View(dt, (2, 3, h, w), (sn, sc, sy, 1), 256 * isz),
                              lambda gen=gen, k=140 + len(cases): [gen((2, 3, h, w), k)],
                              clip_call("nl_means_video", entry, 3, 7, 0.12),
                              f"planar batch, channel stride {sc}, frame stride {sn}: the second frame's planes 1 and 2 "
                              "lie past 2^31 elements", {"in_elems_past": True, "out_elems_past": True},
                              want=per_frame(one, 3), kernels=frozenset(vk), variant=variant))
            # interleaved one frame: the pixel pitch takes the last column past 2^31 elements
            px = 38_000_000
            ientry = "nl_means_interleaved" if dt == np.float32 else "nl_means_u8_interleaved"
            cases.append(Case(f"nl_{tag}_il_v{variant}", [View(dt, (3, h, w), (1, 4, px), 0, il=True)],
                              View(dt, (3, h, w), (1, 4, px), 4 * h * isz + 64, il=True),
                              lambda gen=gen, k=150 + len(cases): [gen((3, h, w), k)],
                              clip_call("nl_means_video", ientry, 3, 7, 0.12),
                              f"interleaved frame, pixel pitch {px}: the last columns 2.09e9 elements away, past 2^31 "
                              "bytes for float", {"in_bytes_past": isz > 1, "out_bytes_past": isz > 1},
                              want=lambda o, xs, one=one: one(o, xs[0]),
                              kernels=frozenset(vk), variant=variant))
    # an interleaved float batch: pitch and frame stride together past 2^31 elements
    px = 22_000_000
    cases.append(Case("nl_f32_il_batch", [View(np.float32, (2, 3, h, w), (1_000_000_000, 1, 4, px), 0, il=True)],
                      View(np.float32, (2, 3, h, w), (1_000_000_000, 1, 4, px), 4 * h * 4 + 64, il=True),
                      lambda: [f32_frame((2, 3, h, w), 160)], clip_call("nl_means_video", "nl_means_interleaved_batch",
                                                                          5, 9, 0.3),
                      "interleaved batch, pixel pitch 2.2e7 and frame stride 1e9: the second frame past 2^31 elements",
                      {"in_elems_past": True, "out_elems_past": True},
                      want=per_frame(lambda o, f: o.nl_means(f, 5, 9, 0.3), 3), kernels=frozenset({"nl_means"})))
    return cases


# ---- camera_pipe ----------------------------------------------------------------------------------------------------

def cp_call(name):
    def call(hb, ins, out):
        m32, m70 = hb.HalideBuffer.from_numpy(CP_M3200.copy()), hb.HalideBuffer.from_numpy(CP_M7000.copy())
        getattr(hb.filters, name)(ins[0], m32, m70, *CP, out)
    return call


def cp_want(o, xs):
    one = lambda f: o.camera_pipe(f, CP_M3200, CP_M7000, *CP, (3, 64, 96))  # noqa: E731
    return np.stack([one(f) for f in xs[0]]) if xs[0].ndim == 3 else one(xs[0])


def cp_cases():
    rh, rw = 100, 140
    cases = [Case("cp_planar", [View(np.uint16, (rh, rw), (21_000_000, 1), 0)],
                  View(np.uint8, (3, 64, 96), (700_000_000, 21_000_000, 1), 4096), lambda: [raw_frame(rh, rw, 170)],
                  cp_call("camera_pipe"), "raw rows 2.1e7 apart (past 2^31 bytes); uint8 planes 7e8 apart, the last "
                  "samples past 2^31 elements", {"in_bytes_past": True, "out_elems_past": True}, want=cp_want,
                  kernels=frozenset({"camera_pipe"})),
             Case("cp_burst", [View(np.uint16, (2, rh, rw), (1_000_000_000, 10_000_000, 1), 0)],
                  View(np.uint8, (2, 3, 64, 96), (1_000_000_000, 300_000_100, 10_000_000, 1), 4096),
                  lambda: [np.stack([raw_frame(rh, rw, 171 + k) for k in range(2)])], cp_call("camera_pipe_batch"),
                  "raw burst, frames 1e9 apart: the second past 2^31 bytes; the uint8 output's second frame past 2^31 "
                  "elements", {"in_bytes_past": True, "out_elems_past": True}, want=cp_want,
                  kernels=frozenset({"camera_pipe"})),
             Case("cp_il_burst", [View(np.uint16, (2, rh, rw), (1_000_000_000, 10_000_000, 1), 0)],
                  View(np.uint8, (2, 3, 64, 96), (1_000_000_500, 1, 20_000_000, 4), 4096, il=True),
                  lambda: [np.stack([raw_frame(rh, rw, 173 + k) for k in range(2)])],
                  cp_call("camera_pipe_interleaved_batch"), "raw burst past 2^31 bytes; an RGBA-pitch interleaved "
                  "output with rows 2e7 apart whose second frame lies past 2^31 elements (alpha untouched)",
                  {"in_bytes_past": True, "out_elems_past": True}, want=cp_want,
                  kernels=frozenset({"camera_pipe_il"})),
             Case("cp_il", [View(np.uint16, (rh, rw), (21_000_000, 1), 0)],
                  View(np.uint8, (3, 64, 96), (1, 8, 22_000_000), 4096, il=True), lambda: [raw_frame(rh, rw, 175)],
                  cp_call("camera_pipe_interleaved"), "raw rows past 2^31 bytes; an interleaved output whose pixels "
                  "are 2.2e7 apart, its last columns past 2^31 - 2^26 elements",
                  {"in_bytes_past": True, "out_elems_past": False, "out_bytes_past": False}, want=cp_want,
                  kernels=frozenset({"camera_pipe_il"}))]
    return cases


# ---- conv_layer_any_shape -------------------------------------------------------------------------------------------

def conv_cases():
    n, ci, co, w, h = 2, 8, 16, 24, 20
    sn, sy = 1_070_000_000, 53_000_000
    inp = View(np.float32, (n, h + 2, w + 2, ci), (sn, sy, ci, 1), 0)
    out = View(np.float32, (n, h, w, co), (1_073_000_000, 58_000_000, co, 1), 256 * 4)
    filt = View(np.float32, (ci, 3, 3, co), (200_000_000, 380_000_000, co, 1), 4096 * 4 + 1_000_000 * 4)
    bias = View(np.float32, (co,), (1,), 8192 * 4 + 1_000_000 * 4)

    def data():
        return list(harness("signed", (n, ci, co, w, h)))

    def check(hb, oracle, got, xs):
        r = worst_ratio(got, *xs)
        assert r <= 1.0, f"error {r:.3g} x the derived bound"

    def call(hb, ins, out_b):
        hb.filters.conv_layer_any_shape(ins[0], ins[1], ins[2], out_b)
    return [Case("conv_any_shape", [inp, filt, bias], out, data, call,
                 "input and output frames 1.07e9 apart, rows 5.3e7 and 5.8e7 apart: both past 2^31 elements; the filter's "
                 "input-channel and ky strides take it past 2^31 elements", {"in_elems_past": True, "out_elems_past": True,
                                                                           "filter_elems_past": True},
                 check=check)]


CASES = ll_cases() + u16_cases() + bg_cases() + nl_cases() + cp_cases() + conv_cases()
assert len({c.id for c in CASES}) == len(CASES)


# ---- the CPU check ---------------------------------------------------------------------------------------------------

def test_cases_sit_where_they_claim():
    """Every case is on the side of each rule its description claims, passes check_shapes' per-dimension limits, keeps
    its frames small, and its views are disjoint and fit an arena of at most ARENA_CAP bytes.  (A case that claims
    idx32_sum gives the exact sum.)"""
    assert len(CASES) >= 50, len(CASES)
    for c in CASES:
        f = facts(c)
        for rule, side in c.claims.items():
            assert f[rule] == side, (c.id, rule, f[rule], side)
        views = c.ins + [c.out]
        for v in views:
            assert check_shapes_ok(v), (c.id, v)
            frame = v.shape[1:] if len(v.shape) == 4 else v.shape
            assert int(np.prod(frame)) <= FRAME_CAP, (c.id, v.shape)
            assert v.at % v.isz == 0
        assert arena_bytes(c) <= ARENA_CAP, (c.id, arena_bytes(c) / 2 ** 30)
        sets = [v.byte_set() for v in views]
        for a in range(len(sets)):
            for b in range(a + 1, len(sets)):
                assert not np.intersect1d(sets[a], sets[b]).size, (c.id, "views overlap", a, b)
    # both sides of each line are covered
    ll = [facts(c) for c in CASES if c.ll]
    assert {f["idx32"] for f in ll} == {True, False}
    assert {f["idx32_sum"] for f in ll} >= {G - 1, G}
    llc = [c for c in CASES if c.ll]
    planar = [f for f, c in zip(ll, llc) if not c.ins[0].il]
    assert {(f["in_span_below"], f["out_span_below"]) for f in planar} >= {(True, True), (True, False), (False, True),
                                                                           (False, False)}
    assert {f["final_form"] for f in ll} >= {"AlignedTma", "Aligned", "General", "GeneralIL"}
    # samples past 2^31 elements within one frame, on the 64-bit side of each rule, planar and interleaved, every mask
    assert any(not f["idx32"] and f["in_frame_elems_past"] for f in ll)
    assert any(not f["in_span_below"] and f["in_frame_elems_past"] for f in planar)
    assert any(not f["out_span_below"] and f["out_frame_elems_past"] for f in planar)
    assert any(c.ins[0].il and f["in_frame_elems_past"] and f["out_frame_elems_past"] for f, c in zip(ll, llc))
    assert {c.force for f, c in zip(ll, llc) if f["in_frame_elems_past"] and f["out_frame_elems_past"]} >= {0, 64, 16}


# ---- the GPU run -----------------------------------------------------------------------------------------------------

def torch_view(arena, v):
    """(a torch view of v with non-negative strides, the axes to flip for the logical order)."""
    import torch
    tdt = {np.dtype(np.uint16): torch.int16, np.dtype(np.uint8): torch.uint8,
           np.dtype(np.float32): torch.float32}[np.dtype(v.dtype)]
    typed = arena.view(tdt)
    lo = v.reach()[0]
    start = v.at // v.isz + lo
    t = torch.as_strided(typed, v.shape, tuple(abs(s) for s in v.strides), start)
    return t, tuple(k for k, s in enumerate(v.strides) if s < 0)


def host_of(t, flip, dtype):
    a = t.cpu().numpy()
    a = np.flip(a, flip) if flip else a
    return np.ascontiguousarray(a).view(dtype)


def wrap(hb, t, v, flip):
    """A device-resident HalideBuffer of v: its first element and Halide strides (negative ones included)."""
    d = v.halide()
    b = hb.HalideBuffer(v.dtype, [e for e, _ in d], [s for _, s in d], v.mins)
    ptr = t.data_ptr() - v.reach()[0] * v.isz
    b._keep = t
    hb.lib.check(hb.capi.halide_cuda_wrap_device_ptr(None, ctypes.byref(b.buf), ctypes.c_uint64(ptr)))
    b._wrapped = True
    return b


def first_stray(arena, pattern):
    """Byte offset of the first arena byte that is not the sentinel, or None (in chunks of 1 GiB)."""
    import torch
    words = arena.view(torch.int64)
    chunk = 1 << 27
    for i in range(0, words.numel(), chunk):
        c = words[i:i + chunk]
        bad = c != pattern
        if bool(bad.any()):
            k = int(bad.nonzero()[0, 0])
            row = c[k:k + 1].view(torch.uint8).cpu().numpy()
            return 8 * (i + k) + int(np.argmax(row != SENTINEL))
    return None


def run_in_arena(hb, case, xs, need):
    """The case's call on views of a fresh sentinel arena: (the output read back, the launches, what went wrong with the
    input or the bytes around the output).  Every device reference is dropped before returning or raising, so the arena
    is freed even when the call fails and a traceback keeps this frame."""
    import torch
    l = hb.load_library()
    arena = t = to = bo = ins = None
    problems = []
    try:
        arena = torch.empty(need, dtype=torch.uint8, device="cuda")
        assert arena.data_ptr() % ARENA_ALIGN == 0, "ll_final_form assumes an aligned arena"
        arena.fill_(SENTINEL)
        ins = []
        for v, x in zip(case.ins, xs):
            t, flip = torch_view(arena, v)
            x = np.ascontiguousarray(np.flip(x, flip) if flip else x)
            t.copy_(torch.from_numpy(x.view({1: np.uint8, 2: np.int16, 4: np.float32}[v.isz])).cuda())
            ins.append((t, flip, wrap(hb, t, v, flip)))
        to, oflip = torch_view(arena, case.out)
        bo = wrap(hb, to, case.out, oflip)
        l.halide_b200_ll_force_generic(case.force)
        try:
            with nl_means_variant(hb, case.variant), kernels_run(hb) as ran:
                case.call(hb, [b for _, _, b in ins], bo)
                torch.cuda.synchronize()
        finally:
            l.halide_b200_ll_force_generic(0)
        got = host_of(to, oflip, case.out.dtype)
        for (t, flip, _), v, x in zip(ins, case.ins, xs):
            if not np.array_equal(host_of(t, flip, v.dtype), x):
                problems.append(f"{case.id}: the call changed its input")
        # everything the views describe back to the sentinel, then the whole arena must be the sentinel
        for t in [t for t, _, _ in ins] + [to]:
            t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).fill_(
                {1: SENTINEL, 2: np.int16(np.uint16(0xA5A5)).item(), 4: np.int32(np.uint32(0xA5A5A5A5)).item()}[
                    t.element_size()])
        stray = first_stray(arena, np.int64(np.uint64(0xA5A5A5A5A5A5A5A5)).item())
        if stray is not None:
            problems.append(f"{case.id}: byte {stray} of the arena, outside the output's elements, was written")
        return got, ran, problems
    finally:
        arena = t = to = bo = ins = None
        gc.collect()
        torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def peak():
    import torch
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"\nwide offsets: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_wide_offsets(hb, oracle, peak, case):
    """The case's call on strided views of a sentinel arena against its oracle rule (the case's `why` says which side
    of which rule it is on); the input unchanged, every byte outside the output's elements still the sentinel."""
    import torch
    need = arena_bytes(case)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need + (1 << 30):
        pytest.skip(f"{case.id}: needs {need / 2 ** 30:.1f} GiB of device memory and {free / 2 ** 30:.1f} GiB is free "
                    "(the device is shared)")
    xs = case.data()
    got, ran, problems = run_in_arena(hb, case, xs, need)
    assert not problems, problems
    assert case.kernels <= set(ran), f"{case.id}: launched {sorted(ran)}, missing {sorted(case.kernels - set(ran))}"
    if case.check is not None:
        case.check(hb, oracle, got, xs)
    else:
        want = case.want(oracle, xs)
        assert got.shape == want.shape, (got.shape, want.shape)
        bad = got != want if got.dtype != np.float32 else got.view(np.uint32) != want.view(np.uint32)
        assert not bad.any(), (f"{case.id}: {int(bad.sum())} of {got.size} samples differ from the oracle, first at "
                               f"{tuple(np.argwhere(bad)[0])}")
