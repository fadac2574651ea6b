"""camera_pipe bit for bit against the oracle where a tiled stencil kernel can be wrong while dense, generously padded
frames stay right.

- Raw buffers that are exactly the filter's bounds query, at every Bayer parity of the output origin: a tile that
  consumed one of the clamped coordinates of its raw tile load would read a wrong value here, not a neighbour's.
- Outputs with padded and odd row pitches, misaligned bases, gaps between planes and channel crops, on the device and on
  the host: the unsharp stage's 32-bit and byte stores, and its relative-to-absolute channel mapping.  Every byte the
  output does not cover must keep its sentinel.
- Raw and matrix buffers with pitches, mins and strides far from the dense defaults.
- Every scalar at its extremes, with the whole 1024-entry tone curve read back out of the frame.
- Row bands cut to the filter's own bounds query, a 7680 x 4320 frame at its corners and tile seams, and back-to-back
  calls with different tables."""
import numpy as np
import pytest
from numpy.lib.stride_tricks import as_strided

from util import CP_EXTREMES, CP_M3200, CP_M7000, cp_matrix_q88, cp_param_id, cp_params, kernels_run

pytestmark = pytest.mark.gpu
HOT = 60000  # a hot pixel: the denoise clamps it to the largest of its four same-colour neighbours
OUT_OF_BOUNDS = -4  # halide_error_code_access_out_of_bounds
DEFAULT = cp_params({})


def raw_frame(h, w, seed, bits=10, hot=1e-3):
    """Smooth content plus noise with a few hot pixels (float32 arithmetic, so that 8K frames stay cheap)."""
    rng = np.random.default_rng(seed)
    f = np.float32
    xx, yy = np.arange(w, dtype=f)[None, :], np.arange(h, dtype=f)[:, None]
    base = f(400) + f(300) * (np.sin(xx / f(23)) * np.cos(yy / f(17)))
    noise = rng.integers(0, 1 << bits, (h, w), dtype=np.uint16)
    raw = np.clip(f(0.5) * base + f(0.5) * noise, 0, (1 << bits) - 1).astype(np.uint16)
    n = max(4, int(h * w * hot))
    raw[rng.integers(0, h, n), rng.integers(0, w, n)] = HOT
    return raw


def mats(hb, m32=CP_M3200, m70=CP_M7000):
    return hb.HalideBuffer.from_numpy(m32.copy()), hb.HalideBuffer.from_numpy(m70.copy())


def out_desc(hb, shape, mins):
    return hb.HalideBuffer.from_numpy(np.zeros(shape, np.uint8), mins, host_dirty=False)


def run(hb, raw, out_shape, params=DEFAULT, in_mins=None, out_mins=None, m32=CP_M3200, m70=CP_M7000):
    out = np.zeros(out_shape, np.uint8)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.camera_pipe(hb.HalideBuffer.from_numpy(raw, in_mins), *mats(hb, m32, m70), *params, bo)
    bo.copy_to_host()
    return out


def ref(oracle, raw, out_shape, params=DEFAULT, in_mins=None, out_mins=None, m32=CP_M3200, m70=CP_M7000, **kw):
    return oracle.camera_pipe(raw, m32, m70, *params, out_shape, in_mins=in_mins, out_mins=out_mins, **kw)


def same(got, want, what="result"):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} of {got.size} bytes differ, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]}, want {want[tuple(bad[0])]}")


def need_region(hb, out_buf, params=DEFAULT):
    """(x0, y0, w, h) of the raw region camera_pipe reads for the output region `out_buf` describes (bounds query)."""
    q = hb.HalideBuffer.bounds_query(np.uint16, 2)
    hb.filters.camera_pipe(q, *mats(hb), *params, out_buf)
    (x0, w, _), (y0, h, _) = q.shape()
    return x0, y0, w, h


# ---- 1. tight inputs at every Bayer parity -------------------------------------------------------------------------
# One raw frame in absolute coordinates, and one GPU call over an output region that holds every tight case below.
WORLD_RAW_MINS = (-40, -20)
WORLD_OUT_MINS, WORLD_OUT_SHAPE = (-40, -20, 0), (3, 120, 192)
ORIGINS = [(0, 0), (-37, -11), (7, 4), (-6, 3)]  # (x, y) parities (even, even), (odd, odd), (odd, even), (even, odd)
WIDTHS = [1, 2, 3, 4, 5, 63, 64, 65, 130]
HEIGHTS = [1, 2, 31, 32, 33, 70]


@pytest.fixture(scope="module")
def world(hb):
    raw = raw_frame(150, 230, 1)
    return raw, run(hb, raw, WORLD_OUT_SHAPE, in_mins=WORLD_RAW_MINS, out_mins=WORLD_OUT_MINS)


def world_crop(hb, world, ox, oy, w, h, trim=None):
    """The exact raw region of output (ox, oy, w, h), cut out of the world frame with its mins, optionally one short on
    side `trim`."""
    raw, _ = world
    x0, y0, qw, qh = need_region(hb, out_desc(hb, (3, h, w), (ox, oy, 0)))
    if trim == "left":
        x0, qw = x0 + 1, qw - 1
    elif trim == "right":
        qw -= 1
    elif trim == "top":
        y0, qh = y0 + 1, qh - 1
    elif trim == "bottom":
        qh -= 1
    ax, ay = x0 - WORLD_RAW_MINS[0], y0 - WORLD_RAW_MINS[1]
    assert ax >= 0 and ay >= 0 and ay + qh <= raw.shape[0] and ax + qw <= raw.shape[1]
    return np.ascontiguousarray(raw[ay:ay + qh, ax:ax + qw]), (x0, y0)


def test_world_matches_oracle(oracle, world):
    raw, whole = world
    same(whole, ref(oracle, raw, WORLD_OUT_SHAPE, in_mins=WORLD_RAW_MINS, out_mins=WORLD_OUT_MINS))


@pytest.mark.parametrize("h", HEIGHTS)
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("ox,oy", ORIGINS)
def test_tight_input(hb, oracle, world, ox, oy, w, h):
    """A raw buffer of exactly the bounds-query region: equal to the oracle on the same buffer and to the matching crop
    of the whole-frame call."""
    tight, in_mins = world_crop(hb, world, ox, oy, w, h)
    shape, mins = (3, h, w), (ox, oy, 0)
    got = run(hb, tight, shape, in_mins=in_mins, out_mins=mins)
    same(got, ref(oracle, tight, shape, in_mins=in_mins, out_mins=mins), "against the oracle")
    wx, wy = ox - WORLD_OUT_MINS[0], oy - WORLD_OUT_MINS[1]
    assert wx >= 0 and wy >= 0 and wx + w <= WORLD_OUT_SHAPE[2] and wy + h <= WORLD_OUT_SHAPE[1]
    same(got, world[1][:, wy:wy + h, wx:wx + w], "against the whole-frame call")


@pytest.mark.parametrize("side", ["left", "right", "top", "bottom"])
@pytest.mark.parametrize("ox,oy", ORIGINS)
def test_one_short_is_rejected(hb, world, ox, oy, side):
    """The bounds-query region less one column or row on any side: -4, and nothing launched."""
    from halide_b200 import HalideError
    for w, h in [(1, 1), (65, 33)]:
        short, in_mins = world_crop(hb, world, ox, oy, w, h, trim=side)
        with kernels_run(hb) as ran, pytest.raises(HalideError) as e:
            run(hb, short, (3, h, w), in_mins=in_mins, out_mins=(ox, oy, 0))
        assert e.value.code == OUT_OF_BOUNDS and not ran, (e.value.code, sorted(ran))


# ---- 2. output layouts, channel crops, input layouts ---------------------------------------------------------------
LAYOUT_RAW_MINS = (1001, -37)
LAYOUT_OUT_MINS = (995, -39)
LH, LW = 37, 93  # two tile rows, and a last tile column of 29 pixels (7 whole 4-pixel groups and one partial)
CROPS = [(0, 3), (0, 1), (1, 3), (2, 3), (0, 2)]


@pytest.fixture(scope="module")
def layout_raw(hb):
    raw = raw_frame(80, 140, 2)
    x0, y0, w, h = need_region(hb, out_desc(hb, (3, LH, LW), LAYOUT_OUT_MINS + (0,)))
    ax, ay = x0 - LAYOUT_RAW_MINS[0], y0 - LAYOUT_RAW_MINS[1]
    assert ax >= 0 and ay >= 0 and ax + w <= raw.shape[1] and ay + h <= raw.shape[0]
    return raw


def planes(pitch, gap, off):
    """A 3-plane uint8 layout of LH x LW: rows `pitch` bytes apart, planes LH * pitch + gap apart (more than a plane),
    the first sample `off` bytes into the allocation.  Returns (allocation size, strides)."""
    ps = LH * pitch + gap
    return off + 2 * ps + (LH - 1) * pitch + LW + 5, (ps, pitch, 1)


def expect_planes(size, off, strides, crop, want, sentinel):
    """The whole allocation as it must be after the call: `want` in the cropped planes, the sentinel everywhere else."""
    expect = np.full(size, sentinel, np.uint8)
    as_strided(expect[off:], (3, LH, LW), strides)[crop[0]:crop[1]] = want
    return expect


def crop_id(crop):
    return f"c[{crop[0]},{crop[1]})"


@pytest.mark.parametrize("crop", CROPS, ids=crop_id)
@pytest.mark.parametrize("off", [0, 1, 2, 3])
@pytest.mark.parametrize("pad", [1, 3])
def test_device_output_layout(hb, oracle, layout_raw, pad, off, crop):
    """Device-resident torch views with row pitch W + pad, base `off` bytes past a 512-byte boundary and a 5-byte gap
    between planes: rows start at every alignment mod 4, so each row's 4-pixel groups take either the 32-bit stores or
    the byte stores, and the last partial group always the byte stores.  Run twice, over 0x00 and over 0xFF."""
    import torch
    c0, c1 = crop
    shape, mins = (c1 - c0, LH, LW), LAYOUT_OUT_MINS + (c0,)
    want = ref(oracle, layout_raw, shape, in_mins=LAYOUT_RAW_MINS, out_mins=mins)
    size, strides = planes(LW + pad, 5, off)
    for sentinel in (0x00, 0xFF):
        backing = torch.full((size,), sentinel, dtype=torch.uint8, device="cuda")
        view = backing.as_strided((3, LH, LW), strides, off)[c0:c1]
        hb.filters.camera_pipe(hb.HalideBuffer.from_numpy(layout_raw, LAYOUT_RAW_MINS), *mats(hb), *DEFAULT,
                               hb.HalideBuffer.from_torch(view, mins))
        torch.cuda.synchronize()
        same(backing.cpu().numpy(), expect_planes(size, off, strides, crop, want, sentinel), f"sentinel {sentinel:#x}")


@pytest.mark.parametrize("crop", CROPS, ids=crop_id)
def test_host_output_channel_crops(hb, oracle, layout_raw, crop):
    """The same crops of a padded host array: the device copy and the copy back touch only the cropped planes' rows."""
    c0, c1 = crop
    shape, mins = (c1 - c0, LH, LW), LAYOUT_OUT_MINS + (c0,)
    want = ref(oracle, layout_raw, shape, in_mins=LAYOUT_RAW_MINS, out_mins=mins)
    off = 1
    size, strides = planes(LW + 3, 7, off)
    for sentinel in (0x00, 0xFF):
        backing = np.full(size, sentinel, np.uint8)
        view = as_strided(backing[off:], (3, LH, LW), strides)[c0:c1]
        bo = hb.HalideBuffer.from_numpy(view, mins, host_dirty=False)
        hb.filters.camera_pipe(hb.HalideBuffer.from_numpy(layout_raw, LAYOUT_RAW_MINS), *mats(hb), *DEFAULT, bo)
        bo.copy_to_host()
        same(backing, expect_planes(size, off, strides, crop, want, sentinel), f"sentinel {sentinel:#x}")


JUNK = 7.5  # around the matrices: any read of it changes the result


def raw_arg(hb, kind, raw):
    """(buffer, the array the oracle reads) for `raw` as a view into wider rows: padded (pitch + 8) or odd (+ 3), two
    columns in, junk around it; on the host or the device."""
    import torch
    h, w = raw.shape
    assert w % 2 == 0
    backing = np.full((h, w + (8 if kind.endswith("padded") else 3)), 0xFFFF, np.uint16)
    backing[:, 2:2 + w] = raw
    view = backing[:, 2:2 + w]
    if kind.startswith("host"):
        return hb.HalideBuffer.from_numpy(view, LAYOUT_RAW_MINS), view
    return hb.HalideBuffer.from_torch(torch.from_numpy(backing).cuda()[:, 2:2 + w], LAYOUT_RAW_MINS), view


def matrix_arg(hb, kind, m):
    """(buffer, the array the oracle reads, its mins) for the 3 x 4 matrix m: dense on the host; at (0..3, 0..2) of a
    6 x 5 host buffer with mins (-1, -1) and junk around it; or columns 0..3 of a (3, 8) CUDA tensor (row stride 8)."""
    import torch
    if kind == "dense":
        return hb.HalideBuffer.from_numpy(m.copy()), m, None
    if kind == "offset":
        a = np.full((5, 6), JUNK, np.float32)
        a[1:4, 1:5] = m
        return hb.HalideBuffer.from_numpy(a, (-1, -1)), a, (-1, -1)
    t = torch.full((3, 8), JUNK, dtype=torch.float32, device="cuda")
    t[:, :4] = torch.from_numpy(m)
    return hb.HalideBuffer.from_torch(t[:, :4]), m, None


@pytest.mark.parametrize("m32_kind,m70_kind", [("dense", "dense"), ("offset", "offset"), ("device", "device"),
                                               ("device", "offset")])
@pytest.mark.parametrize("raw_kind", ["host_padded", "host_odd", "device_padded", "device_odd"])
def test_input_layouts(hb, oracle, layout_raw, raw_kind, m32_kind, m70_kind):
    """Raw rows with padded and odd pitches at mins (1001, -37), and matrices away from dense buffers at (0, 0)."""
    shape, mins = (3, LH, LW), LAYOUT_OUT_MINS + (0,)
    bi, raw_view = raw_arg(hb, raw_kind, layout_raw)
    b32, m32, m32_mins = matrix_arg(hb, m32_kind, CP_M3200)
    b70, m70, m70_mins = matrix_arg(hb, m70_kind, CP_M7000)
    out = np.zeros(shape, np.uint8)
    bo = hb.HalideBuffer.from_numpy(out, mins, host_dirty=False)
    hb.filters.camera_pipe(bi, b32, b70, *DEFAULT, bo)
    bo.copy_to_host()
    want = ref(oracle, raw_view, shape, in_mins=LAYOUT_RAW_MINS, out_mins=mins, m32=m32, m70=m70, m3200_mins=m32_mins,
               m7000_mins=m70_mins)
    same(out, want)
    same(out, ref(oracle, layout_raw, shape, in_mins=LAYOUT_RAW_MINS, out_mins=mins), "against the dense buffers")


# ---- 3. parameters at their extremes -------------------------------------------------------------------------------
@pytest.mark.parametrize("overrides", [{}] + CP_EXTREMES, ids=cp_param_id)
def test_parameter_extremes(hb, oracle, overrides):
    params = cp_params(overrides)
    cp_matrix_q88(CP_M3200, CP_M7000, params[0])  # asserts the matrix stays where Halide defines the result
    raw = raw_frame(88, 160, 7)
    shape = (3, 64, 128)
    same(run(hb, raw, shape, params), ref(oracle, raw, shape, params))


# Large but legal entries: with 16-bit raw noise the demosaiced i16 values go negative and the curve index clamps at
# both ends (at 3700 K |Q8.8| reaches 29 445 and a row's magnitudes sum to 59 202; cp_matrix_q88 checks both limits).
M_LARGE_3200 = np.array([[60, -30, 30, -100], [-30, 60, -30, 100], [30, -30, 60, -100]], np.float32)
M_LARGE_7000 = np.array([[50, -35, 25, -110], [-25, 55, -35, 90], [35, -25, 55, -120]], np.float32)


@pytest.mark.parametrize("sharpen", [1.0, 100.0])
def test_full_range_raw_with_large_matrix(hb, oracle, sharpen):
    params = cp_params(dict(sharpen=sharpen))
    q = cp_matrix_q88(M_LARGE_3200, M_LARGE_7000, params[0])
    assert np.abs(q).max() > 1 << 14 and np.abs(q).sum(axis=1).min() > 1 << 15
    raw = np.random.default_rng(9).integers(0, 65536, (120, 200), dtype=np.uint16)
    shape = (3, 96, 160)
    got = run(hb, raw, shape, params, m32=M_LARGE_3200, m70=M_LARGE_7000)
    same(got, ref(oracle, raw, shape, params, m32=M_LARGE_3200, m70=M_LARGE_7000))
    assert (got == 0).any() and (got == 255).any()


# ---- 4. the whole tone curve read out of a frame -------------------------------------------------------------------
# Both matrices diag(1.001), offsets 0: Q8.8 exactly 256 on the diagonal whatever alpha's rounding, so a pixel whose
# whole footprint is one raw value v demosaics to r = g = b = v, has an unsharp mask of 0, and comes out as curve[v].
DIAG = np.eye(3, 4, dtype=np.float32) * np.float32(1.001)
PATCH, GRID = 24, 32  # 32 x 32 constant patches of 24 x 24: a 768 x 768 output


@pytest.fixture(scope="module")
def patches():
    """Raw frame of one constant patch per value 0..1023, in a seeded order (so neighbouring patches differ a lot and the
    unsharp mask is busy at their edges), with each value's patch centre in output coordinates.  Patch edges fall on
    even raw coordinates; a centre is 11 px or more from its patch's edges, the footprint of an output pixel 8 px."""
    order = np.random.default_rng(8).permutation(GRID * GRID)
    n = PATCH * GRID
    px = np.clip(np.arange(-16, n + 16) // PATCH, 0, GRID - 1)  # raw column c holds shifted x = c - 16
    py = np.clip(np.arange(-12, n + 12) // PATCH, 0, GRID - 1)  # raw row r holds shifted y = r - 12
    raw = order[py[:, None] * GRID + px[None, :]].astype(np.uint16)
    cy, cx = np.divmod(np.argsort(order), GRID)
    return raw, PATCH * cx + PATCH // 2, PATCH * cy + PATCH // 2


@pytest.mark.parametrize("overrides", [{}] + CP_EXTREMES, ids=cp_param_id)
def test_tone_curve_readout(hb, oracle, patches, overrides):
    raw, cx, cy = patches
    params = cp_params(overrides)
    assert np.array_equal(cp_matrix_q88(DIAG, DIAG, params[0]), 256 * np.eye(3, 4, dtype=np.int64))
    n = PATCH * GRID
    got = run(hb, raw, (3, n, n), params, m32=DIAG, m70=DIAG)
    _, curve, _ = oracle.camera_pipe_tables(DIAG, DIAG, *params)
    same(got[:, cy, cx], np.broadcast_to(curve, (3, 1024)), "curve")
    same(got, ref(oracle, raw, (3, n, n), params, m32=DIAG, m70=DIAG), "frame")


# ---- 5. row bands on one GPU ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("band_h", [96, 101])  # three whole row tiles per band; heights 101 and 102
@pytest.mark.parametrize("world_size", [2, 3, 5, 8])
def test_row_bands(hb, oracle, world_size, band_h):
    """What halide_b200.dist.InputHaloSharder.camera_pipe does on each rank, without the row exchange: output rows split
    by band_rows, each band's raw rows exactly dist.camera_pipe_need_rows, band buffers placed at their frame rows.  The
    stacked bands equal the whole-frame call byte for byte."""
    import torch
    from halide_b200 import dist
    out_h, out_w = band_h * world_size + (3 if band_h % 32 else 0), 160
    raw = raw_frame(out_h + 24, out_w + 32, 20 + world_size)
    traw = torch.from_numpy(raw).cuda()
    whole = torch.zeros((3, out_h, out_w), dtype=torch.uint8, device="cuda")
    hb.filters.camera_pipe(hb.HalideBuffer.from_torch(traw), *mats(hb), *DEFAULT, hb.HalideBuffer.from_torch(whole))
    bands = []
    for rank in range(world_size):
        lo, hi = dist.band_rows(rank, world_size, out_h)
        assert hi - lo + 1 >= 96 and (band_h == 96) == ((hi - lo + 1) % 32 == 0)
        band = torch.full((3, hi - lo + 1, out_w), 0xA5, dtype=torch.uint8, device="cuda")
        bo = hb.HalideBuffer.from_torch(band, (0, lo, 0))
        need = dist.camera_pipe_need_rows(bo, *mats(hb), DEFAULT)
        assert 0 <= need[0] and need[1] < raw.shape[0]
        hb.filters.camera_pipe(hb.HalideBuffer.from_torch(traw[need[0]:need[1] + 1], (0, need[0])), *mats(hb), *DEFAULT, bo)
        bands.append(band)
    torch.cuda.synchronize()
    whole = whole.cpu().numpy()
    same(torch.cat(bands, 1).cpu().numpy(), whole, "stacked bands")
    same(whole, ref(oracle, raw, (3, out_h, out_w)), "whole frame against the oracle")


# ---- 6. frame size, repeated calls, kernel names -------------------------------------------------------------------
RW, RH = 70, 40  # region size: each region below crosses a tile seam in both directions
REGIONS_8K = ([(0, 0), (7680 - RW, 0), (0, 4320 - RH), (7680 - RW, 4320 - RH)] +
              [(x, y) for x in (61 * 64 - 1, 61 * 64, 61 * 64 + 1) for y in (64 * 32 - 1, 64 * 32, 64 * 32 + 1)])


@pytest.fixture(scope="module")
def frame_8k(hb):
    """7680 x 4320 output from a 7712 x 4344 raw (the harness's rule: 32 columns and 24 rows fewer, then multiples of
    32)."""
    h, w = 4344, 7712
    assert (((h - 24) // 32) * 32, ((w - 32) // 32) * 32) == (4320, 7680)
    raw = raw_frame(h, w, 12)
    return raw, run(hb, raw, (3, 4320, 7680))


@pytest.mark.parametrize("x0,y0", REGIONS_8K)
def test_8k_regions(hb, oracle, frame_8k, x0, y0):
    """Regions of the 8K frame against the oracle on exactly their bounds-query crop (no boundary condition: the crop
    determines the region)."""
    raw, got = frame_8k
    shape, mins = (3, RH, RW), (x0, y0, 0)
    qx, qy, qw, qh = need_region(hb, out_desc(hb, shape, mins))
    assert qx >= 0 and qy >= 0 and qx + qw <= raw.shape[1] and qy + qh <= raw.shape[0]
    crop = np.ascontiguousarray(raw[qy:qy + qh, qx:qx + qw])
    same(got[:, y0:y0 + RH, x0:x0 + RW], ref(oracle, crop, shape, in_mins=(qx, qy), out_mins=mins))


def test_back_to_back_calls_use_their_own_tables(hb, oracle):
    """A, B, A with different scalars, all on device buffers with no synchronisation in between: each call's matrix,
    curve and sharpen strength live in per-call scratch, which must never be read stale or overwritten early."""
    import torch
    raw = raw_frame(120, 200, 13)
    traw = torch.from_numpy(raw).cuda()
    t32, t70 = torch.from_numpy(CP_M3200).cuda(), torch.from_numpy(CP_M7000).cuda()
    a = DEFAULT
    b = cp_params(dict(color_temp=7000.0, gamma=0.5, contrast=-100.0, sharpen=100.0, black=0, white=900))
    shape = (3, 96, 160)
    outs = [torch.zeros(shape, dtype=torch.uint8, device="cuda") for _ in range(3)]
    bufs = []  # kept alive until the synchronisation
    for params, o in zip((a, b, a), outs):
        bufs.append([hb.HalideBuffer.from_torch(t) for t in (traw, t32, t70, o)])
        bi, b32, b70, bo = bufs[-1]
        hb.filters.camera_pipe(bi, b32, b70, *params, bo)
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in outs]
    want_a, want_b = ref(oracle, raw, shape, a), ref(oracle, raw, shape, b)
    assert not np.array_equal(want_a, want_b)
    same(got[0], want_a, "first A")
    same(got[1], want_b, "B")
    same(got[2], want_a, "second A")


def test_kernel_names(hb):
    with kernels_run(hb) as ran:
        run(hb, raw_frame(56, 96, 0), (3, 32, 64))
    assert set(ran) == {"cp_tables", "camera_pipe"} and all(n == 1 for n, _ in ran.values()), ran
