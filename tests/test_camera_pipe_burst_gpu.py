"""camera_pipe on raw bursts and into pixel-interleaved outputs (halide_b200_camera_pipe_batch, _interleaved,
_interleaved_batch), bit for bit: per frame against the oracle, and against camera_pipe's own planar calls.

- Small bursts against the oracle at the default parameters and two extremes.
- The harness frame (2592 x 1968 raw -> 2560 x 1920) and a 4 x 4K burst against single camera_pipe calls, planar and
  transposed; the launches a burst makes.
- Interleaved outputs filled with a sentinel that must survive outside the covered samples: pitch 3 and 4, channel
  crops, widths that are not a multiple of 4, every Bayer parity of the origin, odd bases and padded rows, on the host
  and on the device.
- Frame geometry: nonzero frame mins over a larger input, reversed and broadcast bursts, raw frames cut to exactly the
  bounds query, and more frames than one grid's z extent."""
import numpy as np
import pytest
from numpy.lib.stride_tricks import as_strided

from test_camera_pipe_edges_gpu import raw_frame
from util import CP_EXTREMES, CP_M3200, CP_M7000, cp_param_id, cp_params, kernels_run

pytestmark = pytest.mark.gpu
DEFAULT = cp_params({})


def mats(hb):
    return hb.HalideBuffer.from_numpy(CP_M3200.copy()), hb.HalideBuffer.from_numpy(CP_M7000.copy())


def ref(oracle, raw, shape, params=DEFAULT, in_mins=None, out_mins=None):
    return oracle.camera_pipe(raw, CP_M3200, CP_M7000, *params, shape, in_mins=in_mins, out_mins=out_mins)


def same(got, want, what="result"):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} of {got.size} bytes differ, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]}, want {want[tuple(bad[0])]}")


def burst(h, w, n, seed):
    return np.stack([raw_frame(h, w, seed + k) for k in range(n)])


def call(hb, fn, bi, bo, params=DEFAULT):
    getattr(hb.filters, fn)(bi, *mats(hb), *params, bo)


def run_batch(hb, raw, out_shape, params=DEFAULT, interleaved=False, in_mins=None, out_mins=None):
    """Host buffers: a raw burst (n, h, w) and an (n, 3, H, W) planar or (n, H, W, 3) interleaved output; returns the
    output as (n, 3, H, W)."""
    n, c, h, w = out_shape
    if interleaved:
        out = np.zeros((n, h, w, c), np.uint8)
        bo = hb.HalideBuffer.from_numpy(out.transpose(0, 3, 1, 2), out_mins, host_dirty=False)
    else:
        out = np.zeros(out_shape, np.uint8)
        bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    call(hb, "camera_pipe_interleaved_batch" if interleaved else "camera_pipe_batch",
         hb.HalideBuffer.from_numpy(raw, in_mins), bo, params)
    bo.copy_to_host()
    return out.transpose(0, 3, 1, 2) if interleaved else out


# ---- 1. small bursts against the oracle ----------------------------------------------------------------------------
@pytest.mark.parametrize("overrides", [{}, dict(sharpen=100.0), dict(black=0, white=1)], ids=cp_param_id)
@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
def test_burst_matches_oracle(hb, oracle, overrides, interleaved):
    assert all(o in CP_EXTREMES for o in [dict(sharpen=100.0), dict(black=0, white=1)])
    params = cp_params(overrides)
    raw = burst(180, 240, 3, 30)
    got = run_batch(hb, raw, (3, 3, 150, 200), params, interleaved)
    for k in range(3):
        same(got[k], ref(oracle, raw[k], (3, 150, 200), params), f"frame {k}")
    if not interleaved:
        return
    one = np.zeros((150, 200, 3), np.uint8)  # the single-frame interleaved entry point on frame 1
    bo = hb.HalideBuffer.from_numpy(one.transpose(2, 0, 1), host_dirty=False)
    call(hb, "camera_pipe_interleaved", hb.HalideBuffer.from_numpy(raw[1]), bo, params)
    bo.copy_to_host()
    same(one.transpose(2, 0, 1), got[1], "single interleaved frame")


# ---- 2. large frames against camera_pipe's planar calls ------------------------------------------------------------
def raw_for(hb, n, h, w, seed):
    """A device raw burst of exactly the frame the bounds query asks for an (h, w) output, with its mins."""
    import torch
    q = hb.HalideBuffer.bounds_query(np.uint16, 3)
    call(hb, "camera_pipe_batch", q, hb.HalideBuffer(np.uint8, (w, h, 3, n)))
    (x0, qw, _), (y0, qh, _), _ = q.shape()
    raw = torch.from_numpy(burst(qh, qw, n, seed).view(np.int16)).cuda().view(torch.uint16)
    return raw, (x0, y0, 0)


@pytest.mark.parametrize("n,h,w", [(1, 1920, 2560), (4, 2160, 3840)], ids=["harness_frame", "4x4k"])
def test_large_frames_match_single_calls(hb, n, h, w):
    import torch
    if n == 1:  # the harness's raw frame and output (apps/camera_pipe/process.cpp)
        raw = torch.from_numpy(burst(1968, 2592, 1, 40).view(np.int16)).cuda().view(torch.uint16)
        mins = None
    else:
        raw, mins = raw_for(hb, n, h, w, 41)
    singles = torch.zeros((n, 3, h, w), dtype=torch.uint8, device="cuda")
    for k in range(n):
        call(hb, "camera_pipe", hb.HalideBuffer.from_torch(raw[k], None if mins is None else mins[:2]),
             hb.HalideBuffer.from_torch(singles[k]))
    planar = torch.full((n, 3, h, w), 0xA5, dtype=torch.uint8, device="cuda")
    il = torch.full((n, h, w, 3), 0xA5, dtype=torch.uint8, device="cuda")
    il1 = torch.full((h, w, 3), 0xA5, dtype=torch.uint8, device="cuda")
    call(hb, "camera_pipe_batch", hb.HalideBuffer.from_torch(raw, mins), hb.HalideBuffer.from_torch(planar))
    call(hb, "camera_pipe_interleaved_batch", hb.HalideBuffer.from_torch(raw, mins),
         hb.HalideBuffer.from_torch(il.permute(0, 3, 1, 2)))
    call(hb, "camera_pipe_interleaved", hb.HalideBuffer.from_torch(raw[0], None if mins is None else mins[:2]),
         hb.HalideBuffer.from_torch(il1.permute(2, 0, 1)))
    torch.cuda.synchronize()
    assert torch.equal(planar, singles), "batch frames differ from single camera_pipe calls"
    assert torch.equal(il, singles.permute(0, 2, 3, 1)), "interleaved batch differs from the planar frames transposed"
    assert torch.equal(il1, singles[0].permute(1, 2, 0)), "interleaved frame differs from the planar frame transposed"


def test_launches(hb):
    """A burst of any size makes camera_pipe's two launches; at N = 1 the batch is byte for byte camera_pipe."""
    raw = burst(56, 96, 5, 50)
    one = np.zeros((3, 32, 64), np.uint8)
    bo = hb.HalideBuffer.from_numpy(one, host_dirty=False)
    with kernels_run(hb) as ran:
        call(hb, "camera_pipe", hb.HalideBuffer.from_numpy(raw[0]), bo)
    bo.copy_to_host()
    assert {k: v[0] for k, v in ran.items()} == {"cp_tables": 1, "camera_pipe": 1}, ran
    for n in (1, 5):
        with kernels_run(hb) as ran:
            got = run_batch(hb, raw[:n], (n, 3, 32, 64))
        assert {k: v[0] for k, v in ran.items()} == {"cp_tables": 1, "camera_pipe": 1}, (n, ran)
        same(got[0], one, f"batch of {n}, frame 0")
        with kernels_run(hb) as ran:
            got_il = run_batch(hb, raw[:n], (n, 3, 32, 64), interleaved=True)
        assert {k: v[0] for k, v in ran.items()} == {"cp_tables": 1, "camera_pipe_il": 1}, (n, ran)
        same(got_il, got, f"interleaved batch of {n}")


# ---- 3. interleaved layouts ----------------------------------------------------------------------------------------
WORLD_RAW_MINS = (-40, -20)
ORIGINS = [(0, 0), (-37, -11), (7, 4), (-6, 3)]  # (x, y) parities (even, even), (odd, odd), (odd, even), (even, odd)
LH, LW = 37, 93  # two tile rows; a last tile column of 29 pixels (7 whole 4-pixel groups and one partial)
FRAMES = 3


@pytest.fixture(scope="module")
def world():
    return burst(150, 230, FRAMES, 60)


# (pixel pitch, channels [c0, c1), base offset in bytes, row padding in bytes)
LAYOUTS = [(3, (0, 3), 0, 0), (3, (0, 3), 1, 0), (3, (0, 3), 0, 5), (3, (0, 3), 2, 4), (4, (0, 3), 0, 0),
           (4, (0, 3), 3, 8), (3, (1, 2), 0, 0), (3, (0, 2), 1, 3), (4, (1, 3), 0, 0)]


def layout_id(lay):
    pitch, (c0, c1), off, pad = lay
    return f"pitch{pitch}-c[{c0},{c1})-off{off}-pad{pad}"


@pytest.mark.parametrize("variant", ["host", "device"])
@pytest.mark.parametrize("lay", LAYOUTS, ids=layout_id)
@pytest.mark.parametrize("ox,oy", ORIGINS)
@pytest.mark.parametrize("frames", [None, FRAMES], ids=["frame", "burst"])
def test_interleaved_layouts(hb, oracle, world, frames, ox, oy, lay, variant):
    """The output is a view into a canvas filled with a sentinel (0x00, then 0xFF): rows `pad` bytes longer than the
    pixels, the first sample `off` bytes in, a burst's frames a further 7 bytes apart.  After the call the covered
    samples hold the oracle's bytes and every other byte of the canvas its sentinel."""
    import torch
    pitch, (c0, c1), off, pad = lay
    n = frames or 1
    row = LW * pitch + pad
    fstride = LH * row + 7
    size = off + (n - 1) * fstride + (LH - 1) * row + LW * pitch + 11
    want = [ref(oracle, world[k], (c1 - c0, LH, LW), in_mins=WORLD_RAW_MINS, out_mins=(ox, oy, c0)) for k in range(n)]
    mins = (ox, oy, c0) + ((0,) if frames else ())
    if frames:
        bi = hb.HalideBuffer.from_numpy(world, WORLD_RAW_MINS + (0,))
    else:
        bi = hb.HalideBuffer.from_numpy(world[0], WORLD_RAW_MINS)
    for sentinel in (0x00, 0xFF):
        expect = np.full(size, sentinel, np.uint8)
        ev = as_strided(expect[off:], (n, LH, LW, pitch), (fstride, row, pitch, 1))
        for k in range(n):
            ev[k, :, :, c0:c1] = want[k].transpose(1, 2, 0)
        shape, strides = (c1 - c0, LH, LW), (1, row, pitch)
        if frames:
            shape, strides = (n,) + shape, (fstride,) + strides
        if variant == "host":
            backing = np.full(size, sentinel, np.uint8)
            view = as_strided(backing[off + c0:], shape, strides)
            bo = hb.HalideBuffer.from_numpy(view, mins, host_dirty=False)
        else:
            backing = torch.full((size,), sentinel, dtype=torch.uint8, device="cuda")
            bo = hb.HalideBuffer.from_torch(backing.as_strided(shape, strides, off + c0), mins)
        call(hb, "camera_pipe_interleaved_batch" if frames else "camera_pipe_interleaved", bi, bo)
        if variant == "host":
            bo.copy_to_host()
        else:
            torch.cuda.synchronize()
            backing = backing.cpu().numpy()
        same(backing, expect, f"sentinel {sentinel:#x}")


@pytest.mark.parametrize("w", [1, 2, 3, 5, 6, 7, 63, 65, 66, 67, 130])
def test_interleaved_widths(hb, oracle, world, w):
    """Widths that are not a multiple of 4 (and 4-pixel groups split at the tile seam), dense RGB on the device."""
    import torch
    ox, oy, h = -37, -11, 33
    want = ref(oracle, world[0], (3, h, w), in_mins=WORLD_RAW_MINS, out_mins=(ox, oy, 0))
    backing = torch.full((h * w * 3 + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    out = backing[4:4 + h * w * 3].view(h, w, 3)
    call(hb, "camera_pipe_interleaved", hb.HalideBuffer.from_numpy(world[0], WORLD_RAW_MINS),
         hb.HalideBuffer.from_torch(out.permute(2, 0, 1), (ox, oy, 0)))
    torch.cuda.synchronize()
    got = backing.cpu().numpy()
    same(got[4:4 + h * w * 3].reshape(h, w, 3).transpose(2, 0, 1), want)
    assert (got[:4] == 0xA5).all() and (got[4 + h * w * 3:] == 0xA5).all()


def test_channels_last_tensor(hb, oracle, world):
    """An (N, 3, H, W) tensor in torch.channels_last memory format is an interleaved output as it stands."""
    import torch
    out = torch.zeros((FRAMES, 3, LH, LW), dtype=torch.uint8, device="cuda").to(memory_format=torch.channels_last)
    call(hb, "camera_pipe_interleaved_batch", hb.HalideBuffer.from_numpy(world, WORLD_RAW_MINS + (0,)),
         hb.HalideBuffer.from_torch(out, (0, 0, 0, 0)))
    torch.cuda.synchronize()
    for k in range(FRAMES):
        same(out[k].cpu().numpy(), ref(oracle, world[k], (3, LH, LW), in_mins=WORLD_RAW_MINS), f"frame {k}")


# ---- 4. frame geometry ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
def test_frame_mins_and_a_larger_input(hb, oracle, interleaved):
    """Input frames 3 .. 8, output frames 5 .. 7: output frame n reads input frame n."""
    raw = burst(100, 140, 6, 70)
    got = run_batch(hb, raw, (3, 3, 64, 96), interleaved=interleaved, in_mins=(0, 0, 3), out_mins=(0, 0, 0, 5))
    for k in range(3):
        same(got[k], ref(oracle, raw[2 + k], (3, 64, 96)), f"output frame {5 + k}")


def test_reversed_and_broadcast_bursts(hb, oracle):
    """A reversed burst (negative frame stride) and one frame broadcast to four (frame stride 0) on the planar batch."""
    raw = burst(100, 140, 4, 80)
    want = [ref(oracle, raw[k], (3, 64, 96)) for k in range(4)]
    rev = raw[::-1]
    assert rev.strides[0] < 0
    got = run_batch(hb, rev, (4, 3, 64, 96))
    for k in range(4):
        same(got[k], want[3 - k], f"reversed, output frame {k}")
    bc = np.broadcast_to(raw[2], (4,) + raw.shape[1:])
    assert bc.strides[0] == 0
    got = run_batch(hb, bc, (4, 3, 64, 96))
    for k in range(4):
        same(got[k], want[2], f"broadcast, output frame {k}")


@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
@pytest.mark.parametrize("ox,oy", ORIGINS)
def test_tight_raw_burst(hb, oracle, world, ox, oy, interleaved):
    """Raw frames cut to exactly the bounds query's region, at every Bayer parity of the output origin."""
    w, h = 65, 33
    q = hb.HalideBuffer.bounds_query(np.uint16, 3)
    call(hb, "camera_pipe_batch", q, hb.HalideBuffer(np.uint8, (w, h, 3, FRAMES), mins=(ox, oy, 0, 0)))
    (x0, qw, _), (y0, qh, _), (n0, qn, _) = q.shape()
    assert (n0, qn) == (0, FRAMES)
    ax, ay = x0 - WORLD_RAW_MINS[0], y0 - WORLD_RAW_MINS[1]
    tight = np.ascontiguousarray(world[:, ay:ay + qh, ax:ax + qw])
    got = run_batch(hb, tight, (FRAMES, 3, h, w), interleaved=interleaved, in_mins=(x0, y0, 0), out_mins=(ox, oy, 0, 0))
    for k in range(FRAMES):
        same(got[k], ref(oracle, tight[k], (3, h, w), in_mins=(x0, y0), out_mins=(ox, oy, 0)), f"frame {k}")


def test_more_frames_than_one_grid_z_extent(hb, oracle):
    """65 537 frames of a 1 x 1 output, each from a 12 x 12 raw frame (the bounds query's region) holding one of four
    tiles, tile n mod 4: frames past 65 535 are walked by the blocks of the first 65 535, from the right places."""
    import torch
    n = 65537
    q = hb.HalideBuffer.bounds_query(np.uint16, 3)
    call(hb, "camera_pipe_batch", q, hb.HalideBuffer(np.uint8, (1, 1, 3, n)))
    (x0, qw, _), (y0, qh, _), _ = q.shape()
    assert (qw, qh) == (12, 12)
    rng = np.random.default_rng(90)
    tiles = rng.integers(0, 1024, (4, 12, 12), dtype=np.uint16)
    tiles[:, 6, 6] = [60000, 0, 1023, 300]
    want = np.stack([ref(oracle, t, (3, 1, 1), in_mins=(x0, y0)) for t in tiles])
    assert len({w.tobytes() for w in want}) == 4
    raw = torch.from_numpy(tiles.view(np.int16)).cuda()[torch.arange(n, device="cuda") % 4].view(torch.uint16)
    planar = torch.full((n, 3, 1, 1), 0xA5, dtype=torch.uint8, device="cuda")
    il = torch.full((n, 1, 1, 4), 0xA5, dtype=torch.uint8, device="cuda")
    with kernels_run(hb) as ran:
        call(hb, "camera_pipe_batch", hb.HalideBuffer.from_torch(raw, (x0, y0, 0)), hb.HalideBuffer.from_torch(planar))
        call(hb, "camera_pipe_interleaved_batch", hb.HalideBuffer.from_torch(raw, (x0, y0, 0)),
             hb.HalideBuffer.from_torch(il[..., :3].permute(0, 3, 1, 2)))
    torch.cuda.synchronize()
    assert {k: v[0] for k, v in ran.items()} == {"cp_tables": 2, "camera_pipe": 1, "camera_pipe_il": 1}, ran
    expect = want[np.arange(n) % 4]
    same(planar.cpu().numpy(), expect, "planar")
    got = il.cpu().numpy()
    same(got[..., :3].transpose(0, 3, 1, 2), expect, "interleaved")
    assert (got[..., 3] == 0xA5).all(), "the fourth byte of each pixel was written"
