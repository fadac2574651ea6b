"""GPU tests of the batch bilateral_grid entry points (float32, uint8, and float32 at any cell size).  Their contract: output
frame n is, bit for bit, what the one-frame entry point (bilateral_grid, halide_b200_bilateral_grid_u8,
halide_b200_bilateral_grid_s_sigma) gives on input frame n with the same arguments.  So every case runs the one-frame
entry point frame by frame on contiguous copies and compares bit patterns (float32 as uint32).  Clips are numpy arrays or
torch tensors [n, y, x]."""
import threading

import numpy as np
import pytest

from bilateral_grid_exact import KERNELS_8, KERNELS_S, dyadic, noise
from util import kernels_run

pytestmark = pytest.mark.gpu
GUARD = {np.float32: np.float32(-7.5), np.uint8: np.uint8(0xA5)}
KINDS = ["f32", "u8", "s_sigma"]
GRID_BUDGET = 256 << 20  # bilateral_grid.cu: kGridBudget
MIN_GROUP = 3            # bilateral_grid.cu: kMinGroup
MAX_GRID_Z = 65535


def dtype_of(kind):
    return np.uint8 if kind == "u8" else np.float32


def clip_of(kind, shape, seed):
    rng = np.random.default_rng(seed)
    if kind == "u8":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    return rng.random(shape, dtype=np.float32)


def fns(kind):
    """(batch call site, one-frame call site)."""
    from halide_b200 import bilateral_grid_video as v, filters as f
    return {"f32": (v.bilateral_grid_batch, f.bilateral_grid), "u8": (v.bilateral_grid_u8_batch, f.bilateral_grid_u8),
            "s_sigma": (v.bilateral_grid_s_sigma_batch, f.bilateral_grid_s_sigma)}[kind]


def params(kind, s, r_sigma):
    return (s, r_sigma) if kind == "s_sigma" else (r_sigma,)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same(got, want, what=""):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def one_frame(hb, kind, frame, args, out_hw=None, in_mins=None, out_mins=None):
    """The one-frame entry point on a contiguous copy of frame [y, x]."""
    out = np.zeros(frame.shape if out_hw is None else tuple(out_hw), frame.dtype)
    bi = hb.HalideBuffer.from_numpy(np.ascontiguousarray(frame), in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    fns(kind)[1](bi, *args, bo)
    bo.copy_to_host()
    return out


def run_batch(hb, kind, clip, out, args, in_mins=None, out_mins=None):
    """The batch entry point on numpy views [n, y, x]; out is written in place.  Returns the kernels it launched."""
    bi = hb.HalideBuffer.from_numpy(clip, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    with kernels_run(hb) as ran:
        fns(kind)[0](bi, *args, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return ran


def check_batch(hb, kind, clip, args, out_n=None, in_n0=0, out_n0=0, out_hw=None, xy_in_mins=(0, 0),
                xy_out_mins=(0, 0)):
    """The batch entry point on clip (any view) into out_n frames starting at frame out_n0 (input frames start at in_n0),
    against the one-frame entry point on each input frame an output frame reads.  Returns the kernels it launched."""
    out_n = clip.shape[0] if out_n is None else out_n
    hw = clip.shape[1:] if out_hw is None else tuple(out_hw)
    out = np.zeros((out_n,) + hw, clip.dtype)
    ran = run_batch(hb, kind, clip, out, args, tuple(xy_in_mins) + (in_n0,), tuple(xy_out_mins) + (out_n0,))
    for k in range(out_n):
        want = one_frame(hb, kind, clip[out_n0 + k - in_n0], args, hw, xy_in_mins, xy_out_mins)
        assert_same(out[k], want, f"{kind} frame {k} args {args}")
    return ran


def frames_per_group(h, w, n, r_sigma, s=8, ox=0, oy=0):
    """bilateral_grid.cu's G: min(N, kMaxGridZ, max(1, kGridBudget / (the two grids of one frame))), and 1 (frame by
    frame, through the one-frame kernels) when fewer than kMinGroup frames fit the budget."""
    inv_r = np.float32(1.0) / np.float32(r_sigma)
    nz = int(np.float32(np.float32(1.0) * inv_r) + np.float32(0.5)) + 2
    gx0, gy0 = ox // s - 2, oy // s - 2
    gw = (ox + w - 1) // s + 1 + 2 - gx0 + 1
    gh = (oy + h - 1) // s + 1 + 2 - gy0 + 1
    fit = max(1, GRID_BUDGET // (2 * gw * gh * nz * 2 * 4))
    return min(n, MAX_GRID_Z, fit) if fit >= MIN_GROUP else 1


# ---- batch = one-frame calls, frame by frame ------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [1, 3, 8])
def test_batches_of_odd_sizes(hb, kind, n):
    for h, w in [(29, 37), (257, 333)]:
        ran = check_batch(hb, kind, clip_of(kind, (n, h, w), 100 * n + h), params(kind, 5, 0.1))
        assert sum(c for c, _ in ran.values()) == 3, ran


@pytest.mark.parametrize("kind", KINDS)
def test_1080p_clip(hb, kind):
    check_batch(hb, kind, clip_of(kind, (3, 1080, 1920), 7), params(kind, 3, 0.1))


@pytest.mark.parametrize("kind", KINDS)
def test_mins_and_a_larger_input(hb, kind):
    """Nonzero, negative and unaligned x/y mins on both buffers; an input larger than the output on every side."""
    clip = clip_of(kind, (3, 140, 190), 11)
    check_batch(hb, kind, clip, params(kind, 6, 0.25), out_hw=(101, 133), xy_in_mins=(-29, -21),
                xy_out_mins=(-13, -7))
    check_batch(hb, kind, clip, params(kind, 12, 0.1), out_hw=(61, 77), xy_in_mins=(5, 3), xy_out_mins=(41, 19))


@pytest.mark.parametrize("kind", KINDS)
def test_output_frames_a_sub_range_of_the_input(hb, kind):
    clip = clip_of(kind, (6, 45, 71), 12)
    check_batch(hb, kind, clip, params(kind, 4, 0.1), out_n=3, in_n0=-2, out_n0=0)
    check_batch(hb, kind, clip, params(kind, 8, 0.1), out_n=2, in_n0=10, out_n0=14)


@pytest.mark.parametrize("kind", KINDS)
def test_reversed_and_broadcast_clips(hb, kind):
    clip = clip_of(kind, (5, 38, 59), 91)
    check_batch(hb, kind, clip[::-1], params(kind, 3, 0.1))                                      # negative frame stride
    check_batch(hb, kind, np.broadcast_to(clip[2], (4,) + clip.shape[1:]), params(kind, 16, 0.2))  # frame stride 0


@pytest.mark.parametrize("kind", KINDS)
def test_padded_rows_and_unaligned_frames_on_the_device(hb, kind):
    """Device-resident torch views over guard-filled storage: rows padded to a pitch of 4k elements, frame strides of
    4k + 1 (so frame n starts n mod 4 elements past an aligned address, and the vector loads and stores run in some frames
    and not others), and an output whose frames are laid out differently from the input's.  Samples outside the output's
    region keep their values."""
    import torch
    dt = dtype_of(kind)
    n, h, w = 6, 53, 131
    tdt = torch.uint8 if dt == np.uint8 else torch.float32
    clip = clip_of(kind, (n, h, w), 44)
    args = params(kind, 7, 0.1)
    in_pitch, in_fs = 136, 136 * h + 1
    out_pitch, out_fs = 140, 140 * (h + 2) + 5
    tin = torch.full((in_fs * n + 8,), float(GUARD[dt]), dtype=tdt, device="cuda")
    vin = tin.as_strided((n, h, w), (in_fs, in_pitch, 1), 3)
    vin.copy_(torch.from_numpy(clip).cuda())
    tout = torch.full((out_fs * n + 8,), float(GUARD[dt]), dtype=tdt, device="cuda")
    vout = tout.as_strided((n, h, w), (out_fs, out_pitch, 1), 1)
    fns(kind)[0](hb.HalideBuffer.from_torch(vin), *args, hb.HalideBuffer.from_torch(vout))
    torch.cuda.synchronize()
    got = vout.cpu().numpy()
    for k in range(n):
        assert_same(got[k], one_frame(hb, kind, clip[k], args), f"{kind} frame {k}")
    mask = torch.ones_like(tout, dtype=torch.bool)
    mask.as_strided((n, h, w), (out_fs, out_pitch, 1), 1).fill_(False)
    outside = tout[mask].cpu().numpy()
    assert (bits(outside) == bits(np.array([GUARD[dt]], dt))).all(), "samples outside the output's region changed"


# ---- cell sizes, groups and grid z ----------------------------------------------------------------------------------

@pytest.mark.parametrize("s", [1, 3, 8, 16, 128])
def test_s_sigma_batch_cell_sizes(hb, s):
    """S = 8 runs bilateral_grid's kernels, any other S the any-S kernels; every frame equals the one-frame call."""
    clip = clip_of("s_sigma", (4, 97, 203), s)
    ran = check_batch(hb, "s_sigma", clip, (s, 0.1))
    assert set(ran) == (KERNELS_8 if s == 8 else KERNELS_S), sorted(ran)
    assert all(c == 1 for c, _ in ran.values()), ran


@pytest.mark.parametrize("kind", KINDS)
def test_groups_of_frames(hb, kind):
    """7 frames of 1920 x 1080 at r_sigma = 1/128 (130 planes: about 71 MB of grids a frame at S = 8) run in groups of
    frames_per_group (3 at S = 8, 4 at S = 9), three launches each; every frame, those on both sides of each group
    boundary included, equals its one-frame call.  A clip that fits in one group takes three launches."""
    r = float(np.float32(1.0) / np.float32(128))
    n, h, w = 7, 1080, 1920
    s = 9 if kind == "s_sigma" else 8
    g = frames_per_group(h, w, n, r, s)
    assert 1 < g < n
    clip = clip_of(kind, (n, h, w), 128)
    ran = check_batch(hb, kind, clip, params(kind, s, r))
    assert sum(c for c, _ in ran.values()) == 3 * -(-n // g), (g, ran)
    assert all(c == -(-n // g) for c, _ in ran.values()), (g, ran)
    ran = check_batch(hb, kind, clip[:g], params(kind, s, r))
    assert sum(c for c, _ in ran.values()) == 3, ran


@pytest.mark.parametrize("kind", KINDS)
def test_frames_too_large_for_a_group_run_one_by_one(hb, kind):
    """Frames whose grids leave room for fewer than kMinGroup of them in the budget (7680 x 4320 at r_sigma 0.1: 101 MB;
    1920 x 1080 at S = 6 and r_sigma 1/128: 93 MB) run frame by frame, three launches each, and equal their one-frame
    calls.  Two frames of 8 x 8 still run as one group."""
    if kind == "s_sigma":
        n, h, w, s, r = 3, 1080, 1920, 6, float(np.float32(1.0) / np.float32(128))
    else:
        n, h, w, s, r = 2, 4320, 7680, 8, 0.1
    assert frames_per_group(h, w, n, r, s) == 1
    ran = check_batch(hb, kind, clip_of(kind, (n, h, w), 77), params(kind, s, r))
    assert all(c == n for c, _ in ran.values()) and len(ran) == 3, ran
    ran = check_batch(hb, kind, clip_of(kind, (2, 8, 8), 78), params(kind, s, r))
    assert all(c == 1 for c, _ in ran.values()) and len(ran) == 3, ran


@pytest.mark.parametrize("kind", ["f32", "u8"])
def test_more_frames_than_the_grid_z_extent(hb, kind):
    """65 537 frames of 8 x 8: more than one launch's grid z extent.  The frames repeat seven distinct ones, so each
    output frame is checked against the one-frame result of its distinct frame, the frames at each group boundary among
    them."""
    n, k, r = 65537, 7, 0.1
    g = frames_per_group(8, 8, n, r)
    distinct = clip_of(kind, (k, 8, 8), 65537)
    clip = np.ascontiguousarray(np.concatenate([distinct] * (n // k + 1))[:n])
    out = np.zeros(clip.shape, clip.dtype)
    ran = run_batch(hb, kind, clip, out, (r,))
    assert sum(c for c, _ in ran.values()) == 3 * -(-n // g), (g, ran)
    wants = [one_frame(hb, kind, distinct[j], (r,)) for j in range(k)]
    for j in range(k):
        assert_same(out[j::k], np.broadcast_to(wants[j], out[j::k].shape), f"frames {j} mod {k}")
    for b in range(g, n, g):
        for f in (b - 1, b):
            assert_same(out[f], wants[f % k], f"frame {f} at a group boundary")


@pytest.mark.parametrize("kind", ["f32", "s_sigma"])
def test_non_finite_pixels_stay_in_their_frame(hb, kind):
    """A frame holding NaN and +-inf pixels gives the one-frame result, and the frames around it are unaffected."""
    clip = clip_of(kind, (3, 64, 96), 5)
    clip[1, 10, 10:20] = np.nan
    clip[1, 30, 40:44] = np.inf
    clip[1, 50:53, 5] = -np.inf
    check_batch(hb, kind, clip, params(kind, 3, 0.1))


@pytest.mark.parametrize("kind", KINDS)
def test_samples_outside_the_output_keep_their_values(hb, kind):
    """The output is a crop, in x, y and frames, of a guard-filled device array."""
    import torch
    dt = dtype_of(kind)
    tdt = torch.uint8 if dt == np.uint8 else torch.float32
    clip = clip_of(kind, (4, 41, 67), 3)
    full = torch.full((6, 47, 77), float(GUARD[dt]), dtype=tdt, device="cuda")
    view = full[1:5, 2:43, 3:70]
    args = params(kind, 8, 0.1)
    fns(kind)[0](hb.HalideBuffer.from_torch(torch.from_numpy(clip).cuda()), *args, hb.HalideBuffer.from_torch(view))
    torch.cuda.synchronize()
    got = full.cpu().numpy()
    for k in range(4):
        assert_same(got[1 + k, 2:43, 3:70], one_frame(hb, kind, clip[k], args), f"frame {k}")
    got[1:5, 2:43, 3:70] = GUARD[dt]
    assert (bits(got) == bits(np.array([GUARD[dt]], dt))).all(), "samples outside the output changed"


# ---- against the oracle ---------------------------------------------------------------------------------------------

def test_clips_against_the_oracle(hb, oracle):
    """A dyadic clip at S = 8 (where bg_hist_blurz's two partial sums are exact) and a noise clip at S = 3, bit for bit
    frame by frame against oracle/oracle_bilateral_grid.cpp."""
    from halide_b200 import bilateral_grid_video as v
    for s, clip in [(8, np.stack([dyadic((45, 77), 30 + k) for k in range(3)])),
                    (3, np.stack([noise((45, 77), 40 + k) for k in range(3)]))]:
        out = np.zeros_like(clip)
        bi, bo = hb.HalideBuffer.from_numpy(clip), hb.HalideBuffer.from_numpy(out, host_dirty=False)
        if s == 8:
            v.bilateral_grid_batch(bi, 0.125, bo)
        else:
            v.bilateral_grid_s_sigma_batch(bi, s, 0.125, bo)
        bo.copy_to_host()
        for k in range(3):
            assert_same(out[k], oracle.bilateral_grid(clip[k], 0.125, s_sigma=s), f"S = {s} frame {k}")


# ---- concurrent callers ---------------------------------------------------------------------------------------------

def test_two_threads_on_two_streams(hb):
    """Two threads, each bound to a stream of its own, call _batch and _u8_batch with different r_sigma at the same time,
    three rounds each; every result equals the one-frame calls on its frames."""
    jobs = []
    for i, (kind, r) in enumerate([("f32", 0.1), ("u8", 0.2), ("u8", 0.05), ("f32", 0.25)]):
        clip = clip_of(kind, (5, 97, 143), 500 + i)
        jobs.append((kind, clip, r, np.stack([one_frame(hb, kind, f, (r,)) for f in clip])))
    l = hb.load_library()
    errors, mismatches = [], []

    def thread(i):
        s = l.halide_b200_stream_create()
        try:
            assert s, "halide_b200_stream_create failed"
            l.halide_b200_set_stream(s)
            mine = jobs[i::2]  # thread 0: f32 at 0.1 and u8 at 0.05, thread 1: u8 at 0.2 and f32 at 0.25
            for rnd in range(3):
                for kind, clip, r, want in mine + mine[::-1]:
                    out = np.zeros_like(clip)
                    bi, bo = hb.HalideBuffer.from_numpy(clip), hb.HalideBuffer.from_numpy(out, host_dirty=False)
                    fns(kind)[0](bi, r, bo)
                    bo.copy_to_host()
                    if not np.array_equal(bits(out), bits(want)):
                        mismatches.append(f"thread {i} round {rnd}: {kind} r_sigma {r}")
        except BaseException as e:
            errors.append(e)
        finally:
            if s:
                l.halide_b200_set_stream(None)
                l.halide_b200_stream_destroy(s)

    threads = [threading.Thread(target=thread, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert not mismatches, "\n".join(mismatches)
