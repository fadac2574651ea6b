"""GPU tests of the batch halide_blur and stencil_chain entry points.  Their contract: output frame n is, bit for bit,
what the one-frame entry point (halide_blur, stencil_chain, halide_b200_stencil_chain_stencils) gives on input frame n
with the same arguments.  So every case runs the one-frame entry point frame by frame on contiguous copies and compares.
Clips are uint16 numpy arrays or torch tensors [n, y, x]."""
import threading

import numpy as np
import pytest

from util import kernels_run

pytestmark = pytest.mark.gpu
GUARD = np.uint16(0xA5C3)
KINDS = ["blur", "sc", "scs"]
SCRATCH_BUDGET = 256 << 20  # stencil_chain.cu: kScratchBudget
MAX_GRID_Z = 65535


def clip_of(shape, seed):
    return np.random.default_rng(seed).integers(0, 65536, shape, dtype=np.uint16)


def fns(kind):
    """(batch call site, one-frame call site)."""
    from halide_b200 import blur_video as b, filters as f, stencil_chain_video as c
    return {"blur": (b.blur_batch, f.halide_blur), "sc": (c.stencil_chain_batch, f.stencil_chain),
            "scs": (c.stencil_chain_stencils_batch, f.stencil_chain_stencils)}[kind]


def params(kind, s):
    return (s,) if kind == "scs" else ()


def stages(kind, args):
    return args[0] if kind == "scs" else 32


def out_hw_of(kind, hw):
    return (hw[0] - 2, hw[1] - 2) if kind == "blur" else tuple(hw)


def assert_same(got, want, what=""):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def one_frame(hb, kind, frame, args, out_hw=None, in_mins=None, out_mins=None):
    """The one-frame entry point on a contiguous copy of frame [y, x]."""
    out = np.zeros(out_hw_of(kind, frame.shape) if out_hw is None else tuple(out_hw), np.uint16)
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
    hw = out_hw_of(kind, clip.shape[1:]) if out_hw is None else tuple(out_hw)
    out = np.zeros((out_n,) + hw, np.uint16)
    ran = run_batch(hb, kind, clip, out, args, tuple(xy_in_mins) + (in_n0,), tuple(xy_out_mins) + (out_n0,))
    for k in range(out_n):
        want = one_frame(hb, kind, clip[out_n0 + k - in_n0], args, hw, xy_in_mins, xy_out_mins)
        assert_same(out[k], want, f"{kind} frame {k} args {args}")
    return ran


def launches(ran):
    return sum(c for c, _ in ran.values())


def frames_per_group(h, w, n, s):
    """stencil_chain.cu's G: min(N, kMaxGridZ, max(1, kScratchBudget / (one frame's scratch planes)))."""
    launches_ = -(-s // 4)
    max_r = 2 * (s - 4) if launches_ > 1 else 0
    planes = 2 if launches_ > 2 else 1 if launches_ > 1 else 0
    bw, bh = (w + 2 * max_r + 1) & ~1, h + 2 * max_r
    fit = max(1, SCRATCH_BUDGET // (planes * bw * bh * 2)) if planes else MAX_GRID_Z
    return min(n, MAX_GRID_Z, fit)


def want_launches(kind, args, h, w, n):
    if kind == "blur":
        return 1
    s = stages(kind, args)
    return -(-s // 4) * -(-n // frames_per_group(h, w, n, s))


# ---- batch = one-frame calls, frame by frame ------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [1, 3, 8])
def test_batches_of_odd_sizes(hb, kind, n):
    for h, w in [(29, 37), (257, 333), (6, 5)]:
        args = params(kind, 7)
        ran = check_batch(hb, kind, clip_of((n, h, w), 100 * n + h), args)
        assert launches(ran) == want_launches(kind, args, h, w, n), ran


@pytest.mark.parametrize("kind", KINDS)
def test_1080p_clip(hb, kind):
    ran = check_batch(hb, kind, clip_of((3, 1082, 1922) if kind == "blur" else (3, 1080, 1920), 7), params(kind, 9))
    assert launches(ran) == (1 if kind == "blur" else -(-stages(kind, params(kind, 9)) // 4)), ran


@pytest.mark.parametrize("kind", KINDS)
def test_mins_and_a_larger_input(hb, kind):
    """Nonzero, negative and odd x/y mins on both buffers; an input larger than the output on every side (and, for
    stencil_chain, an output reaching past the input, where repeat_edge applies)."""
    clip = clip_of((3, 140, 190), 11)
    check_batch(hb, kind, clip, params(kind, 6), out_hw=(101, 133), xy_in_mins=(-29, -21), xy_out_mins=(-13, -7))
    check_batch(hb, kind, clip, params(kind, 3), out_hw=(61, 77), xy_in_mins=(5, 3), xy_out_mins=(41, 19))
    if kind != "blur":
        check_batch(hb, kind, clip, params(kind, 5), out_hw=(150, 201), xy_in_mins=(5, 3), xy_out_mins=(-1, 2))


@pytest.mark.parametrize("kind", KINDS)
def test_output_frames_a_sub_range_of_the_input(hb, kind):
    clip = clip_of((6, 45, 71), 12)
    check_batch(hb, kind, clip, params(kind, 4), out_n=3, in_n0=-2, out_n0=0)
    check_batch(hb, kind, clip, params(kind, 8), out_n=2, in_n0=10, out_n0=14)


@pytest.mark.parametrize("kind", KINDS)
def test_reversed_and_broadcast_clips(hb, kind):
    clip = clip_of((5, 38, 59), 91)
    check_batch(hb, kind, clip[::-1], params(kind, 3))                                      # negative frame stride
    check_batch(hb, kind, np.broadcast_to(clip[2], (4,) + clip.shape[1:]), params(kind, 11))  # frame stride 0


def device_views(n, h, w, ih, iw, in_pitch, in_fs, out_pitch, out_fs, offset, seed):
    """A clip of n (ih, iw) frames as a device view with row pitch in_pitch and frame stride in_fs (elements), and a
    guard-filled output of n (h, w) frames with out_pitch / out_fs, both `offset` elements into their storage."""
    import torch
    clip = clip_of((n, ih, iw), seed)
    tin = torch.full((in_fs * n + 8,), int(GUARD), dtype=torch.uint16, device="cuda")
    vin = tin.as_strided((n, ih, iw), (in_fs, in_pitch, 1), offset)
    vin.copy_(torch.from_numpy(clip).cuda())
    tout = torch.full((out_fs * n + 8,), int(GUARD), dtype=torch.uint16, device="cuda")
    vout = tout.as_strided((n, h, w), (out_fs, out_pitch, 1), offset)
    return clip, vin, tout, vout


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("odd_frames", [True, False])
def test_padded_rows_and_unaligned_frames_on_the_device(hb, kind, odd_frames):
    """Device-resident torch views over guard-filled storage.  odd_frames: aligned bases, rows padded to even pitches of
    136 and 140 elements and odd frame strides, so the even frames keep pixel pairs 4-byte aligned and the odd ones do
    not.  Otherwise odd pitches (137, 141) and bases (element 3), even frame strides.  blur takes its general kernel
    whenever any frame is unaligned, and stencil_chain may take 32-bit accesses only on frames that allow them; samples
    outside the output's region keep their values."""
    import torch
    n, h, w = 6, 53, 131
    a = 2 if kind == "blur" else 0
    in_pitch, out_pitch, offset = (136, 140, 0) if odd_frames else (137, 141, 3)
    in_fs = in_pitch * (h + a) + (1 if odd_frames else 3)
    out_fs = out_pitch * (h + 2) + (5 if odd_frames else 1)
    clip, vin, tout, vout = device_views(n, h, w, h + a, w + a, in_pitch, in_fs, out_pitch, out_fs, offset, 44)
    args = params(kind, 7)
    bo = hb.HalideBuffer.from_torch(vout)
    with kernels_run(hb) as ran:
        fns(kind)[0](hb.HalideBuffer.from_torch(vin), *args, bo)
        torch.cuda.synchronize()
    if kind == "blur":
        assert set(ran) == {"blur3x3_u16"}, ran
    got = vout.cpu().numpy()
    for k in range(n):
        assert_same(got[k], one_frame(hb, kind, clip[k], args), f"{kind} frame {k}")
    mask = torch.ones_like(tout, dtype=torch.bool)
    mask.as_strided((n, h, w), (out_fs, out_pitch, 1), offset).fill_(False)
    outside = tout.view(torch.int16)[mask].cpu().numpy().view(np.uint16)  # (torch has no uint16 indexing)
    assert (outside == GUARD).all(), "samples outside the output's region changed"


@pytest.mark.parametrize("fs_odd", [False, True])
def test_blur_kernel_choice_follows_every_frame(hb, fs_odd):
    """Aligned bases and even row pitches: the pair kernel when every frame stride is even too, the general kernel when
    the input's frame stride is odd (every other frame then starts on an odd element)."""
    import torch
    n, h, w = 5, 40, 300
    in_fs = 304 * 42 + (1 if fs_odd else 0)
    clip = clip_of((n, 42, 302), 8)
    tin = torch.zeros((in_fs * n + 8,), dtype=torch.uint16, device="cuda")
    vin = tin.as_strided((n, 42, 302), (in_fs, 304, 1), 0)
    vin.copy_(torch.from_numpy(clip).cuda())
    vout = torch.zeros((n, h, w), dtype=torch.uint16, device="cuda")
    with kernels_run(hb) as ran:
        fns("blur")[0](hb.HalideBuffer.from_torch(vin), hb.HalideBuffer.from_torch(vout))
        torch.cuda.synchronize()
    assert set(ran) == {"blur3x3_u16" if fs_odd else "blur3x3_u16_quad"}, ran
    got = vout.cpu().numpy()
    for k in range(n):
        assert_same(got[k], one_frame(hb, "blur", clip[k], ()), f"frame {k}")


def test_blur_forced_general(hb):
    """halide_b200_blur_force_general(1) routes aligned clips through the general kernel too."""
    l = hb.load_library()
    l.halide_b200_blur_force_general(1)
    try:
        for n, h, w in [(3, 66, 130), (8, 29, 37)]:
            ran = check_batch(hb, "blur", clip_of((n, h, w), n + h), ())
            assert set(ran) == {"blur3x3_u16"} and launches(ran) == 1, ran
    finally:
        l.halide_b200_blur_force_general(0)
    ran = check_batch(hb, "blur", clip_of((3, 66, 130), 3), ())
    assert set(ran) == {"blur3x3_u16_quad"}, ran


@pytest.mark.parametrize("kind", KINDS)
def test_samples_outside_the_output_keep_their_values(hb, kind):
    """The output is a crop, in x, y and frames, of a guard-filled device array."""
    import torch
    clip = clip_of((4, 43, 69), 3)
    full = torch.full((6, 47, 77), int(GUARD), dtype=torch.uint16, device="cuda")
    view = full[1:5, 2:43, 3:70]
    args = params(kind, 6)
    src = clip if kind == "blur" else clip[:, :41, :67]
    fns(kind)[0](hb.HalideBuffer.from_torch(torch.from_numpy(np.ascontiguousarray(src)).cuda()), *args,
                 hb.HalideBuffer.from_torch(view))
    torch.cuda.synchronize()
    got = full.cpu().numpy()
    for k in range(4):
        assert_same(got[1 + k, 2:43, 3:70], one_frame(hb, kind, src[k], args, (41, 67)), f"frame {k}")
    got[1:5, 2:43, 3:70] = GUARD
    assert (got == GUARD).all(), "samples outside the output changed"


# ---- depths, groups and grid z --------------------------------------------------------------------------------------

@pytest.mark.parametrize("s", [1, 2, 3, 4, 5, 7, 8, 9, 32, 33, 99, 100])
def test_stencils(hb, s):
    """Every launch-plan shape: one short launch, whole launches, one plane of scratch (5..8) and two (9 up).  A clip that
    fits one group takes ceil(S / 4) launches."""
    clip = clip_of((4, 37, 70), s)
    ran = check_batch(hb, "scs", clip, (s,))
    assert launches(ran) == -(-s // 4), ran
    assert set(ran) == {"stencil_chain_window"}, ran


@pytest.mark.parametrize("kind,s,n", [("sc", 32, 9), ("scs", 100, 7)])
def test_groups_of_frames(hb, kind, s, n):
    """3840 x 2160 frames: 7 a group at S = 32 (36 MB of scratch a frame), 6 at S = 100 (43 MB).  A clip of one group more
    than that runs in two groups, ceil(S / 4) launches each; every frame, those on both sides of the group boundary
    included, equals its one-frame call."""
    h, w = 2160, 3840
    g = frames_per_group(h, w, n, s)
    assert 1 < g < n < 2 * g
    args = params(kind, s)
    ran = check_batch(hb, kind, clip_of((n, h, w), s), args)
    assert launches(ran) == 2 * -(-s // 4), (g, ran)


def test_frames_too_large_for_a_group(hb):
    """7680 x 4320 at S = 100: one frame's two scratch planes (152 MB) leave no room for a second in the budget, so the
    frames run one at a time through the one-frame kernels, 25 launches each."""
    n, h, w, s = 2, 4320, 7680, 100
    assert frames_per_group(h, w, n, s) == 1
    ran = check_batch(hb, "scs", clip_of((n, h, w), 4320), (s,))
    assert launches(ran) == n * 25, ran


@pytest.mark.parametrize("kind,s", [("blur", None), ("scs", 4), ("sc", None)])
def test_more_frames_than_the_grid_z_extent(hb, kind, s):
    """65 537 frames of 8 x 8: more than one launch's grid z extent.  blur walks them in its one launch; stencil_chain
    runs them in groups.  The frames repeat seven distinct ones, so each output frame is checked against the one-frame
    result of its distinct frame, the frames around each multiple of 65 535 among them."""
    n, k = 65537, 7
    args = () if s is None else (s,)
    ih = 10 if kind == "blur" else 8
    distinct = clip_of((k, ih, ih), 65537)
    clip = np.ascontiguousarray(np.concatenate([distinct] * (n // k + 1))[:n])
    out = np.zeros((n, 8, 8), np.uint16)
    ran = run_batch(hb, kind, clip, out, args)
    assert launches(ran) == want_launches(kind, args, 8, 8, n), ran
    wants = [one_frame(hb, kind, distinct[j], args) for j in range(k)]
    for j in range(k):
        assert_same(out[j::k], np.broadcast_to(wants[j], out[j::k].shape), f"frames {j} mod {k}")
    g = MAX_GRID_Z if kind == "blur" else frames_per_group(8, 8, n, stages(kind, args))
    for b in range(g, n, g):
        for f in (b - 1, b):
            assert_same(out[f], wants[f % k], f"frame {f} at a group boundary")


# ---- against the oracle ---------------------------------------------------------------------------------------------

def test_clips_against_the_oracle(hb, oracle):
    """A clip of ragged frames at odd mins, frame by frame against oracle/oracle_blur.cpp and
    oracle/oracle_stencil_chain.cpp (S = 32 and S = 13)."""
    from halide_b200 import blur_video, stencil_chain_video
    clip = clip_of((3, 47, 83), 4783)
    out = np.zeros((3, 45, 81), np.uint16)
    bi, bo = hb.HalideBuffer.from_numpy(clip, (-3, 5, 0)), hb.HalideBuffer.from_numpy(out, (-3, 5, 0), host_dirty=False)
    blur_video.blur_batch(bi, bo)
    bo.copy_to_host()
    for k in range(3):
        assert_same(out[k], oracle.blur(clip[k], (45, 81), (-3, 5), (-3, 5)), f"blur frame {k}")
    for s in (32, 13):
        out = np.zeros((3, 51, 80), np.uint16)
        bi = hb.HalideBuffer.from_numpy(clip, (4, -7, 0))
        bo = hb.HalideBuffer.from_numpy(out, (1, -9, 0), host_dirty=False)
        if s == 32:
            stencil_chain_video.stencil_chain_batch(bi, bo)
        else:
            stencil_chain_video.stencil_chain_stencils_batch(bi, s, bo)
        bo.copy_to_host()
        for k in range(3):
            want = oracle.stencil_chain(clip[k], (51, 80), (4, -7), (1, -9), stencils=s)
            assert_same(out[k], want, f"stencil_chain S = {s} frame {k}")


# ---- concurrent callers ---------------------------------------------------------------------------------------------

def test_two_threads_on_two_streams(hb):
    """Two threads, each bound to a stream of its own, call blur_batch and stencil_chain_stencils_batch at the same time,
    three rounds each; every result equals the one-frame calls on its frames."""
    jobs = []
    for i, (kind, args) in enumerate([("blur", ()), ("scs", (13,)), ("scs", (6,)), ("blur", ())]):
        clip = clip_of((5, 97, 143), 500 + i)
        jobs.append((kind, clip, args, np.stack([one_frame(hb, kind, f, args) for f in clip])))
    l = hb.load_library()
    errors, mismatches = [], []

    def thread(i):
        s = l.halide_b200_stream_create()
        try:
            assert s, "halide_b200_stream_create failed"
            l.halide_b200_set_stream(s)
            mine = jobs[i::2]
            for rnd in range(3):
                for kind, clip, args, want in mine + mine[::-1]:
                    out = np.zeros_like(want)
                    bi, bo = hb.HalideBuffer.from_numpy(clip), hb.HalideBuffer.from_numpy(out, host_dirty=False)
                    fns(kind)[0](bi, *args, bo)
                    bo.copy_to_host()
                    if not np.array_equal(out, want):
                        mismatches.append(f"thread {i} round {rnd}: {kind} {args}")
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
