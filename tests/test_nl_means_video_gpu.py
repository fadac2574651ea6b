"""GPU tests of the batch and interleaved nl_means entry points (float32 and uint8).  Their contract:
- batch: output frame n is, bit for bit, what nl_means (nl_means_u8) gives on input frame n;
- interleaved: the result is, bit for bit, what the planar entry point gives on planar copies of the same buffers, and
  output samples outside channels [0, 3) (an RGBA frame's alpha) keep their values.
So every case runs the planar one-frame entry point frame by frame on planar copies and compares bit patterns (float32
as uint32).  Interleaved frames are numpy arrays [(n,) y, x, pitch], planar ones [(n,) c, y, x]."""
import ctypes
import inspect
import threading

import numpy as np
import pytest

from util import kernels_run, nl_means_variant

pytestmark = pytest.mark.gpu
SIGMA = 0.12
GUARD = {np.float32: np.float32(-7.5), np.uint8: np.uint8(0xA5)}
DTYPES = [np.float32, np.uint8]
ROUTES = [(3, 7, 0, True), (7, 7, 0, True), (5, 9, 0, False), (3, 7, 1, False)]  # patch, search, variant hook, window
ROUTE_IDS = ["3/7", "7/7", "5/9", "3/7-generic"]
VIDEO_ENTRIES = {"nl_means_batch", "nl_means_interleaved", "nl_means_interleaved_batch", "nl_means_u8_batch",
                 "nl_means_u8_interleaved", "nl_means_u8_interleaved_batch"}


def frame(shape, dtype, seed):
    rng = np.random.default_rng(seed)
    if dtype == np.uint8:
        return rng.integers(0, 256, shape, dtype=np.uint8)
    return rng.random(shape, dtype=np.float32)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same(got, want, what=""):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def entry(dtype, batch, interleaved):
    """The Python call site: halide_b200.filters for the planar one-frame entry points, else halide_b200.nl_means_video."""
    from halide_b200 import filters, nl_means_video
    name = "nl_means" + ("_u8" if dtype == np.uint8 else "") + ("_interleaved" if interleaved else "") + \
        ("_batch" if batch else "")
    return getattr(nl_means_video if batch or interleaved else filters, name)


def xyc(arr, interleaved):
    """The (x, y, c[, n]) view of a numpy array (see the module docstring)."""
    if interleaved:
        return arr.transpose((2, 0, 1) if arr.ndim == 3 else (0, 3, 1, 2))
    return arr


def run(hb, fn, inp, out, args, interleaved, in_mins=None, out_mins=None):
    """fn(input, *args, output) on numpy views; out is written in place."""
    bi = hb.HalideBuffer.from_numpy(xyc(inp, interleaved), in_mins)
    bo = hb.HalideBuffer.from_numpy(xyc(out, interleaved), out_mins, host_dirty=False)
    fn(bi, *args, bo)
    assert bo.device_dirty
    bo.copy_to_host()


def planar_frame(hb, inp, out_hw, args, in_mins=None, out_mins=None):
    """The planar one-frame entry point on a planar copy of one frame (inp planar [c, y, x]); returns [3, y, x]."""
    out = np.zeros((3,) + tuple(out_hw), inp.dtype)
    run(hb, entry(inp.dtype, False, False), np.ascontiguousarray(inp), out, args, False, in_mins, out_mins)
    return out


def check_interleaved(hb, inp, args, out_pitch=3, out_hw=None, in_mins=None, out_mins=None, kernel=None):
    """The interleaved entry point on inp ([(n,) y, x, pitch] view) into channels [0, 3) of a guard-filled output of
    out_pitch samples per pixel, against the planar one-frame entry point frame by frame on planar copies.  Returns the
    output's channels."""
    batch = inp.ndim == 4
    hw = inp.shape[-3:-1] if out_hw is None else tuple(out_hw)
    n = inp.shape[:1] if batch else ()
    full = np.full(n + hw + (out_pitch,), GUARD[inp.dtype.type], inp.dtype)
    out = full[..., :3]
    with kernels_run(hb) as ran:
        run(hb, entry(inp.dtype, batch, True), inp, out, args, True, in_mins, out_mins)
    assert sum(c for c, _ in ran.values()) == 1 and (kernel is None or set(ran) == {kernel}), ran
    frames = list(inp) if batch else [inp]
    outs = list(out) if batch else [out]
    fm = lambda m: None if m is None else m[:3]  # noqa: E731  (a frame's mins)
    for k, (f, o) in enumerate(zip(frames, outs)):
        want = planar_frame(hb, np.moveaxis(f, -1, 0), hw, args, fm(in_mins), fm(out_mins))
        assert_same(np.moveaxis(o, -1, 0), want, f"frame {k} args {args} pitch {inp.shape[-1]}->{out_pitch}")
    assert (bits(full[..., 3:]) == bits(GUARD[inp.dtype.type])).all(), "samples outside channels [0, 3) changed"
    return out


def check_batch(hb, inp, args, out_n=None, in_n0=0, out_n0=0, out_hw=None, xy_in_mins=(0, 0, 0), xy_out_mins=(0, 0, 0),
                kernel=None):
    """The planar batch entry point on inp ([n, c, y, x], any view) into out_n frames starting at frame out_n0 (input frames
    start at in_n0), against the one-frame entry point on each input frame the output frame reads."""
    out_n = inp.shape[0] if out_n is None else out_n
    hw = inp.shape[-2:] if out_hw is None else tuple(out_hw)
    out = np.zeros((out_n, 3) + hw, inp.dtype)
    with kernels_run(hb) as ran:
        run(hb, entry(inp.dtype, True, False), inp, out, args, False, tuple(xy_in_mins) + (in_n0,),
            tuple(xy_out_mins) + (out_n0,))
    assert sum(c for c, _ in ran.values()) == 1 and (kernel is None or set(ran) == {kernel}), ran
    for k in range(out_n):
        want = planar_frame(hb, inp[out_n0 + k - in_n0], hw, args, xy_in_mins, xy_out_mins)
        assert_same(out[k], want, f"frame {k} args {args}")
    return out


# ---- interleaved = planar on planar copies ---------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("patch,search,hook,window", ROUTES, ids=ROUTE_IDS)
@pytest.mark.parametrize("in_pitch,in_c,out_pitch", [(3, 3, 3), (4, 4, 3), (3, 3, 4), (6, 3, 5), (1, 1, 3)],
                         ids=["rgb", "rgba-in", "rgba-out", "pitch6-to-5", "one-channel"])
def test_interleaved_pitches_and_routes(hb, dtype, patch, search, hook, window, in_pitch, in_c, out_pitch):
    """RGB, an RGBA input, an RGBA output whose alpha keeps its guard, a pitch above 4 on both sides, a 1-channel input
    of pitch 1; every kernel route."""
    img = frame((53, 71, in_pitch), dtype, in_pitch * 100 + patch * 10 + search)[..., :in_c]
    with nl_means_variant(hb, hook):
        check_interleaved(hb, img, (patch, search, SIGMA), out_pitch, kernel="nl_means_window" if window else "nl_means")


@pytest.mark.parametrize("dtype", DTYPES)
def test_rgba_input_alpha_is_never_read(hb, dtype):
    """Two RGBA inputs that differ only in alpha give the same bytes."""
    img = frame((40, 57, 4), dtype, 5)
    a = check_interleaved(hb, img[..., :3].copy(), (3, 7, SIGMA))
    img2 = img.copy()
    img2[..., 3] = frame((40, 57), dtype, 6)
    b = check_interleaved(hb, img2, (3, 7, SIGMA))
    c = check_interleaved(hb, img, (3, 7, SIGMA))
    assert_same(b, c, "alpha changed the result")
    assert_same(a, c, "RGB and RGBA inputs differ")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("hook", [0, 1])
def test_interleaved_mins_crops_odd_widths_unaligned_bases(hb, dtype, hook):
    big = frame((120, 181, 4), dtype, 21 + hook)
    with nl_means_variant(hb, hook):
        # padded rows and an odd width, nonzero mins on both sides, input larger than the output
        check_interleaved(hb, big[7:107, 3:176, :3], (3, 7, SIGMA), in_mins=(-5, 3, 0), out_mins=(-2, 5, 0),
                          out_hw=(91, 167))
        # a base 546 samples into a dense RGB array (2 bytes off 4-byte alignment for uint8), an input away from the
        # output (clamped), an RGBA output
        rgb = np.ascontiguousarray(big[..., :3])
        check_interleaved(hb, rgb[1:50, 1:60], (7, 7, SIGMA), out_pitch=4, in_mins=(40, 30, 0), out_mins=(0, 0, 0),
                          out_hw=(61, 77))
        # input channels starting at 1: channels 0, 1, 2 clamp to 1, 1, 2
        check_interleaved(hb, big[:33, :47, 1:3], (5, 9, SIGMA), in_mins=(0, 0, 1), out_mins=(0, 0, 0))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("patch,search,hook,window", ROUTES, ids=ROUTE_IDS)
def test_interleaved_batches(hb, dtype, patch, search, hook, window):
    clip = frame((3, 37, 66, 4), dtype, patch + search + hook)
    with nl_means_variant(hb, hook):
        check_interleaved(hb, clip[..., :3], (patch, search, SIGMA), out_pitch=4,
                          kernel="nl_means_window" if window else "nl_means")
        # frame mins: output frames 0..1 read input frames 0..1 of an input whose frames start at -1 (indices 1..2)
        inp = clip[..., :3]
        out = np.full((2, 37, 66, 3), GUARD[dtype], dtype)
        run(hb, entry(dtype, True, True), inp, out, (patch, search, SIGMA), True, (0, 0, 0, -1), (0, 0, 0, 0))
        for k in range(2):
            want = planar_frame(hb, np.moveaxis(inp[k + 1], -1, 0), (37, 66), (patch, search, SIGMA))
            assert_same(np.moveaxis(out[k], -1, 0), want, f"shifted frame {k}")


# ---- batch = frame by frame ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("patch,search,hook,window", ROUTES, ids=ROUTE_IDS)
@pytest.mark.parametrize("n", [1, 8])
def test_batches(hb, dtype, patch, search, hook, window, n):
    clip = frame((n, 3, 45, 70), dtype, n * 10 + patch + search + hook)
    with nl_means_variant(hb, hook):
        check_batch(hb, clip, (patch, search, SIGMA), kernel="nl_means_window" if window else "nl_means")


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_frame_mins_and_spare_input_frames(hb, dtype):
    clip = frame((7, 4, 50, 61), dtype, 77)
    # input frames [-2, 5), output frames [0, 4): output frame k reads input frame k (index k + 2)
    check_batch(hb, clip, (3, 7, SIGMA), out_n=4, in_n0=-2, out_n0=0)
    # x / y mins, a 4-channel input, an output crop, input frames [3, 10) and output frames [5, 8)
    check_batch(hb, clip, (7, 7, SIGMA), out_n=3, in_n0=3, out_n0=5, out_hw=(41, 53), xy_in_mins=(-4, 2, 0),
                xy_out_mins=(-1, 4, 0))


@pytest.mark.parametrize("dtype", DTYPES)
def test_reversed_and_broadcast_bursts(hb, dtype):
    clip = frame((5, 3, 38, 59), dtype, 91)
    check_batch(hb, clip[::-1], (3, 7, SIGMA))                                      # negative frame stride
    check_batch(hb, np.broadcast_to(clip[2], (4,) + clip.shape[1:]), (5, 9, SIGMA))  # frame stride 0


@pytest.mark.parametrize("dtype,interleaved", [(np.float32, False), (np.uint8, True)])
def test_more_frames_than_the_grid_z_extent(hb, dtype, interleaved):
    """65 537 tiny frames in one launch: the blocks walk frames beyond the grid's z limit.  The frames repeat seven
    distinct ones, so each output frame is checked against the one-frame result of its distinct frame."""
    n, k = 65537, 7
    distinct = frame((k, 5, 6, 3) if interleaved else (k, 3, 5, 6), dtype, 65537)
    clip = np.ascontiguousarray(np.concatenate([distinct] * (n // k + 1))[:n])
    out = np.zeros(clip.shape, dtype)
    with kernels_run(hb) as ran:
        run(hb, entry(dtype, True, interleaved), clip, out, (3, 7, SIGMA), interleaved)
    assert ran["nl_means_window"][0] == 1, ran
    for j in range(k):
        f = np.moveaxis(distinct[j], -1, 0) if interleaved else distinct[j]
        want = planar_frame(hb, f, (5, 6), (3, 7, SIGMA))
        got = np.moveaxis(out[j::k], -1, 1) if interleaved else out[j::k]
        assert_same(got, np.broadcast_to(want, got.shape), f"frames {j} mod {k}")


def test_batch_against_the_oracle(hb, oracle):
    clip = frame((3, 3, 41, 57), np.float32, 5)
    for patch, search, sigma in [(3, 7, 0.12), (7, 7, 0.3), (5, 9, 1.0)]:
        out = np.zeros_like(clip)
        run(hb, hb.nl_means_video.nl_means_batch, clip, out, (patch, search, sigma), False)
        for k in range(3):
            assert_same(out[k], oracle.nl_means(clip[k], patch, search, sigma), f"oracle frame {k} {patch}/{search}")
        il = np.zeros((3, 41, 57, 3), np.float32)
        run(hb, hb.nl_means_video.nl_means_interleaved_batch, np.ascontiguousarray(np.moveaxis(clip, 1, -1)), il,
            (patch, search, sigma), True)
        assert_same(np.moveaxis(il, -1, 1), out, "interleaved batch")


# ---- torch sources ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", ["float32", "uint8"])
def test_torch_clips_planar_and_channels_last(hb, dtype):
    """A device-resident (N, 3, H, W) tensor through the planar batch entry point, and the same clip in channels_last
    memory format through the interleaved one, on torch's current stream; against the one-frame entry point."""
    import torch
    from halide_b200 import HalideBuffer
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    np_clip = frame((4, 3, 97, 143), np.dtype(dtype).type, 12)
    want = np.stack([planar_frame(hb, f, (97, 143), (3, 7, SIGMA)) for f in np_clip])
    try:
        l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        x = torch.from_numpy(np_clip).cuda()
        y = torch.zeros_like(x)
        entry(np.dtype(dtype).type, True, False)(HalideBuffer.from_torch(x), 3, 7, SIGMA, HalideBuffer.from_torch(y))
        assert_same(y.cpu().numpy(), want, "planar device clip")
        xc = x.contiguous(memory_format=torch.channels_last)
        yc = torch.zeros_like(x).contiguous(memory_format=torch.channels_last)
        bi, bo = HalideBuffer.from_torch(xc), HalideBuffer.from_torch(yc)
        assert bi.shape()[2] == (0, 3, 1) and bo.shape()[0][2] == 3
        entry(np.dtype(dtype).type, True, True)(bi, 3, 7, SIGMA, bo)
        assert_same(yc.contiguous().cpu().numpy(), want, "channels_last device clip")
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
        torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", DTYPES)
def test_numpy_hwc_photo(hb, dtype):
    """A host (H, W, 3) array, as PIL or OpenCV return it, through HalideBuffer.from_numpy(arr.transpose(2, 0, 1))."""
    photo = frame((211, 307, 3), dtype, 8)
    out = np.zeros_like(photo)
    fn = entry(dtype, False, True)
    bi = hb.HalideBuffer.from_numpy(photo.transpose(2, 0, 1))
    bo = hb.HalideBuffer.from_numpy(out.transpose(2, 0, 1), host_dirty=False)
    fn(bi, 7, 7, SIGMA, bo)
    bo.copy_to_host()
    want = planar_frame(hb, np.ascontiguousarray(photo.transpose(2, 0, 1)), (211, 307), (7, 7, SIGMA))
    assert_same(out.transpose(2, 0, 1), want, "numpy HWC photo")


# ---- concurrent callers ----------------------------------------------------------------------------------------------

def video_jobs():
    """(name, fn, input view, output shape, dtype, interleaved, args) covering the six entry points."""
    jobs = []
    for dtype in DTYPES:
        for batch in (False, True):
            for il in (False, True):
                if not batch and not il:
                    continue
                shape = ((3,) if batch else ()) + ((49, 75, 3) if il else (3, 49, 75))
                inp = frame(shape, dtype, len(jobs) + 300)
                jobs.append((f"{np.dtype(dtype).name} batch={batch} il={il}", entry(dtype, batch, il), inp, dtype,
                             il, (3, 7, SIGMA) if len(jobs) % 2 else (5, 9, 0.3)))
    return jobs


def test_two_threads_on_two_streams_get_the_serial_bytes(hb):
    jobs = video_jobs()

    def one(job):
        _, fn, inp, dt, il, args = job
        out = np.zeros(inp.shape, dt)
        run(hb, fn, inp, out, args, il)
        return out

    serial = [one(j) for j in jobs]
    l = hb.load_library()
    errors, mismatches = [], []

    def thread(i):
        s = l.halide_b200_stream_create()
        try:
            assert s, "halide_b200_stream_create failed"
            l.halide_b200_set_stream(s)
            order = np.random.default_rng(i).permutation(len(jobs))
            for rnd in range(3):
                for k in order:
                    if not np.array_equal(bits(one(jobs[k])), bits(serial[k])):
                        mismatches.append(f"thread {i} round {rnd}: {jobs[k][0]}")
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


def test_threaded_jobs_cover_every_entry_point_of_the_module():
    """Every public function of halide_b200.nl_means_video runs in the threaded test above."""
    from halide_b200 import nl_means_video
    public = {n for n, f in inspect.getmembers(nl_means_video, inspect.isfunction)
              if f.__module__ == nl_means_video.__name__ and not n.startswith("_")}
    assert public == VIDEO_ENTRIES == {fn.__name__ for _, fn, *_ in video_jobs()}
