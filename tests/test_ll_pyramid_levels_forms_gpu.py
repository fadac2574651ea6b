"""GPU tests of the seven pyramid_levels forms of local_laplacian (batch, 8-bit and interleaved, in every combination):
every depth J in [1, 20] on every form against halide_b200_local_laplacian_pyramid_levels on planar uint16 copies (which
tests/test_ll_pyramid_levels_gpu.py pins to the oracle) and a subset against the oracle itself; batches of distinct
frames, reordered, negative and zero frame strides, deep batches whose levels past the eighth get launches of their own
or all run in the fused tail; the J = 1 tone kernel's forms; J = 8 against the fixed-depth entry points, byte for byte and
launch for launch; and calls on delayed and concurrent streams."""
import ctypes
import threading

import numpy as np
import pytest

import ll_bordered
from util import kernels_run, smooth_u16_frame, u16_frame

pytestmark = pytest.mark.gpu

# suffix -> (element type, batch, interleaved)
FORMS = {
    "_batch": (np.uint16, True, False),
    "_u8": (np.uint8, False, False),
    "_u8_batch": (np.uint8, True, False),
    "_interleaved": (np.uint16, False, True),
    "_interleaved_batch": (np.uint16, True, True),
    "_u8_interleaved": (np.uint8, False, True),
    "_u8_interleaved_batch": (np.uint8, True, True),
}
PARAMS = [(levels, 1.0 / (levels - 1), beta) for levels in (8, 3, 5) for beta in (1.0, 0.5)]


def to_u16(a):
    return a.astype(np.uint16) * np.uint16(257) if a.dtype == np.uint8 else a


def to_u8(w):
    return (((w.astype(np.uint32) + 128) * 255 + 255) >> 16).astype(np.uint8)


def frames(suffix, n, h, w, seed, c=3):
    """n distinct (c, h, w) frames of the form's element type, as one [n, c, h, w] array."""
    t = FORMS[suffix][0]
    out = np.stack([(smooth_u16_frame((c, h, w), seed + i) if (seed + i) % 2 else u16_frame((c, h, w), seed + i)) for i in range(n)])
    return (out >> 8).astype(np.uint8) if t == np.uint8 else out


def layout(arr, il, pitch=None):
    """[n, c, h, w] (or [c, h, w]) samples as a numpy view the filter's buffer describes: planar as is, interleaved with
    channels adjacent and the given pixel pitch (the samples past the channels hold a sentinel)."""
    if not il:
        return arr
    c = arr.shape[-3]
    pitch = pitch or c
    lead = arr.shape[:-3]
    back = np.full(lead + arr.shape[-2:] + (pitch,), 0xA5, arr.dtype)
    back[..., :c] = np.moveaxis(arr, -3, -1)
    view = back[..., :c]
    return np.moveaxis(view, -1, -3), back


def run_form(hb, suffix, x, J, levels, alpha, beta, out_pitch=None, in_pitch=None):
    """The form on [n, c, h, w] frames x (a batch form) or x[0] (a one-frame form): the output as [n, c, h, w] (and the
    interleaved output's backing array, pitch included)."""
    t, batch, il = FORMS[suffix]
    src = x if batch else x[0]
    out = np.zeros_like(src)
    if il:
        vi, _ = layout(src, True, in_pitch)
        vo, back = layout(out, True, out_pitch)
    else:
        vi, vo, back = src, out, None
    bi = hb.HalideBuffer.from_numpy(vi)
    bo = hb.HalideBuffer.from_numpy(vo, host_dirty=False)
    getattr(hb.local_laplacian_depth, "local_laplacian_pyramid_levels" + suffix)(bi, J, levels, alpha, beta, bo)
    bo.copy_to_host()
    got = np.ascontiguousarray(vo)
    return (got if batch else got[None]), back


def reference(hb, x, J, levels, alpha, beta):
    """halide_b200_local_laplacian_pyramid_levels frame by frame on planar uint16 copies (8-bit frames widened and the
    result narrowed as the 8-bit entry points convert)."""
    res = []
    for f in x:
        src = np.ascontiguousarray(to_u16(f))
        out = np.zeros_like(src)
        bi, bo = hb.HalideBuffer.from_numpy(src), hb.HalideBuffer.from_numpy(out, host_dirty=False)
        hb.filters.local_laplacian_pyramid_levels(bi, J, levels, alpha, beta, bo)
        bo.copy_to_host()
        res.append(to_u8(out) if x.dtype == np.uint8 else out)
    return np.stack(res)


def oracle_ref(oracle, x, J, levels, alpha, beta):
    evaluate = ll_bordered.local_laplacian if J > 11 else oracle.local_laplacian
    res = [evaluate(np.ascontiguousarray(to_u16(f)), levels, alpha, beta, pyramid_levels=J) for f in x]
    return np.stack([to_u8(r) if x.dtype == np.uint8 else r for r in res])


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b)


# ---- every depth on every form ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("J", range(1, 21))
def test_every_depth(hb, J):
    """Every form at depth J, on both sizes, every level count and both betas (the odd size takes half of PARAMS, the
    even size the other half).  The forms of one element type share their frames, so one reference serves them all."""
    for i, (W, H) in enumerate([(17, 9), (32, 20)]):
        for t in (np.uint16, np.uint8):
            forms = [s for s, f in FORMS.items() if f[0] == t]
            x = frames(forms[0], 2, H, W, 10 * J + W)
            for levels, alpha, beta in PARAMS[i::2]:
                want = reference(hb, x, J, levels, alpha, beta)
                for suffix in forms:
                    got, _ = run_form(hb, suffix, x, J, levels, alpha, beta)
                    ref = want if FORMS[suffix][1] else want[:1]
                    assert same(got, ref), (suffix, W, H, levels, beta, int(np.count_nonzero(got != ref)))


@pytest.mark.parametrize("suffix,J", [("_u8_batch", 1), ("_interleaved_batch", 2), ("_u8_interleaved", 3), ("_u8_batch", 8),
                                      ("_interleaved_batch", 11), ("_u8_interleaved", 12)])
def test_against_the_oracle(hb, oracle, suffix, J):
    x = frames(suffix, 2, 19, 27, J)
    for levels, alpha, beta in [(8, 1.0 / 7.0, 1.0), (5, 0.25, 0.5)]:
        got, _ = run_form(hb, suffix, x, J, levels, alpha, beta)
        want = oracle_ref(oracle, x if FORMS[suffix][1] else x[:1], J, levels, alpha, beta)
        assert same(got, want), (levels, int(np.count_nonzero(got != want)))


# ---- batches ------------------------------------------------------------------------------------------------------------

BATCHES = [s for s, (_, batch, _) in FORMS.items() if batch]


@pytest.mark.parametrize("J", [1, 2, 9, 14])
@pytest.mark.parametrize("suffix", BATCHES)
@pytest.mark.parametrize("n", [1, 2, 3])
def test_batch_sizes(hb, suffix, J, n):
    x = frames(suffix, n, 37, 45, 3 * J + n)
    got, _ = run_form(hb, suffix, x, J, 8, 1.0 / 7.0, 0.5)
    assert same(got, reference(hb, x, J, 8, 1.0 / 7.0, 0.5))


@pytest.mark.parametrize("J", [1, 2, 4, 10, 16])
@pytest.mark.parametrize("suffix", ["_batch", "_u8_batch"])
def test_frame_strides(hb, suffix, J):
    """Planar batches whose frames lie in reverse order (a negative frame stride), interleaved with the channels (the
    frame stride below the channel stride), or are one frame repeated (a zero input frame stride)."""
    x = frames(suffix, 3, 23, 29, J)
    want = reference(hb, x, J, 8, 1.0 / 7.0, 1.0)
    fn = getattr(hb.local_laplacian_depth, "local_laplacian_pyramid_levels" + suffix)

    def call(vi, vo):
        bi, bo = hb.HalideBuffer.from_numpy(vi), hb.HalideBuffer.from_numpy(vo, host_dirty=False)
        fn(bi, J, 8, 1.0 / 7.0, 1.0, bo)
        bo.copy_to_host()

    # negative: both buffers walk their frames backwards
    rev_in, rev_out = np.ascontiguousarray(x[::-1])[::-1], np.zeros_like(x)[::-1]
    call(rev_in, rev_out)
    assert same(np.ascontiguousarray(rev_out), want)
    # reordered: memory (c, n, h, w), described as (x, y, c, n)
    cn_in = np.ascontiguousarray(x.transpose(1, 0, 2, 3)).transpose(1, 0, 2, 3)
    cn_out = np.zeros((3,) + x.shape[:1] + x.shape[2:], x.dtype).transpose(1, 0, 2, 3)
    call(cn_in, cn_out)
    assert same(np.ascontiguousarray(cn_out), want)
    # zero: frame 1 broadcast over three output frames
    out = np.zeros_like(x)
    call(np.broadcast_to(x[1], x.shape), out)
    assert all(same(out[i], want[1]) for i in range(3))


def test_deep_batch_with_levels_of_their_own(hb):
    """Two 2^22 x 1 frames at J = 14: levels 8 and up are too big for the fused tail, so they get ll_down_rows / ll_up2
    launches with real frame strides past the 8 slots of the per-level stride arrays.  (The level arrays do not depend on
    the frame's element type or layout: one form stands for all.)"""
    suffix = "_u8_interleaved_batch"
    l = hb.load_library()
    assert l.halide_b200_ll_last_own_level(1 << 22, 1, 14) >= 8
    x = frames(suffix, 2, 1, 1 << 22, 5)
    with kernels_run(hb) as ran:
        got, _ = run_form(hb, suffix, x, 14, 8, 1.0 / 7.0, 1.0)
    assert ran.get("ll_down_rows", (0,))[0] >= 6, ran
    want = reference(hb, x, 14, 8, 1.0 / 7.0, 1.0)
    assert same(got, want), int(np.count_nonzero(got != want))


@pytest.mark.parametrize("levels", [8, 3])
@pytest.mark.parametrize("suffix", ["_batch", "_u8_interleaved_batch"])
def test_deep_batch_in_the_fused_tail(hb, suffix, levels):
    """Three small frames at J = 13: every level from 2 on runs in one ll_coarse_fused launch (the deep batch
    instantiation, with the strides of every level)."""
    x = frames(suffix, 3, 40, 56, levels)
    with kernels_run(hb) as ran:
        got, _ = run_form(hb, suffix, x, 13, levels, 1.0 / (levels - 1), 1.0)
    assert ran.get("ll_coarse_fused", (0,))[0] == 1, ran
    assert "ll_down_rows" not in ran and "ll_down" not in ran, ran
    assert same(got, reference(hb, x, 13, levels, 1.0 / (levels - 1), 1.0))


# ---- J = 1 --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("generic", [0, 16])
@pytest.mark.parametrize("suffix,in_pitch,out_pitch", [
    ("_u8", None, None), ("_batch", None, None), ("_u8_batch", None, None),
    ("_interleaved", 3, 3), ("_interleaved", 4, 3), ("_interleaved", 4, 4), ("_interleaved_batch", 4, 4),
    ("_u8_interleaved", 3, 3), ("_u8_interleaved", 4, 3), ("_u8_interleaved", 4, 4), ("_u8_interleaved_batch", 3, 3),
    ("_u8_interleaved_batch", 4, 3), ("_interleaved", 5, 6),
])
def test_tone_forms(hb, suffix, in_pitch, out_pitch, generic):
    """J = 1 runs only ll_tone: its aligned forms (whole 8-pixel units on a 64-pixel-wide frame, row tails on a 67-wide
    one) and its general form (the force-generic hook's 16, or pitches 5 / 6).  An interleaved output's samples past its
    channels keep the sentinel."""
    l = hb.load_library()
    for W in (64, 67):
        x = frames(suffix, 2, 13, W, W)
        if in_pitch == 4 or in_pitch == 5:  # the input describes every sample of its pixels
            x = np.concatenate([x, frames(suffix, 2, 13, W, W + 1)[:, :in_pitch - 3]], axis=1)
        l.halide_b200_ll_force_generic(generic)
        try:
            with kernels_run(hb) as ran:
                got, back = run_form_channels(hb, suffix, x, in_pitch, out_pitch)
        finally:
            l.halide_b200_ll_force_generic(0)
        assert set(ran) == {"ll_tone"} or set(ran) == {"ll_tone", "ll_lut"}, ran
        want = reference(hb, x[:, :3] if FORMS[suffix][1] else x[:1, :3], 1, 8, 1.0 / 7.0, 0.5)
        assert same(got, want), (W, int(np.count_nonzero(got != want)))
        if back is not None and out_pitch > 3:
            assert (back[..., 3:] == 0xA5).all(), "samples past the output's channels were written"


def run_form_channels(hb, suffix, x, in_pitch, out_pitch):
    """run_form with an input of all of x's channels (its pitch) and an output of channels [0, 3)."""
    t, batch, il = FORMS[suffix]
    src = x if batch else x[0]
    out = np.zeros(src.shape[:-3] + (3,) + src.shape[-2:], src.dtype)
    if il:
        vi, _ = layout(src, True, in_pitch)
        vo, back = layout(out, True, out_pitch)
    else:
        vi, vo, back = src, out, None
    bi, bo = hb.HalideBuffer.from_numpy(vi), hb.HalideBuffer.from_numpy(vo, host_dirty=False)
    getattr(hb.local_laplacian_depth, "local_laplacian_pyramid_levels" + suffix)(bi, 1, 8, 1.0 / 7.0, 0.5, bo)
    bo.copy_to_host()
    got = np.ascontiguousarray(vo)
    return (got if batch else got[None]), back


@pytest.mark.parametrize("suffix", ["_u8", "_u8_interleaved_batch", "_interleaved"])
def test_tone_tables_above_48k(hb, suffix):
    """levels 26 and 30: the remap table ll_tone stages is more than 48 KB, in turn."""
    x = frames(suffix, 2, 21, 40, 26)
    for levels in (30, 26, 30):
        alpha = 1.0 / (levels - 1)
        with kernels_run(hb) as ran:
            got, _ = run_form(hb, suffix, x, 1, levels, alpha, 1.0)
        assert "ll_tone" in ran, ran
        assert same(got, reference(hb, x if FORMS[suffix][1] else x[:1], 1, levels, alpha, 1.0)), levels


# ---- J = 8 is the fixed-depth form ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("suffix", list(FORMS))
@pytest.mark.parametrize("W,H,levels", [(480, 270, 8), (255, 129, 3)])
def test_depth_8_is_the_fixed_depth_form(hb, suffix, W, H, levels):
    t, batch, il = FORMS[suffix]
    x = frames(suffix, 2, H, W, W)
    src = x if batch else x[0]
    alpha = 1.0 / (levels - 1)
    vi = layout(src, True)[0] if il else src

    def call(fn, *j):
        out = np.zeros_like(src)
        vo = layout(out, True)[0] if il else out
        bi, bo = hb.HalideBuffer.from_numpy(vi), hb.HalideBuffer.from_numpy(vo, host_dirty=False)
        fn(bi, *j, levels, alpha, 1.0, bo)  # (the remap table exists for the timed calls)
        with kernels_run(hb) as ran:
            fn(bi, *j, levels, alpha, 1.0, bo)
        bo.copy_to_host()
        return np.ascontiguousarray(vo), {k: v[0] for k, v in ran.items()}

    a, ran_a = call(getattr(hb.filters, "local_laplacian" + suffix))
    b, ran_b = call(getattr(hb.local_laplacian_depth, "local_laplacian_pyramid_levels" + suffix), 8)
    assert same(a, b)
    assert ran_a == ran_b


# ---- streams and concurrency ----------------------------------------------------------------------------------------------

SEQ = [("_u8_batch", 1), ("_interleaved", 14), ("_batch", 2), ("_u8_interleaved_batch", 9), ("_u8", 20), ("_interleaved_batch", 1),
       ("_u8_interleaved", 3), ("_batch", 11), ("_u8_batch", 8)]


def test_back_to_back_forms_and_depths(hb):
    xs = {s: frames(s, 3, 41, 53, 7) for s in FORMS}
    fresh = {(s, J): run_form(hb, s, xs[s], J, 5, 0.25, 0.5)[0] for s, J in reversed(SEQ)}
    for _ in range(2):
        for s, J in SEQ:
            assert same(run_form(hb, s, xs[s], J, 5, 0.25, 0.5)[0], fresh[s, J]), (s, J)


def _device(x, il):
    """uint8 [n, c, h, w] frames as a device tensor, channels_last (pixel-interleaved) for an interleaved form."""
    import torch
    t = torch.from_numpy(x).cuda()
    return t.contiguous(memory_format=torch.channels_last) if il else t


def test_calls_wait_for_the_callers_stream(hb):
    """A call on a stream busy with a sleep, its input written and its output cleared after the sleep: a launch or copy
    that did not wait for the caller's stream would read the sentinel input or be overwritten by the sentinel fill.
    (uint8 clips: the device tensors are filled and copied by torch.)"""
    suffix, J = "_u8_interleaved_batch", 14
    import torch
    t, batch, il = FORMS[suffix]
    x = frames(suffix, 3, 270, 480, J)
    want = reference(hb, x, J, 8, 1.0 / 7.0, 1.0)
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    stream = torch.cuda.Stream()
    real = _device(x, il)
    hb.capi.halide_cuda_release_unused_device_allocations(None)
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    try:
        l.halide_b200_set_stream(ctypes.c_void_p(stream.cuda_stream))
        with torch.cuda.stream(stream):
            inp, out = torch.empty_like(real), torch.empty_like(real)
            inp.fill_(0x55)
            torch.cuda._sleep(1 << 28)
            slept = torch.cuda.Event()
            slept.record(stream)
            inp.copy_(real)
            out.fill_(0x33)
            bi, bo = hb.HalideBuffer.from_torch(inp), hb.HalideBuffer.from_torch(out)
            getattr(hb.local_laplacian_depth, "local_laplacian_pyramid_levels" + suffix)(bi, J, 8, 1.0 / 7.0, 1.0, bo)
            clone = out.clone()
            sleeping = not slept.query()
        stream.synchronize()
        del bi, bo
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
    got = clone.contiguous().cpu().numpy()
    assert same(got, want), int(np.count_nonzero(got != want))
    assert sleeping, "the sleep had ended when the call was enqueued"


def test_two_callers_on_their_own_streams(hb):
    import torch
    jobs = [("_u8_interleaved_batch", 14), ("_batch", 3), ("_u8", 1), ("_interleaved_batch", 11), ("_u8_batch", 2),
            ("_interleaved", 20)]
    xs = {s: frames(s, 3, 67, 91, J) for s, J in jobs}
    serial = {(s, J): run_form(hb, s, xs[s], J, 8, 1.0 / 7.0, 0.5)[0] for s, J in jobs}
    errors = []

    def caller(order):
        l = hb.load_library()
        stream = torch.cuda.Stream()
        l.halide_b200_set_stream(ctypes.c_void_p(stream.cuda_stream))
        try:
            for _ in range(3):
                for s, J in order:
                    got = run_form(hb, s, xs[s], J, 8, 1.0 / 7.0, 0.5)[0]
                    if not same(got, serial[s, J]):
                        errors.append((s, J))
        except Exception as e:  # noqa: BLE001 (reported below)
            errors.append(repr(e))
        finally:
            l.halide_b200_set_stream(None)

    threads = [threading.Thread(target=caller, args=(o,)) for o in (jobs, jobs[::-1])]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
