"""GPU tests of the 8-bit local_laplacian entry points.  Their contract is the composition
    out8 = to_u8(local_laplacian(to_u16(in8)))
with the reference's element conversions (image_io.convert), so every case compares bit for bit against that composition
built from the uint16 GPU filter, and the small frames also against the oracle composed the same way.  The 8-bit inputs
here are numpy host buffers (copied to the device by the runtime, outputs read back with copy_to_host) unless a test
says otherwise."""
import ctypes
from contextlib import contextmanager

import numpy as np
import pytest

from halide_b200.image_io import convert
from util import kernels_run, run_local_laplacian, smooth_u16_frame

pytestmark = pytest.mark.gpu
ALPHA = 1.0 / 7.0


def u8_frame(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def smooth_u8_frame(shape, seed):
    return (smooth_u16_frame(shape, seed) >> 8).astype(np.uint8)


def run_u8(hb, inp, levels, alpha, beta, out=None, out_shape=None, in_mins=None, out_mins=None):
    """The 8-bit filter on numpy arrays (3-D: halide_b200_local_laplacian_u8, 4-D: the batch entry point)."""
    if out is None:
        out = np.zeros(inp.shape if out_shape is None else out_shape, np.uint8)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    (hb.filters.local_laplacian_u8 if inp.ndim == 3 else hb.filters.local_laplacian_u8_batch)(bi, levels, alpha, beta, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out


def composed(hb, inp, levels, alpha, beta, out_shape=None, in_mins=None, out_mins=None):
    """to_u8(uint16 GPU filter(to_u16(inp))) of one frame."""
    out16 = run_local_laplacian(hb, convert(inp, np.uint16), levels, alpha, beta, out_shape=out_shape, in_mins=in_mins,
                                out_mins=out_mins)
    return convert(out16, np.uint8)


def oracle_composed(oracle, inp, levels, alpha, beta, **kw):
    return convert(oracle.local_laplacian(convert(inp, np.uint16), levels, alpha, beta, **kw), np.uint8)


def assert_same(got, want, what=""):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


@contextmanager
def force_generic(hb, mask):
    l = hb.load_library()
    l.halide_b200_ll_force_generic(mask)
    try:
        yield
    finally:
        l.halide_b200_ll_force_generic(0)


def check(hb, oracle, img, levels=8, alpha=ALPHA, beta=1.0, with_oracle=True, **kw):
    got = run_u8(hb, img, levels, alpha, beta, **kw)
    assert_same(got, composed(hb, img, levels, alpha, beta, **kw), f"levels {levels} alpha {alpha} beta {beta}: uint16 GPU")
    if with_oracle:
        assert_same(got, oracle_composed(oracle, img, levels, alpha, beta, **kw), f"levels {levels} beta {beta}: oracle")
    return got


# ---- frame sizes, parameters, content -----------------------------------------------------------------------------

@pytest.mark.parametrize("w,h", [(67, 91), (517, 333)])
@pytest.mark.parametrize("levels,beta", [(8, 1.0), (8, 0.5), (5, 1.0), (5, 0.5), (2, 1.0), (2, 0.5)])
@pytest.mark.parametrize("smooth", [False, True])
def test_small_frames(hb, oracle, w, h, levels, beta, smooth):
    """levels 8 takes the fast kernels, 5 and 2 the generic ones; beta 1 and 0.5 are the two BETA1 instantiations."""
    img = (smooth_u8_frame if smooth else u8_frame)((3, h, w), w + h + levels)
    check(hb, oracle, img, levels, 1.0 / (levels - 1), beta)


@pytest.mark.parametrize("alpha", [0.0, 1.0 / 7.0, 1.0])
@pytest.mark.parametrize("beta", [1.0, 0.5])
def test_alpha(hb, oracle, alpha, beta):
    check(hb, oracle, u8_frame((3, 333, 517), 77), 8, alpha, beta)


@pytest.mark.parametrize("w,h,beta,smooth", [(1920, 1080, 1.0, False), (1920, 1080, 0.5, True), (3840, 2160, 1.0, False),
                                             (3840, 2160, 0.5, False), (3840, 2160, 1.0, True)])
def test_video_frames(hb, oracle, w, h, beta, smooth):
    img = (smooth_u8_frame if smooth else u8_frame)((3, h, w), w + int(smooth))
    check(hb, oracle, img, 8, ALPHA, beta, with_oracle=False)


def test_all_values_and_constant_frames(hb, oracle):
    """Every channel holds all 256 values (each channel in another order), and constant 0 and 255 frames: both ends of
    both conversions."""
    h, w = 64, 96
    rng = np.random.default_rng(5)
    img = np.stack([rng.permutation(np.tile(np.arange(256, dtype=np.uint8), h * w // 256)).reshape(h, w) for _ in range(3)])
    for c in range(3):
        assert len(np.unique(img[c])) == 256
    for beta in (1.0, 0.5):
        check(hb, oracle, img, 8, ALPHA, beta)
        check(hb, oracle, img, 5, 0.25, beta)
    for v in (0, 255):
        for levels in (8, 5):
            got = check(hb, oracle, np.full((3, h, w), v, np.uint8), levels, 1.0 / (levels - 1), 1.0)
            assert (got == v).all(), f"constant {v} frame changed by the filter"


# ---- bounds, channels and layouts ---------------------------------------------------------------------------------

@pytest.mark.parametrize("levels", [8, 5])
def test_mins_and_a_larger_input(hb, oracle, levels):
    """Negative and odd mins; the input is larger than the output in x, y and c (repeat_edge clamps at the input's own
    bounds)."""
    h, w = 71, 97
    img = u8_frame((4, h + 9, w + 14), 3)
    kw = dict(out_shape=(3, h, w), in_mins=(-5, 3, -1), out_mins=(-3, 5, 0))
    check(hb, oracle, img, levels, 1.0 / (levels - 1), 1.0, **kw)
    check(hb, oracle, img, levels, 1.0 / (levels - 1), 0.5, **kw)


def expected_kernels(mask, out_c):
    down = "ll_level1_generic" if mask & 1 else "ll_level1"
    final = "ll_final" if (mask & 4) or out_c > 3 else "ll_final2"
    return down, final


@pytest.mark.parametrize("in_c,out_c,out_c0", [(3, 1, 0), (3, 2, 1), (3, 1, 2), (1, 1, 0), (2, 2, 0), (2, 1, 1),
                                               (4, 4, 0), (4, 3, 1)])
@pytest.mark.parametrize("mask", [0, 4])
def test_channels(hb, oracle, in_c, out_c, out_c0, mask):
    """Output channel crops, 1- and 2-channel inputs, and 4 output channels (the generic final kernel)."""
    h, w = 53, 74
    img = u8_frame((in_c, h, w), 10 * in_c + out_c)
    with force_generic(hb, mask), kernels_run(hb) as ran:
        got = run_u8(hb, img, 8, ALPHA, 1.0, out_shape=(out_c, h, w), out_mins=(0, 0, out_c0))
    kw = dict(out_shape=(out_c, h, w), out_mins=(0, 0, out_c0))
    assert_same(got, composed(hb, img, 8, ALPHA, 1.0, **kw), "uint16 GPU")
    assert_same(got, oracle_composed(oracle, img, 8, ALPHA, 1.0, **kw), "oracle")
    down, final = expected_kernels(mask, out_c)
    assert down in ran and final in ran, sorted(ran)


def padded(a, row_pad):
    """A view of `a`'s values (c, h, w) whose rows are row_pad elements longer than dense."""
    c, h, w = a.shape
    pitch = w + row_pad
    base = np.zeros(c * h * pitch, np.uint8)
    v = np.lib.stride_tricks.as_strided(base, shape=a.shape, strides=(h * pitch, pitch, 1))
    v[...] = a
    return v


@pytest.mark.parametrize("w,row_pad", [
    (250, 6),   # rows 256 bytes apart: the TMA frame tile, staged level-1 words
    (250, 2),   # rows 252 bytes apart: aligned loads in the final kernel, staged level-1 words
    (250, 4),   # rows 254 bytes apart: aligned loads in the final kernel, unstaged level-1 pairs
    (250, 3),   # odd rows: the general-layout final kernel
    (256, 0),   # dense
])
@pytest.mark.parametrize("beta", [1.0, 0.5])
def test_padded_rows(hb, oracle, w, row_pad, beta):
    h = 150
    a = u8_frame((3, h, w), w + row_pad)
    want = composed(hb, a, 8, ALPHA, beta)
    out = padded(np.zeros_like(a), row_pad + 2)
    got = run_u8(hb, padded(a, row_pad), 8, ALPHA, beta, out=out)
    assert_same(np.ascontiguousarray(got), want, f"row pad {row_pad}")


@pytest.mark.parametrize("mask", [0, 64, 16])
@pytest.mark.parametrize("h,w,pad", [(80, 128, 0), (80, 128, 16), (57, 98, 3)])
def test_channel_stride_smaller_than_row_stride(hb, oracle, h, w, pad, mask):
    """Memory order (x, c, y): strides (1, 3W + pad, W), device buffers wrapped from torch.  The output's padding must
    stay untouched."""
    import torch
    from halide_b200 import HalideBuffer, filters
    pitch = 3 * w + pad
    img = u8_frame((3, h, w), h + w + pad)
    want = composed(hb, img, 8, ALPHA, 1.0)
    base = np.zeros(h * pitch, np.uint8)
    np.lib.stride_tricks.as_strided(base, shape=(3, h, w), strides=(w, pitch, 1))[...] = img
    t_in_base = torch.from_numpy(base).cuda()
    t_out_base = torch.zeros(h * pitch, dtype=torch.uint8, device="cuda")
    t_in = t_in_base.as_strided((3, h, w), (w, pitch, 1))
    t_out = t_out_base.as_strided((3, h, w), (w, pitch, 1))
    bi, bo = HalideBuffer.from_torch(t_in), HalideBuffer.from_torch(t_out)
    assert [d[2] for d in bi.shape()] == [1, pitch, w]
    with force_generic(hb, mask), kernels_run(hb) as ran:
        filters.local_laplacian_u8(bi, 8, ALPHA, 1.0, bo)
        bo.device_sync()
    torch.cuda.synchronize()
    out_base = t_out_base.cpu().numpy()
    got = np.lib.stride_tricks.as_strided(out_base, shape=(3, h, w), strides=(w, pitch, 1))
    assert_same(np.ascontiguousarray(got), want, f"pitch {pitch} mask {mask}")
    if pad:
        assert not out_base.reshape(h, pitch)[:, 3 * w:].any(), "the filter wrote into the row padding"
    assert "ll_level1" in ran and "ll_final2" in ran, sorted(ran)
    del bi, bo


@pytest.mark.parametrize("mask", [1, 2, 4, 8, 16, 64, 7, 1 | 8, 16 | 64])
def test_force_generic_masks(hb, oracle, mask):
    """Each hook bit routes the 8-bit call to the kernel it routes a uint16 call to: generic level 1 (1), generic
    up-sweep (2), generic final (4), no cooperative tail (8), general-layout final (16), no TMA frame tile (64)."""
    img = u8_frame((3, 131, 204), mask)
    want = composed(hb, img, 8, ALPHA, 1.0)
    with force_generic(hb, mask), kernels_run(hb) as ran:
        got = run_u8(hb, img, 8, ALPHA, 1.0)
    assert_same(got, want, f"mask {mask}")
    down, final = expected_kernels(mask, 3)
    assert down in ran and final in ran, sorted(ran)
    assert ("ll_coarse_fused" in ran) == (not mask & 8), sorted(ran)
    if mask & 8:  # (every level then has its own up-sweep launch: only generic ones under bit 2)
        assert ("ll_up2" in ran) != bool(mask & 2), sorted(ran)


# ---- batches -----------------------------------------------------------------------------------------------------

def make_batch(n, h, w, seed, c=3):
    """(n, c, h, w) uint8: frame k from its own seed; frame 1 (when there is one) constant per channel."""
    a = np.stack([u8_frame((c, h, w), 1000 * seed + k) for k in range(n)])
    if n >= 2:
        for ch in range(c):
            a[1, ch] = (80, 160, 35, 255)[ch % 4]
    return a


def strided_batch(a, row_pad=0, frame_pad=0):
    n, c, h, w = a.shape
    pitch = w + row_pad
    fs = c * h * pitch + frame_pad
    flat = np.zeros(n * fs, np.uint8)
    v = np.lib.stride_tricks.as_strided(flat, shape=a.shape, strides=(fs, h * pitch, pitch, 1))
    v[...] = a
    return v


def assert_frames(got, want, what=""):
    for k in range(got.shape[0]):
        assert_same(got[k], want[k], f"{what} frame {k}")


@pytest.mark.parametrize("n,w,h,levels,beta", [(1, 67, 91, 8, 1.0), (2, 67, 91, 8, 0.5), (3, 517, 333, 5, 1.0),
                                               (4, 200, 150, 8, 1.0), (5, 67, 91, 8, 1.0)])
def test_batches_match_single_calls_and_composition(hb, oracle, n, w, h, levels, beta):
    alpha = 1.0 / (levels - 1)
    a = make_batch(n, h, w, n * 31 + levels)
    got = run_u8(hb, a, levels, alpha, beta)
    assert_frames(got, np.stack([run_u8(hb, np.ascontiguousarray(a[k]), levels, alpha, beta) for k in range(n)]), "single")
    assert_frames(got, np.stack([composed(hb, a[k], levels, alpha, beta) for k in range(n)]), "uint16 GPU")
    if w * h < 40000:
        assert_frames(got, np.stack([oracle_composed(oracle, a[k], levels, alpha, beta) for k in range(n)]), "oracle")


@pytest.mark.parametrize("w,row_pad,frame_pad", [
    (256, 0, 0),    # frame stride a 16-byte multiple: the final kernel's 4-D TMA frame tile
    (250, 6, 0),    # padded rows, frame stride still a 16-byte multiple
    (256, 0, 4),    # frame stride a 4-byte multiple only: aligned loads without TMA
    (256, 0, 2),    # frame stride even only: aligned loads in the final kernel, unstaged level-1 pairs
    (250, 3, 5),    # odd row and frame strides: general addressing
])
def test_batch_strides(hb, w, row_pad, frame_pad):
    h = 150
    a = make_batch(3, h, w, w + row_pad + frame_pad)
    want = np.stack([composed(hb, a[k], 8, ALPHA, 1.0) for k in range(3)])
    out = strided_batch(np.zeros_like(a), row_pad + 2, frame_pad + 2)
    assert_frames(run_u8(hb, strided_batch(a, row_pad, frame_pad), 8, ALPHA, 1.0, out=out), want)


def test_batch_mins_and_a_larger_input(hb, oracle):
    """Negative mins in every dimension; the output takes frames 1..3 of the input's 5."""
    h, w = 71, 97
    inp = make_batch(5, h + 9, w + 14, 3, c=4)
    in_mins, out_mins = (-5, 3, -1, -2), (-2, 5, 0, -1)
    got = run_u8(hb, inp, 8, ALPHA, 1.0, out=np.zeros((3, 3, h, w), np.uint8), in_mins=in_mins, out_mins=out_mins)
    kw = dict(out_shape=(3, h, w), in_mins=in_mins[:3], out_mins=out_mins[:3])
    assert_frames(got, np.stack([composed(hb, inp[k], 8, ALPHA, 1.0, **kw) for k in range(1, 4)]), "uint16 GPU")
    assert_frames(got, np.stack([oracle_composed(oracle, np.ascontiguousarray(inp[k]), 8, ALPHA, 1.0, **kw)
                                 for k in range(1, 4)]), "oracle")


# ---- device-resident frames ----------------------------------------------------------------------------------------

def torch_to_u16(t8):
    """to_u16 of a uint8 device tensor, as a uint16 device tensor (through int32: torch has little uint16 arithmetic)."""
    import torch
    return (t8.to(torch.int32) * 257).to(torch.int16).view(torch.uint16)


def torch_to_u8(t16):
    import torch
    w = t16.view(torch.int16).to(torch.int32) & 0xFFFF
    return (((w + 128) * 255 + 255) >> 16).to(torch.uint8)


def test_torch_clip_on_the_current_stream(hb):
    """An (N, 3, H, W) uint8 clip already on the device, filtered in one call on torch's current stream."""
    import torch
    from halide_b200 import HalideBuffer, filters
    a = make_batch(4, 240, 320, 11)
    want = np.stack([composed(hb, a[k], 8, ALPHA, 1.0) for k in range(4)])
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    stream = torch.cuda.Stream()
    try:
        with torch.cuda.stream(stream):
            t_in = torch.from_numpy(a).cuda()
            t_out = torch.zeros_like(t_in)
            l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
            filters.local_laplacian_u8_batch(HalideBuffer.from_torch(t_in), 8, ALPHA, 1.0, HalideBuffer.from_torch(t_out))
            got = t_out.cpu().numpy()  # (ordered after the filter on the same stream)
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
    assert_frames(got, want)


def test_16k_frame(hb):
    """One 16384 x 16384 frame on the device against the uint16 filter composed with the conversions on the device."""
    import torch
    from halide_b200 import HalideBuffer, filters
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    try:
        l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        g = torch.Generator(device="cuda")
        g.manual_seed(16384)
        x8 = torch.randint(0, 256, (3, 16384, 16384), dtype=torch.uint8, device="cuda", generator=g)
        y8 = torch.zeros_like(x8)
        filters.local_laplacian_u8(HalideBuffer.from_torch(x8), 8, ALPHA, 1.0, HalideBuffer.from_torch(y8))
        x16 = torch_to_u16(x8)
        y16 = torch.zeros_like(x16)
        filters.local_laplacian(HalideBuffer.from_torch(x16), 8, ALPHA, 1.0, HalideBuffer.from_torch(y16))
        del x16
        want = torch.empty_like(y8)
        for c in range(3):
            want[c] = torch_to_u8(y16[c])
        torch.cuda.synchronize()
        n_bad = int((want != y8).sum())
        assert n_bad == 0, f"{n_bad} mismatching samples at 16K"
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
        torch.cuda.synchronize()


def test_consecutive_calls_mixing_u8_and_u16(hb):
    """The remap-table cache and the scratch are shared between the entry points: alternate u8 and u16 calls with
    different (levels, alpha)."""
    img = u8_frame((3, 120, 160), 9)
    img16 = convert(img, np.uint16)
    params = [(8, ALPHA), (5, 0.25), (8, 0.5), (8, ALPHA), (5, 0.25)]
    for levels, alpha in params:
        want16 = run_local_laplacian(hb, img16, levels, alpha, 1.0)
        got = run_u8(hb, img, levels, alpha, 1.0)
        assert_same(got, convert(want16, np.uint8), f"levels {levels} alpha {alpha}")
        assert_same(run_local_laplacian(hb, img16, levels, alpha, 1.0), want16, "uint16 after u8")
