"""GPU tests of the interleaved local_laplacian entry points (uint16 / uint8, one frame / batch).  Their contract: the
result equals, bit for bit, what the matching planar entry point gives on planar copies of the same buffers.  So every
case runs the planar entry point on a planar copy and compares; the small uint16 frames are also compared against the
oracle.  Frames are numpy arrays indexed [(n,) y, x, pitch] (host buffers, copied by the runtime) unless a test says
otherwise; an output whose pitch exceeds its channels is pre-filled with a pattern that must survive."""
import ctypes
from contextlib import contextmanager

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ALPHA = 1.0 / 7.0
GUARD = 0xA5  # pre-filled output samples the filter must not touch (0xA5A5 for uint16)


# ---- fixtures -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hb():
    """The product binding (raises, does not skip, if libhalide_b200.so is missing)."""
    import halide_b200
    halide_b200.load_library()
    return halide_b200


@pytest.fixture(scope="module")
def oracle():
    """The CPU oracle, built on demand by oracle/Makefile, on at most 16 threads (its small OpenMP regions crawl on very
    wide hosts)."""
    from oracle import pyoracle
    pyoracle.lib()
    pyoracle.set_threads(min(16, pyoracle.use_all_cores()))
    return pyoracle


def frame(shape, dtype, seed, smooth=False):
    """Random or smooth (low-frequency + mild noise) content of the given numpy shape, last axis = samples of a pixel."""
    rng = np.random.default_rng(seed)
    top = np.iinfo(dtype).max
    if not smooth:
        return rng.integers(0, top + 1, shape, dtype=dtype)
    h, w = shape[-3], shape[-2]
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = np.empty(shape, dtype)
    for ch in range(shape[-1]):
        base = 0.5 + 0.45 * np.sin(xx / (7.0 + ch) + seed) * np.cos(yy / (11.0 - ch)) + rng.normal(0, 0.02, (h, w))
        out[..., ch] = np.clip(base * top, 0, top).astype(dtype)
    return out


def hwc_buffer(hb, arr, mins=None, host_dirty=True):
    """(x, y, c[, n]) interleaved buffer over a numpy [(n,) y, x, c] array (any view)."""
    perm = (2, 0, 1) if arr.ndim == 3 else (0, 3, 1, 2)
    return hb.HalideBuffer.from_numpy(arr.transpose(perm), mins, host_dirty=host_dirty)


def planar_copy(arr):
    perm = (2, 0, 1) if arr.ndim == 3 else (0, 3, 1, 2)
    return np.ascontiguousarray(arr.transpose(perm))


def entry(hb, dtype, batch, interleaved):
    f = hb.filters
    u8 = np.dtype(dtype) == np.uint8
    if interleaved:
        return {(False, False): f.local_laplacian_interleaved, (False, True): f.local_laplacian_interleaved_batch,
                (True, False): f.local_laplacian_u8_interleaved, (True, True): f.local_laplacian_u8_interleaved_batch}[u8, batch]
    return {(False, False): f.local_laplacian, (False, True): f.local_laplacian_batch,
            (True, False): f.local_laplacian_u8, (True, True): f.local_laplacian_u8_batch}[u8, batch]


def run_interleaved(hb, inp, out, levels, alpha, beta, in_mins=None, out_mins=None):
    """The interleaved filter on numpy views inp / out ([(n,) y, x, c]); returns nothing (out is written)."""
    bi, bo = hwc_buffer(hb, inp, in_mins), hwc_buffer(hb, out, out_mins, host_dirty=False)
    entry(hb, inp.dtype, inp.ndim == 4, True)(bi, levels, alpha, beta, bo)
    assert bo.device_dirty
    bo.copy_to_host()


def run_planar(hb, inp, out_shape, levels, alpha, beta, in_mins=None, out_mins=None):
    """The planar entry point on a planar copy of inp; returns the output as an [(n,) y, x, c] array."""
    pin = planar_copy(inp)
    pout = np.zeros(out_shape[:-3] + (out_shape[-1],) + out_shape[-3:-1], inp.dtype)
    bi = hb.HalideBuffer.from_numpy(pin, in_mins)
    bo = hb.HalideBuffer.from_numpy(pout, out_mins, host_dirty=False)
    entry(hb, inp.dtype, inp.ndim == 4, False)(bi, levels, alpha, beta, bo)
    bo.copy_to_host()
    return np.moveaxis(pout, -3, -1)


def assert_same(got, want, what=""):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def check(hb, inp, levels=8, alpha=ALPHA, beta=1.0, out_c=3, out_pitch=None, in_mins=None, out_mins=None, out_hw=None):
    """Interleaved call into an output of `out_c` channels in a pitch of `out_pitch` samples (guard-filled), against the
    planar entry point on a planar copy; the samples past out_c must keep the guard.  Returns the output's channels."""
    out_pitch = out_c if out_pitch is None else out_pitch
    hw = inp.shape[-3:-1] if out_hw is None else out_hw
    full = np.full(inp.shape[:-3] + tuple(hw) + (out_pitch,), GUARD * (257 if inp.dtype == np.uint16 else 1), inp.dtype)
    out = full[..., :out_c]
    run_interleaved(hb, inp, out, levels, alpha, beta, in_mins, out_mins)
    want = run_planar(hb, inp, out.shape, levels, alpha, beta, in_mins, out_mins)
    assert_same(out, want, f"levels {levels} beta {beta} pitch {inp.shape[-1]}->{out_pitch}")
    assert (full[..., out_c:] == full.dtype.type(GUARD * (257 if inp.dtype == np.uint16 else 1))).all(), "uncovered samples changed"
    return out


@contextmanager
def force_generic(hb, mask):
    l = hb.load_library()
    l.halide_b200_ll_force_generic(mask)
    try:
        yield
    finally:
        l.halide_b200_ll_force_generic(0)


@contextmanager
def on_torch_stream(hb, stream):
    import torch
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    try:
        with torch.cuda.stream(stream):
            l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
            yield
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))


DTYPES = [np.uint16, np.uint8]


# ---- pitches, channels, parameters ----------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("in_pitch,out_c,out_pitch", [(3, 3, 3), (4, 4, 4), (4, 3, 3), (4, 3, 4), (3, 3, 4)])
@pytest.mark.parametrize("levels,beta", [(8, 1.0), (8, 0.5), (5, 1.0), (2, 0.5)])
def test_pitches_and_channels(hb, dtype, in_pitch, out_c, out_pitch, levels, beta):
    """RGB and RGBA frames; RGBA in -> RGB out; RGBA in -> channels [0, 3) of an RGBA out (alpha untouched)."""
    img = frame((133, 217, in_pitch), dtype, in_pitch * 10 + levels, smooth=levels == 5)
    check(hb, img, levels, 1.0 / (levels - 1), beta, out_c=out_c, out_pitch=out_pitch)


@pytest.mark.parametrize("levels,beta", [(8, 1.0), (8, 0.5), (5, 1.0), (2, 1.0)])
@pytest.mark.parametrize("pitch", [3, 4])
def test_against_the_oracle(hb, oracle, levels, beta, pitch):
    img = frame((91, 67, pitch), np.uint16, 7 + levels + pitch)
    got = check(hb, img, levels, 1.0 / (levels - 1), beta)
    want = oracle.local_laplacian(planar_copy(img)[:3], levels, 1.0 / (levels - 1), beta)
    assert_same(planar_copy(got), want, f"oracle levels {levels} beta {beta} pitch {pitch}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("alpha,beta", [(1.0, 1.0), (1.0, 0.25), (0.0, 2.0)])
def test_saturating_content(hb, dtype, alpha, beta):
    """Strong detail boost on noise (outputs clamp at both ends), and constant black / white frames."""
    top = np.iinfo(dtype).max
    img = frame((96, 130, 3), dtype, 3)
    img[:, ::2, 0] = top
    img[::3, :, 1] = 0
    out = check(hb, img, 8, alpha, beta)
    assert (out == 0).any() and (out == top).any()
    for v in (0, top):
        check(hb, np.full((40, 70, 4), v, dtype), 8, alpha, beta, out_c=3, out_pitch=4)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("in_pitch,out_pitch", [(3, 3), (4, 3), (4, 4)])
@pytest.mark.parametrize("beta", [1.0, 0.5])
@pytest.mark.parametrize("batch", [False, True])
def test_tma_frame_tile_path(hb, dtype, in_pitch, out_pitch, beta, batch):
    """Even widths and mins, whole RGB / RGBA pixels: the final kernel's TMA frame tile with fixed pitches and pixel-pair
    stores (alpha of an RGBA output untouched), including a tile grid that does not divide the frame and an output crop
    whose first column lies 16 bytes into the input (still the TMA path) or at another even offset (the general path)."""
    shape = ((3,) if batch else ()) + (70, 322, in_pitch)
    img = frame(shape, dtype, in_pitch * 7 + out_pitch + int(batch), smooth=beta != 1.0)
    check(hb, img, 8, ALPHA, beta, out_c=3, out_pitch=out_pitch)
    n = (0,) if batch else ()
    for off in (16 // np.dtype(dtype).itemsize, 2):
        check(hb, img, 8, ALPHA, beta, out_c=3, out_pitch=out_pitch, in_mins=(0, 0, 0) + n, out_mins=(off, 3, 0) + n,
              out_hw=(61, 240))


# ---- layouts and bounds ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("levels", [8, 5])
def test_padded_rows_mins_odd_widths_and_crops(hb, dtype, levels):
    """A padded row stride, nonzero mins, odd widths and crops that start on odd columns (the non-TMA paths), and an
    input larger than the output (repeat_edge clamps at the input's own edges)."""
    big = frame((150, 260, 4), dtype, 21)
    # padded rows: a (100, 201) RGB view inside wider rows
    inp = big[10:110, 7:208, :3]
    check(hb, inp, levels, 1.0 / (levels - 1), 1.0, in_mins=(-5, 3, 0), out_mins=(-5, 3, 0))
    # output = a crop of the input region at odd offsets, odd width, RGBA pitch on both sides
    inp = big[5:140, 3:250]
    check(hb, inp, levels, 1.0 / (levels - 1), 0.5, out_c=3, out_pitch=4, in_mins=(-2, -1, 0), out_mins=(1, 4, 0),
          out_hw=(97, 131))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mask", [1, 2, 4, 8, 16, 64, 1 | 2 | 4 | 8, 127])
def test_force_generic_masks(hb, dtype, mask):
    img = frame((120, 250, 4), dtype, mask)
    with force_generic(hb, mask):
        check(hb, img, 8, ALPHA, 1.0, out_c=3, out_pitch=4)
        check(hb, img[:, 1:, :3], 8, ALPHA, 0.5)


@pytest.mark.parametrize("dtype", DTYPES)
def test_host_buffers_copy_exactly(hb, dtype):
    """Host (H, W, 3) and (H, W, 4) numpy arrays: the runtime's H2D copy of the interleaved input and D2H copy of the
    output are element-exact, and the D2H copy leaves the alpha samples of an RGBA output alone."""
    img = frame((257, 383, 4), dtype, 99)
    out = check(hb, img, 8, ALPHA, 1.0, out_c=3, out_pitch=4)
    check(hb, np.ascontiguousarray(img[..., :3]), 8, ALPHA, 1.0)
    assert out.shape == (257, 383, 3)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batches(hb, dtype):
    clip = frame((3, 90, 161, 4), dtype, 5)
    check(hb, clip, 8, ALPHA, 1.0, out_c=3, out_pitch=4)
    check(hb, np.ascontiguousarray(clip[..., :3]), 5, 0.25, 0.5)
    # frames shifted: output frames 0..1 read input frames 0..1 of an input whose frames start at -1
    check(hb, clip[..., :3], 8, ALPHA, 1.0, in_mins=(0, 0, 0, -1), out_mins=(0, 0, 0, -1))


# ---- torch device tensors -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", ["uint16", "uint8"])
def test_torch_channels_last_batch_on_a_side_stream(hb, dtype):
    """An (N, 3, H, W) channels_last clip on the device, filtered on a non-default current stream, against the planar
    batch entry point on the contiguous copy."""
    import torch
    from halide_b200 import HalideBuffer
    np_clip = frame((4, 3, 181, 243), np.dtype(dtype), 17)
    stream = torch.cuda.Stream()
    with on_torch_stream(hb, stream):
        # (built by copies only: torch's uint16 CUDA support covers copies, not fills)
        x = torch.from_numpy(np_clip).cuda().contiguous(memory_format=torch.channels_last)
        y = torch.from_numpy(np.zeros_like(np_clip)).cuda().contiguous(memory_format=torch.channels_last)
        assert x.stride()[1] == 1 and y.stride()[1] == 1
        bi, bo = HalideBuffer.from_torch(x), HalideBuffer.from_torch(y)
        assert bi.shape()[2] == (0, 3, 1) and bi.shape()[0][2] == 3
        entry(hb, np.dtype(dtype), True, True)(bi, 8, ALPHA, 1.0, bo)
        xp = x.contiguous()
        yp = torch.from_numpy(np.zeros_like(np_clip)).cuda()
        entry(hb, np.dtype(dtype), True, False)(HalideBuffer.from_torch(xp), 8, ALPHA, 1.0, HalideBuffer.from_torch(yp))
        got, want = y.contiguous().cpu().numpy(), yp.cpu().numpy()  # (ordered after both filters on the same stream)
    assert_same(got, want, "channels_last clip")


def test_16k_u8_rgb_frame(hb):
    """One 16384 x 16384 uint8 RGB frame on the device, against the planar 8-bit entry point."""
    import torch
    from halide_b200 import HalideBuffer
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    try:
        l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        g = torch.Generator(device="cuda")
        g.manual_seed(1616)
        x = torch.randint(0, 256, (16384, 16384, 3), dtype=torch.uint8, device="cuda", generator=g)
        y = torch.zeros_like(x)
        hb.filters.local_laplacian_u8_interleaved(HalideBuffer.from_torch(x.permute(2, 0, 1)), 8, ALPHA, 1.0,
                                                  HalideBuffer.from_torch(y.permute(2, 0, 1)))
        xp = x.permute(2, 0, 1).contiguous()
        del x
        yp = torch.zeros_like(xp)
        hb.filters.local_laplacian_u8(HalideBuffer.from_torch(xp), 8, ALPHA, 1.0, HalideBuffer.from_torch(yp))
        n_bad = int((y.permute(2, 0, 1) != yp).sum())
        assert n_bad == 0, f"{n_bad} mismatching samples at 16K"
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
        torch.cuda.synchronize()
