"""GPU tests of the 8-bit float-pipeline entry points.  Their contract is the composition
    bilateral_grid_u8(in8, r_sigma)                      = to_u8(bilateral_grid(to_f32(in8), r_sigma))
    nl_means_u8(in8, patch_size, search_area, sigma)     = to_u8(nl_means(to_f32(in8), patch_size, search_area, sigma))
with the reference's element conversions (image_io.convert: to_f32(v) = v / 255.0f, to_u8(f) = lround(f * 255.0f)), so
every case compares byte for byte against that composition built from the float GPU filter.  Every float result the file
computes is also checked for the premise the 8-bit store relies on: finite, and f * 255.0f in [0, 255.5), where lround
gives 0..255 without a wrap.  The 8-bit inputs are numpy host buffers unless a test says otherwise."""
import ctypes

import numpy as np
import pytest

from halide_b200 import image_io
from halide_b200.image_io import convert
from util import kernels_run, nl_means_variant

pytestmark = pytest.mark.gpu
BG_KERNELS = {"bg_hist_blurz", "bg_blur_xy", "bg_slice"}
R_SIGMAS = [float(np.float32(1) / np.float32(199)), 0.01, 0.1, 0.37, 1.0, 5.0, float("inf")]


def u8_frame(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def assert_range(f, what=""):
    """The float path's output is what the 8-bit store converts: finite, and f * 255.0f in [0, 255.5)."""
    assert np.isfinite(f).all(), f"{what}: non-finite float output"
    y = f * np.float32(255.0)
    assert y.dtype == np.float32
    assert (y >= 0).all() and (y < np.float32(255.5)).all(), f"{what}: f * 255 in [{y.min()}, {y.max()}]"


def halfway(f):
    """Mask of the samples whose f * 255.0f (in float32) is exactly k + 0.5."""
    y = f * np.float32(255.0)
    return y == np.floor(y) + np.float32(0.5)


def assert_same(got, want, what=""):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def run(hb, fn, inp, args, out, in_mins=None, out_mins=None):
    """fn(input, *args, output) on numpy host buffers; returns out, read back."""
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    fn(bi, *args, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out


def float_path(hb, filt, in8, args, out_shape, in_mins=None, out_mins=None):
    """The float GPU filter on to_f32(in8), range-checked."""
    fn = hb.filters.bilateral_grid if filt == "bg" else hb.filters.nl_means
    f = run(hb, fn, convert(in8, np.float32), args, np.zeros(out_shape, np.float32), in_mins, out_mins)
    assert_range(f, f"{filt} {args} {out_shape}")
    return f


def u8_path(hb, filt, in8, args, out_shape, in_mins=None, out_mins=None):
    """The 8-bit entry point; returns (output, {kernel: (launches, ms)})."""
    fn = hb.filters.bilateral_grid_u8 if filt == "bg" else hb.filters.nl_means_u8
    with kernels_run(hb) as ran:
        got = run(hb, fn, in8, args, np.zeros(out_shape, np.uint8), in_mins, out_mins)
    return got, ran


def check(hb, filt, in8, args, out_shape=None, in_mins=None, out_mins=None):
    """8-bit entry point == to_u8(float path(to_f32(in8))); returns (u8 output, float output, kernels run)."""
    out_shape = in8.shape if out_shape is None else out_shape
    f = float_path(hb, filt, in8, args, out_shape, in_mins, out_mins)
    got, ran = u8_path(hb, filt, in8, args, out_shape, in_mins, out_mins)
    assert_same(got, convert(f, np.uint8), f"{filt} {args} in {in8.shape} {in_mins} out {out_shape} {out_mins}")
    return got, f, ran


def assert_bg_kernels(ran):
    assert BG_KERNELS <= set(ran) and "bg_hist_blurz_s" not in ran and "bg_slice_s" not in ran, sorted(ran)


def assert_nl_kernel(ran, window):
    assert set(ran) == {"nl_means_window" if window else "nl_means"}, sorted(ran)


# ---- bilateral_grid: equality with the float path ------------------------------------------------------------------

@pytest.mark.parametrize("h,w", [(1, 1), (37, 53), (333, 517)])
@pytest.mark.parametrize("r_sigma", R_SIGMAS)
def test_bg_sizes_and_r_sigma(hb, h, w, r_sigma):
    _, _, ran = check(hb, "bg", u8_frame((h, w), h * w + int(min(r_sigma, 9) * 100)), (r_sigma,))
    assert_bg_kernels(ran)


# (input shape, input mins (x, y), output shape, output mins, input column offset into a wider array)
BG_CROPS = [
    ((300, 400), (-13, -7), (250, 333), (-9, -5), 0),    # negative, unaligned mins; input larger than the output
    ((120, 257), (3, 5), (117, 251), (5, 6), 0),          # positive unaligned mins
    ((64, 131), (-64, -8), (64, 131), (-64, -8), 1),      # input pointer 1 byte off 4-byte alignment
    ((64, 131), (0, 0), (61, 127), (2, 3), 3),            # 3 bytes off
    ((17, 9), (-4, -4), (17, 9), (-4, -4), 2),            # narrower than a vector lane's 4 pixels x 2
]


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins,col", BG_CROPS)
@pytest.mark.parametrize("r_sigma", [0.1, R_SIGMAS[0]])
def test_bg_crops(hb, in_shape, in_mins, out_shape, out_mins, col, r_sigma):
    """Crops with negative and unaligned mins and unaligned row starts, so both the uchar4 and the scalar paths of
    bg_hist_blurz and bg_slice run."""
    h, w = in_shape
    base = u8_frame((h, w + col), h + w + col)
    img = base[:, col:]
    _, _, ran = check(hb, "bg", img, (r_sigma,), out_shape, in_mins, out_mins)
    assert_bg_kernels(ran)


def test_bg_8k(hb):
    """BASELINE config 3: 7680 x 4320, r_sigma 0.1."""
    img = u8_frame((4320, 7680), 3)
    _, f, ran = check(hb, "bg", img, (0.1,))
    assert_bg_kernels(ran)
    print(f"bilateral_grid 7680x4320: {int(halfway(f).sum())} half-way samples")


# ---- bilateral_grid against the oracle -----------------------------------------------------------------------------

@pytest.mark.parametrize("h,w,r_sigma,kw", [
    (64, 96, 0.1, {}),
    (200, 300, 0.25, {}),
    (211, 173, R_SIGMAS[0], {}),
    (150, 190, 0.1, dict(out_shape=(120, 160), in_mins=(-13, -7), out_mins=(-9, -5))),
])
def test_bg_against_the_oracle(hb, oracle, h, w, r_sigma, kw):
    """bg_hist_blurz's re-association gives the oracle's bits only where every partial bin sum is exact, which v / 255
    does not guarantee: where the library's float result equals the oracle's the bytes must be equal, and nowhere may
    they differ by more than 1."""
    img = u8_frame((h, w), h + w)
    out_shape = kw.get("out_shape", (h, w))
    got, f, _ = check(hb, "bg", img, (r_sigma,), out_shape, kw.get("in_mins"), kw.get("out_mins"))
    want_f = oracle.bilateral_grid(convert(img, np.float32), r_sigma, **kw)
    assert_range(want_f, "oracle")
    want = convert(want_f, np.uint8)
    same_f = f == want_f
    assert_same(got[same_f], want[same_f], "where the float results agree")
    assert np.abs(got.astype(np.int16) - want.astype(np.int16)).max() <= 1


def test_bg_halfway_rounding(hb):
    """Samples whose f * 255.0f is exactly k + 0.5 exist and go to k + 1 (halves away from zero, not to even)."""
    img = u8_frame((1000, 1500), 11)
    got, f, _ = check(hb, "bg", img, (0.1,))
    half = halfway(f)
    n = int(half.sum())
    print(f"bilateral_grid 1500x1000: {n} half-way samples")
    assert n > 0
    y = f[half] * np.float32(255.0)
    assert (got[half] == np.floor(y).astype(np.int64) + 1).all()


# ---- nl_means: equality with the float path ------------------------------------------------------------------------

NL_SIZES = [(3, 7, 0, True), (7, 7, 0, True), (5, 9, 0, False), (1, 1, 0, False), (3, 7, 1, False), (7, 7, 1, False)]


@pytest.mark.parametrize("patch,search,variant,window", NL_SIZES)
@pytest.mark.parametrize("h,w", [(1, 1), (37, 53), (150, 201)])
@pytest.mark.parametrize("sigma", [0.12, 1.0])
def test_nl_sizes(hb, patch, search, variant, window, h, w, sigma):
    """patch / search 3/7 and 7/7 take the register-window kernels, 5/9 and 1/1 the generic one, and the variant hook
    routes 3/7 and 7/7 to the generic kernel as well."""
    img = u8_frame((3, h, w), h * w + patch * 10 + search)
    with nl_means_variant(hb, variant):
        _, _, ran = check(hb, "nl", img, (patch, search, sigma))
    assert_nl_kernel(ran, window)


@pytest.mark.parametrize("channels", [1, 3, 4])
@pytest.mark.parametrize("patch,search,variant,window", [(3, 7, 0, True), (3, 7, 1, False), (5, 9, 0, False)])
def test_nl_channels(hb, channels, patch, search, variant, window):
    """A 1- or 4-channel input works as in the float path: channel accesses are clamped to the input's channels."""
    img = u8_frame((channels, 70, 90), channels)
    with nl_means_variant(hb, variant):
        _, _, ran = check(hb, "nl", img, (patch, search, 0.12), (3, 70, 90))
    assert_nl_kernel(ran, window)


@pytest.mark.parametrize("in_shape,in_mins,out_shape,out_mins", [
    ((3, 60, 80), (-7, -5, 0), (3, 50, 70), (-3, -2, 0)),      # negative mins, input larger
    ((3, 40, 50), (10, 20, 0), (3, 70, 90), (0, 0, 0)),        # input smaller than, and away from, the output: clamped
    ((2, 33, 47), (5, -9, 1), (3, 33, 47), (5, -9, 0)),        # channel min 1: channels 0, 1, 2 clamp to 1, 1, 2
])
@pytest.mark.parametrize("variant", [0, 1])
def test_nl_crops(hb, in_shape, in_mins, out_shape, out_mins, variant):
    img = u8_frame(in_shape, sum(in_shape))
    with nl_means_variant(hb, variant):
        _, _, ran = check(hb, "nl", img, (3, 7, 0.12), out_shape, in_mins, out_mins)
    assert_nl_kernel(ran, variant == 0)


def test_nl_4k(hb):
    """BASELINE config 4 on one GPU: 3840 x 2160 x 3, patch 3, search 7."""
    img = u8_frame((3, 2160, 3840), 4)
    _, f, ran = check(hb, "nl", img, (3, 7, 0.12))
    assert_nl_kernel(ran, True)
    print(f"nl_means 3840x2160 sigma 0.12: {int(halfway(f).sum())} half-way samples")


# ---- nl_means against the oracle (its float path is bit-exact) -----------------------------------------------------

@pytest.mark.parametrize("patch,search,sigma,in_shape,kw", [
    (3, 7, 0.12, (3, 123, 217), {}),
    (7, 7, 0.5, (3, 123, 217), {}),
    (5, 9, 1.0, (3, 123, 217), {}),
    (1, 1, 0.12, (3, 123, 217), {}),
    (3, 7, 1.0, (3, 60, 80), dict(out_shape=(3, 50, 70), in_mins=(-7, -5, 0), out_mins=(-3, -2, 0))),
    (7, 7, 0.3, (3, 40, 50), dict(out_shape=(3, 70, 90), in_mins=(10, 20, 0), out_mins=(0, 0, 0))),
])
@pytest.mark.parametrize("variant", [0, 1])
def test_nl_against_the_oracle(hb, oracle, patch, search, sigma, in_shape, kw, variant):
    img = u8_frame(in_shape, patch + search)
    out_shape = kw.get("out_shape", in_shape)
    with nl_means_variant(hb, variant):
        got, _, _ = check(hb, "nl", img, (patch, search, sigma), out_shape, kw.get("in_mins"), kw.get("out_mins"))
    want_f = oracle.nl_means(convert(img, np.float32), patch, search, sigma, **kw)
    assert_range(want_f, "oracle")
    assert_same(got, convert(want_f, np.uint8), "oracle")


def test_nl_halfway_rounding(hb):
    """At sigma 1 the weights spread over the search window and some samples land exactly on k + 0.5 (at sigma 0.12 on
    noise the centre weight dominates and the output stays on the input's codes)."""
    img = u8_frame((3, 1000, 1000), 1)
    got, f, _ = check(hb, "nl", img, (3, 7, 1.0))
    half = halfway(f)
    n = int(half.sum())
    print(f"nl_means 1000x1000 sigma 1: {n} half-way samples")
    assert n > 0
    y = f[half] * np.float32(255.0)
    assert (got[half] == np.floor(y).astype(np.int64) + 1).all()


# ---- the reference harnesses' sequence -----------------------------------------------------------------------------

def test_harness_equivalence(hb, tmp_path):
    """apps/bilateral_grid/filter.cpp and apps/nl_means/process.cpp on a random 8-bit PNG: load_and_convert_image to
    float, the float filter, convert_and_save_image.  Given a float image, convert_and_save_image writes a PNG at 16 bits
    (the closest depth PNG holds); the 8-bit file is the same sequence with the float output converted to uint8
    (image_io.convert) before the save.  That file, read back, equals the 8-bit entry point's output on the input file
    loaded as uint8."""
    gray, rgb = str(tmp_path / "gray.png"), str(tmp_path / "rgb.png")
    image_io.save(u8_frame((240, 320), 21), gray)
    image_io.save(u8_frame((3, 180, 250), 22), rgb)
    for filt, path, args in (("bg", gray, (0.1,)), ("nl", rgb, (7, 7, 0.12))):
        fin = image_io.load_and_convert_image(path, np.float32)
        assert fin.dtype == np.float32
        fn = hb.filters.bilateral_grid if filt == "bg" else hb.filters.nl_means
        fout = run(hb, fn, fin, args, np.zeros(fin.shape, np.float32))
        assert_range(fout, filt)
        saved16, saved8 = str(tmp_path / f"{filt}_out16.png"), str(tmp_path / f"{filt}_out8.png")
        image_io.convert_and_save_image(fout, saved16)
        assert image_io.load(saved16).dtype == np.uint16
        image_io.convert_and_save_image(convert(fout, np.uint8), saved8)
        want = image_io.load(saved8)
        in8 = image_io.load(path)
        assert in8.dtype == np.uint8
        got, _ = u8_path(hb, filt, in8, args, in8.shape)
        assert want.dtype == np.uint8 and want.shape == got.shape
        assert_same(got, want, f"{filt} harness")


# ---- residency and layouts -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("filt", ["bg", "nl"])
def test_host_padded_rows_leave_the_padding_alone(hb, filt):
    """Row pitches wider than the frame on both buffers; the bytes around the output region keep their sentinel."""
    h, w, pad = 97, 131, 13
    shape = (h, w) if filt == "bg" else (3, h, w)
    args = (0.1,) if filt == "bg" else (3, 7, 0.12)
    img_base = u8_frame(shape[:-1] + (w + pad,), 31)
    img = img_base[..., :w]
    want = convert(float_path(hb, filt, np.ascontiguousarray(img), args, shape), np.uint8)
    out_base = np.full(shape[:-1] + (w + pad,), 0xAB, np.uint8)
    out = out_base[..., 2:w + 2]
    fn = hb.filters.bilateral_grid_u8 if filt == "bg" else hb.filters.nl_means_u8
    run(hb, fn, img, args, out)
    assert_same(np.ascontiguousarray(out), want, f"{filt} padded")
    assert (out_base[..., :2] == 0xAB).all() and (out_base[..., w + 2:] == 0xAB).all(), "wrote into the row padding"


@pytest.mark.parametrize("filt", ["bg", "nl"])
def test_device_resident_torch_tensors(hb, filt):
    """(H, W) / (3, H, W) uint8 torch tensors on the device (HalideBuffer.from_torch): a dense frame, then crops of
    padded tensors whose padding keeps its sentinel."""
    import torch
    from halide_b200 import HalideBuffer
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    try:
        h, w, pad = 211, 301, 19
        shape = (h, w) if filt == "bg" else (3, h, w)
        args = (0.1,) if filt == "bg" else (7, 7, 0.12)
        fn = hb.filters.bilateral_grid_u8 if filt == "bg" else hb.filters.nl_means_u8
        img = u8_frame(shape, 41)
        want = convert(float_path(hb, filt, img, args, shape), np.uint8)
        x8 = torch.from_numpy(img).cuda()
        y8 = torch.zeros_like(x8)
        fn(HalideBuffer.from_torch(x8), *args, HalideBuffer.from_torch(y8))
        assert_same(y8.cpu().numpy(), want, f"{filt} dense device tensors")
        xb = torch.zeros(shape[:-1] + (w + pad,), dtype=torch.uint8, device="cuda")
        xb[..., 5:w + 5] = x8
        yb = torch.full(shape[:-1] + (w + pad,), 0xAB, dtype=torch.uint8, device="cuda")
        fn(HalideBuffer.from_torch(xb[..., 5:w + 5]), *args, HalideBuffer.from_torch(yb[..., 3:w + 3]))
        out = yb.cpu().numpy()
        assert_same(out[..., 3:w + 3], want, f"{filt} padded device tensors")
        assert (out[..., :3] == 0xAB).all() and (out[..., w + 3:] == 0xAB).all(), "wrote into the row padding"
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
        torch.cuda.synchronize()
