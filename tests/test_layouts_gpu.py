"""Every filter on buffers whose strides are negative, zero or ordered other than planar, against the oracle.

The Halide C ABI lets a caller describe memory with any stride but dim[0].stride == 1, and the filters accept such
buffers: bottom-up images (a negative row stride), an RGB <-> BGR view (a negative channel stride), broadcast inputs
(stride 0, as np.broadcast_to and torch.expand make them), line-interleaved planes (channel stride smaller than row
stride) and reversed clips.  Several host conditions pick a kernel path from the sign or alignment of a stride, so the
same frame is run in each layout:

- integer pipelines bit for bit against the oracle on dense copies of the logical arrays;
- float pipelines within 1e-4 of the oracle, and bit for bit against the same entry point on dense copies (no kernel's
  arithmetic depends on the layout);
- every output is a view into a larger canvas filled with a sentinel: the bytes outside the view must keep it.

Buffers are built twice: numpy views over host memory (copied to the device by the runtime, which keeps their strides),
and the same memory as a torch CUDA tensor described by hand and wrapped with halide_cuda_wrap_device_ptr (torch cannot
express a negative stride itself).  Also here: the row-sharded local_laplacian on bands in these layouts, and uploads of
broadcast buffers."""
import ctypes

import numpy as np
import pytest

import conv_any_exact as cx
from halide_b200.image_io import convert
from test_dist_loopback_gpu import _RANK_THREADS, _settings, _single, FRAMES
from util import CP_M3200, CP_M7000, cp_params, f32_frame, kernels_run, nl_means_variant, smooth_u16_frame, u16_frame

pytestmark = pytest.mark.gpu
RTOL = 1e-4  # the float pipelines' tolerance, as in test_bilateral_grid_gpu.py / test_nl_means_gpu.py
SENTINEL = 0xA5  # every byte of an output canvas before the call
H, W = 37, 53  # ragged
WIDE = (40, 256)  # dense: the aligned / TMA / vector paths; padded to an even pitch (258): only the 4-byte ones
VARIANTS = ["host", "device"]


# ---- layouts ---------------------------------------------------------------------------------------------------------
# A layout maps a logical array (numpy shape, outermost first: [n,] [c,] y, x) to memory.  Named ones act on the planar
# axes; conv_layer's (n, y, x, ci) arrays give ("flip", axis) / ("bcast", axis) directly.
NAMED = {"dense": ("dense", None), "pad": ("pad", None), "flip_y": ("flip", -2), "flip_y_odd": ("flip_odd", -2),
         "flip_c": ("flip", -3), "flip_n": ("flip", -4), "xcy": ("xcy", None),
         "bcast_y": ("bcast", -2), "bcast_c": ("bcast", -3), "bcast_n": ("bcast", -4),
         "flip_y16": ("flip16", -2), "flip_c16": ("flip16", -3)}


def pitch(w, kind):
    """Row pitch: dense; a multiple of 16 samples for a kind ending in "16" (every row 16-byte aligned, as the vector
    and TMA paths need); odd for "flip_odd"; else padded to an even pitch, whose rows are 4-byte aligned for 16-bit
    samples (the pair / word paths) but not 16-byte aligned."""
    if kind == "dense":
        return w
    if kind.endswith("16"):
        return -(-w // 16) * 16
    return w + 1 + (w & 1) if kind == "flip_odd" else w + 2 + (w & 1)


def layout(shape, lay):
    """(memory shape, view(mem) -> (writable view, view of the logical shape)) for `lay` (a name or a (kind, axis)
    pair, or a function of the shape giving that pair for a layout of the caller's own).  A broadcast view is written
    through its writable view of extent 1 on the broadcast axis."""
    if callable(lay):
        return lay(tuple(shape))
    kind, axis = NAMED[lay] if isinstance(lay, str) else lay
    shape = tuple(shape)
    p = pitch(shape[-1], kind)
    kind = kind.removesuffix("16")
    if kind == "xcy":  # memory [..., y, c, x]: channel stride = pitch, row stride = C * pitch
        mshape = shape[:-3] + (shape[-2], shape[-3], p)
        return mshape, lambda m: (lambda v: (v, v))(m[..., :shape[-1]].swapaxes(-2, -3))
    if kind == "bcast":
        mshape = list(shape[:-1]) + [p]
        mshape[axis] = 1
        return tuple(mshape), lambda m: (m[..., :shape[-1]], np.broadcast_to(m[..., :shape[-1]], shape))
    mshape = shape[:-1] + (p,)
    if kind in ("flip", "flip_odd"):
        return mshape, lambda m: (lambda v: (v, v))(np.flip(m[..., :shape[-1]], axis))
    return mshape, lambda m: (m[..., :shape[-1]], m[..., :shape[-1]])


def _torch_dtype(dtype):
    return np.int16 if dtype == np.uint16 else dtype  # (torch.from_numpy: uint16 memory moves as int16)


class Buf:
    """A buffer of logical shape `shape` in layout `lay` over memory filled with the sentinel and then, for an input, with
    `data`: on the host or, wrapped, on the device."""

    def __init__(self, hb, shape, dtype, lay, variant, mins=None, data=None):
        self.hb, self.shape, self.dtype, self.lay, self.variant = hb, tuple(shape), np.dtype(dtype), lay, variant
        self.mshape, self.view_of = layout(shape, lay)
        self.mem = np.empty(self.mshape, dtype)
        self.mem.view(np.uint8)[...] = SENTINEL
        wv, v = self.view_of(self.mem)
        if data is not None:  # (a broadcast layout keeps index 0 of the broadcast axis)
            wv[...] = data[tuple(slice(0, n) for n in wv.shape)]
        self.logical = np.ascontiguousarray(v)
        if variant == "host":
            self.buf = hb.HalideBuffer.from_numpy(v, mins, host_dirty=data is not None)
        else:
            import torch
            self.t = torch.from_numpy(self.mem.view(_torch_dtype(self.dtype))).cuda()
            off = v.ctypes.data - self.mem.ctypes.data  # (bytes from the memory's start to the element at the mins)
            strides = [s // v.itemsize for s in reversed(v.strides)]
            self.buf = hb.HalideBuffer(dtype, tuple(reversed(v.shape)), strides, mins)
            hb.lib.check(hb.capi.halide_cuda_wrap_device_ptr(None, self.buf.ptr, ctypes.c_uint64(self.t.data_ptr() + off)))
            self.buf._keep, self.buf._wrapped = self.t, True

    @property
    def ptr(self):
        return self.buf.ptr

    def strides(self):
        return [self.buf.dims[d].stride for d in range(self.buf.buf.dimensions)]

    def read(self):
        """The whole canvas after a call, and the logical view's values: asserts that nothing outside the view changed."""
        if self.variant == "host":
            assert self.buf.device_dirty
            self.buf.copy_to_host()
            mem = self.mem
        else:
            import torch
            torch.cuda.synchronize()
            mem = self.t.cpu().numpy().view(self.dtype)
        inside = np.zeros(self.mshape, bool)
        self.view_of(inside)[0][...] = True
        outside = mem.view(np.uint8).reshape(self.mshape + (-1,))[~inside]
        bad = np.count_nonzero(outside != SENTINEL)
        assert bad == 0, f"{self.lay} ({self.variant}): {bad} bytes outside the output's view were written"
        return np.ascontiguousarray(self.view_of(mem)[1])


def out_buf(hb, shape, dtype, lay, variant, mins=None):
    return Buf(hb, shape, dtype, lay, variant, mins)


def same(got, want, what=""):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} of {got.size} samples differ, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def close(got, want, floor, what=""):
    assert np.isfinite(got).all(), what
    err = np.abs(got - want) / np.maximum(np.abs(want), floor)
    assert err.max() <= RTOL, f"{what}: max rel err {err.max()} at {np.unravel_index(err.argmax(), err.shape)}"


def dense_call(hb, call, ins, out_shape, out_dtype, in_mins=None, out_mins=None):
    """`call` on dense host copies of the logical inputs."""
    in_mins = in_mins or [None] * len(ins)
    bi = [hb.HalideBuffer.from_numpy(np.ascontiguousarray(a), m) for a, m in zip(ins, in_mins)]
    out = np.zeros(out_shape, out_dtype)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    call(*bi, bo)
    bo.copy_to_host()
    return out


def layout_call(hb, call, datas, in_lays, out_shape, out_dtype, out_lay, variant, in_mins=None, out_mins=None):
    """`call` on the inputs `datas` in layouts `in_lays` and an output in `out_lay`: (logical inputs, output, the kernels
    that ran, the buffers)."""
    in_mins = in_mins or [None] * len(datas)
    bi = [Buf(hb, d.shape, d.dtype, l, variant, m, d) for d, l, m in zip(datas, in_lays, in_mins)]
    bo = out_buf(hb, out_shape, out_dtype, out_lay, variant, out_mins)
    with kernels_run(hb) as ran:
        call(*bi, bo)
        got = bo.read()
    return [b.logical for b in bi], got, ran, bi + [bo]


def pairs(in_lays, out_lays, extra=()):
    """Each input layout with a dense output, each output layout with a dense input, and `extra` pairs."""
    return ([(l, "dense") for l in in_lays] + [("dense", l) for l in out_lays if l != "dense"] + list(extra))


# ---- blur -----------------------------------------------------------------------------------------------------------

def blur_pair_ok(bi, bo):
    """blur.cu: pixel pairs 4-byte aligned on every row of both buffers -> the pair kernel (input and output at the same
    mins, so the input's first read is its element at the mins)."""
    (isy, osy) = bi.strides()[1], bo.strides()[1]
    return ((bi.buf.buf.device | bo.buf.buf.device) & 3) == 0 and isy % 2 == 0 and osy % 2 == 0


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("general", [0, 1])
@pytest.mark.parametrize("size", [(H, W), WIDE], ids=["ragged", "wide"])
@pytest.mark.parametrize("in_lay,out_lay", pairs(["dense", "pad", "flip_y", "flip_y_odd", "bcast_y"], ["flip_y", "flip_y_odd"],
                                                 [("flip_y", "flip_y_odd"), ("flip_y_odd", "flip_y")]))
def test_blur(hb, oracle, in_lay, out_lay, size, general, variant):
    h, w = size
    img = u16_frame((h + 2, w + 2), h * w + len(in_lay))
    l = hb.load_library()
    l.halide_b200_blur_force_general(general)
    try:
        (logical,), got, ran, (bi, bo) = layout_call(hb, hb.filters.halide_blur, [img], [in_lay], (h, w), np.uint16, out_lay,
                                                     variant)
    finally:
        l.halide_b200_blur_force_general(0)
    same(got, oracle.blur(logical), f"{in_lay} -> {out_lay}")
    pair = blur_pair_ok(bi, bo) and not general
    assert list(ran) == ["blur3x3_u16_quad" if pair else "blur3x3_u16"], sorted(ran)
    if (in_lay, out_lay, variant, size) == ("dense", "dense", "host", WIDE) and not general:
        assert pair  # (the layouts alone move this frame off the pair kernel)


# ---- local_laplacian --------------------------------------------------------------------------------------------------
LEVELS, ALPHA = 8, 1.0 / 7.0
LL_IN = ["dense", "flip_y", "flip_y_odd", "flip_c", "xcy", "bcast_y", "bcast_c"]
LL_OUT = ["flip_y", "flip_y_odd", "flip_c", "xcy"]
LL_PAIRS = pairs(LL_IN, LL_OUT, [("flip_y", "xcy"), ("xcy", "flip_c"), ("flip_c", "flip_y")])


def ll_call(levels=LEVELS, alpha=ALPHA, beta=1.0, fn=None):
    return lambda bi, bo: (fn or _ll)(bi, levels, alpha, beta, bo)


def _ll(*a):
    import halide_b200
    return halide_b200.filters.local_laplacian(*a)


def ll_final_fast_path(bi, bo, wb=4):
    """local_laplacian.cu launch_final, planar: the aligned path (and from it the TMA one) needs positive row and channel
    strides and wb-byte aligned bases, strides and widths.  Restated for a 3-channel frame at mins 0."""
    isy, isc = bi.strides()[1:3]
    osy, osc = bo.strides()[1:3]
    w = bo.buf.dims[0].extent
    return (all(s > 0 for s in (isy, isc, osy, osc)) and all((2 * s) % wb == 0 for s in (isy, isc, osy, osc, w)) and
            bi.buf.buf.device % wb == 0 and bo.buf.buf.device % wb == 0)


@pytest.fixture(scope="module")
def ll_frames():
    return {(H, W): smooth_u16_frame((3, H, W), 5), WIDE: smooth_u16_frame((3,) + WIDE, 6)}


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mask", [0, 16, 64, 1 | 2 | 4])
@pytest.mark.parametrize("in_lay,out_lay", LL_PAIRS)
def test_local_laplacian(hb, oracle, ll_frames, in_lay, out_lay, mask, variant):
    """halide_b200_ll_force_generic: 16 = the final kernel's general-layout path, 64 = no TMA, 1|2|4 = the generic
    down-sweep, up-sweep and final kernels."""
    l = hb.load_library()
    for size in ll_frames:
        l.halide_b200_ll_force_generic(mask)
        try:
            (logical,), got, ran, (bi, bo) = layout_call(hb, ll_call(), [ll_frames[size]], [in_lay], (3,) + size, np.uint16,
                                                         out_lay, variant)
        finally:
            l.halide_b200_ll_force_generic(0)
        same(got, oracle.local_laplacian(logical, LEVELS, ALPHA, 1.0), f"{size} {in_lay} -> {out_lay}")
        if mask == 0:
            assert "ll_final2" in ran and "ll_level1" in ran, sorted(ran)
            if size == WIDE and variant == "host":
                assert ll_final_fast_path(bi, bo) == (in_lay in ("dense", "xcy") and out_lay in ("dense", "xcy"))


def batch_data(n, shape, dtype, seed):
    if dtype == np.uint8:
        return np.stack([(u16_frame(shape, 100 * seed + k) >> 8).astype(np.uint8) for k in range(n)])
    return np.stack([u16_frame(shape, 100 * seed + k) for k in range(n)])


LL_BATCH_PAIRS = pairs(["flip_y", "flip_c", "xcy", "bcast_c", "bcast_n", "flip_n"], ["flip_y", "flip_c", "xcy", "flip_n"],
                       [("flip_n", "flip_n"), ("bcast_n", "flip_y")])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("entry", ["batch", "u8", "u8_batch"])
@pytest.mark.parametrize("in_lay,out_lay", LL_BATCH_PAIRS)
def test_local_laplacian_batch_and_u8(hb, oracle, in_lay, out_lay, entry, variant):
    """The 4-D and 8-bit entry points: frame k against the oracle on frame k (8-bit: through the reference's u8 <-> u16
    conversions)."""
    batch, u8 = entry.endswith("batch"), entry.startswith("u8")
    if not batch and ("_n" in in_lay or "_n" in out_lay):
        pytest.skip("no frame dimension")
    dtype = np.uint8 if u8 else np.uint16
    fn = {"batch": hb.filters.local_laplacian_batch, "u8": hb.filters.local_laplacian_u8,
          "u8_batch": hb.filters.local_laplacian_u8_batch}[entry]
    shape = ((3,) if batch else ()) + (3, H, W)
    data = batch_data(shape[0], shape[1:], dtype, 7) if batch else batch_data(1, shape, dtype, 7)[0]
    (logical,), got, _, _ = layout_call(hb, ll_call(fn=fn), [data], [in_lay], shape, dtype, out_lay, variant)
    frames = logical if batch else logical[None]
    for k, f in enumerate(frames):
        want = oracle.local_laplacian(convert(f, np.uint16) if u8 else f, LEVELS, ALPHA, 1.0)
        same((got if batch else got[None])[k], convert(want, np.uint8) if u8 else want, f"frame {k}")


A16 = ("flip_y16", "flip_c16")  # flipped rows or channels whose every row starts on 16 bytes


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("J,levels", [(1, 8), (1, 5), (2, 8), (2, 5), (8, 8), (8, 5)])
@pytest.mark.parametrize("in_lay,out_lay", pairs(["dense", "flip_y", "flip_c", "xcy", "bcast_c"], ["flip_y", "flip_c", "xcy"],
                                                 [(l, m) for l in A16 for m in A16] + [("flip_y16", "flip_y")]))
def test_local_laplacian_pyramid_levels(hb, oracle, ll_frames, in_lay, out_lay, J, levels, variant):
    """J = 1 is ll_tone alone.  Its 16-byte vector path needs 16-byte aligned rows and planes, not positive strides:
    the wide dense frame takes it, and so do frames flipped in rows or channels whose pitch is a multiple of 16 samples,
    on both sides; every other case on the wide frame takes the scalar path."""
    alpha = 1.0 / (levels - 1)

    def call(bi, bo):
        hb.filters.local_laplacian_pyramid_levels(bi, J, levels, alpha, 1.0, bo)
    for size, img in ll_frames.items():
        (logical,), got, ran, (bi, bo) = layout_call(hb, call, [img], [in_lay], (3,) + size, np.uint16, out_lay, variant)
        same(got, oracle.local_laplacian(logical, levels, alpha, 1.0, pyramid_levels=J), f"{size} {in_lay} -> {out_lay}")
        if J == 1:
            assert set(ran) <= {"ll_lut", "ll_tone"} and "ll_tone" in ran, sorted(ran)
            if size == WIDE:
                a16 = lambda lay: lay in A16 or lay == "dense"
                assert ll_tone_vec(bi, bo) == (a16(in_lay) and a16(out_lay)), (in_lay, out_lay)
            elif in_lay in A16 and out_lay in A16:  # (53 columns pad to 56, itself 16-byte aligned: no "not" here)
                assert ll_tone_vec(bi, bo), (in_lay, out_lay)


def ll_tone_vec(bi, bo):
    """local_laplacian.cu launch_tone: the 16-byte vector form needs the first sample read and written, and every row
    and channel stride, 16-byte aligned (input and output at the same mins)."""
    a16 = lambda b: b % 16 == 0
    return (a16(bi.buf.buf.device) and a16(bo.buf.buf.device) and
            all(a16(2 * s) for s in bi.strides()[1:3] + bo.strides()[1:3]))


# ---- bilateral_grid ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("s_sigma", [None, 3, 128])
@pytest.mark.parametrize("in_lay,out_lay", pairs(["pad", "flip_y", "flip_y_odd", "bcast_y"], ["flip_y", "flip_y_odd"],
                                                 [("flip_y", "flip_y")]))
def test_bilateral_grid(hb, oracle, in_lay, out_lay, s_sigma, variant):
    """None: bilateral_grid (s_sigma 8); otherwise bilateral_grid_s_sigma."""
    r = 0.1
    if s_sigma is None:
        call = lambda bi, bo: hb.filters.bilateral_grid(bi, r, bo)
    else:
        call = lambda bi, bo: hb.filters.bilateral_grid_s_sigma(bi, s_sigma, r, bo)
    for size in [(H, W), WIDE]:
        img = f32_frame(size, size[1])
        (logical,), got, _, _ = layout_call(hb, call, [img], [in_lay], size, np.float32, out_lay, variant)
        close(got, oracle.bilateral_grid(logical, r, s_sigma=s_sigma or 8), 1e-6, f"{size} {in_lay} -> {out_lay}")
        same(got, dense_call(hb, call, [logical], size, np.float32), "against the dense call")


# ---- nl_means ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kernel_variant,kernel", [(0, "nl_means_window"), (1, "nl_means")])
@pytest.mark.parametrize("in_lay,out_lay", pairs(["flip_c", "bcast_c", "flip_y", "xcy"], ["flip_y", "flip_c", "xcy"]))
def test_nl_means(hb, oracle, in_lay, out_lay, kernel_variant, kernel, variant):
    """bcast_c: one grey plane read as 3 channels."""
    img = f32_frame((3, H, W), 9)
    call = lambda bi, bo: hb.filters.nl_means(bi, 3, 7, 0.12, bo)
    with nl_means_variant(hb, kernel_variant):
        (logical,), got, ran, _ = layout_call(hb, call, [img], [in_lay], (3, H, W), np.float32, out_lay, variant)
        dense = dense_call(hb, call, [logical], (3, H, W), np.float32)
    assert list(ran) == [kernel], sorted(ran)
    close(got, oracle.nl_means(logical, 3, 7, 0.12), 1e-3, f"{in_lay} -> {out_lay}")
    same(got, dense, "against the dense call")


# ---- stencil_chain ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("stencils", [None, 1, 5, 32])
@pytest.mark.parametrize("in_lay,out_lay", pairs(["pad", "flip_y", "flip_y_odd", "bcast_y"], ["flip_y", "flip_y_odd"],
                                                 [("flip_y_odd", "flip_y")]))
def test_stencil_chain(hb, oracle, in_lay, out_lay, stencils, variant):
    """None: stencil_chain; otherwise stencil_chain_stencils."""
    if stencils is None:
        call = hb.filters.stencil_chain
    else:
        call = lambda bi, bo: hb.filters.stencil_chain_stencils(bi, stencils, bo)
    for size in [(H, W), WIDE]:
        img = u16_frame(size, size[0] + (stencils or 0))
        (logical,), got, _, _ = layout_call(hb, call, [img], [in_lay], size, np.uint16, out_lay, variant)
        same(got, oracle.stencil_chain(logical, stencils=stencils or 32), f"{size} {in_lay} -> {out_lay}")


# ---- camera_pipe ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("raw_lay,mat_lay,out_lay", [("flip_y", "dense", "dense"), ("flip_y_odd", "dense", "dense"),
                                                     ("dense", "flip_y", "dense"), ("dense", "dense", "flip_y"),
                                                     ("dense", "dense", "flip_y_odd"), ("flip_y", "flip_y", "flip_y")])
def test_camera_pipe(hb, oracle, raw_lay, mat_lay, out_lay, variant):
    params = cp_params({})
    out_shape = (3, 37, 61)
    q = hb.HalideBuffer.bounds_query(np.uint16, 2)
    hb.filters.camera_pipe(q, hb.HalideBuffer.from_numpy(CP_M3200.copy()), hb.HalideBuffer.from_numpy(CP_M7000.copy()),
                           *params, hb.HalideBuffer.from_numpy(np.zeros(out_shape, np.uint8), host_dirty=False))
    (x0, w, _), (y0, h, _) = q.shape()
    raw = (u16_frame((h, w), 11) & np.uint16(1023))

    def call(br, b32, b70, bo):
        hb.filters.camera_pipe(br, b32, b70, *params, bo)
    (lraw, m32, m70), got, _, _ = layout_call(hb, call, [raw, CP_M3200, CP_M7000], [raw_lay, mat_lay, mat_lay], out_shape,
                                              np.uint8, out_lay, variant, in_mins=[(x0, y0), None, None])
    same(got, oracle.camera_pipe(lraw, m32, m70, *params, out_shape, in_mins=(x0, y0)), f"{raw_lay}/{mat_lay} -> {out_lay}")


# ---- conv_layer_any_shape --------------------------------------------------------------------------------------------
# numpy axes: input [n, y, x, ci], filter [ci, ky, kx, co], output [n, y, x, co]
# CI = 19 with even padded pitches: the split-input kernel's scalar loads; CI = 20 with pitches of 16 samples: its vector
# form (vec4, conv_layer_tc.cu), for flipped and broadcast inputs alike
CONV_SHAPES = {False: (2, 19, 24, 13, 9), True: (2, 20, 24, 13, 9)}  # (N, CI, CO, W, H)
D = "dense"


def conv_vec4(bi, ci):
    """conv_layer_tc.cu: the split-input kernel reads float4s when CI, the input's x / y / n strides are multiples of 4
    and its element at the mins is 16-byte aligned."""
    return ci % 4 == 0 and bi.buf.buf.device % 16 == 0 and all(s % 4 == 0 for s in bi.strides()[1:4])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("aligned", [False, True], ids=["ci19", "ci20_a16"])
@pytest.mark.parametrize("lays", [(("bcast", 0), D, D), (("flip", 2), D, D), (("flip", 1), D, D), (D, ("flip", 0), D),
                                  (D, D, ("flip", 2)), (D, D, ("flip", 1)), (("flip", 1), ("flip", 0), ("flip", 2))],
                         ids=["bcast_n", "in_flip_x", "in_flip_y", "filter_flip_ci", "out_flip_x", "out_flip_y", "all"])
def test_conv_layer_any_shape(hb, oracle, lays, aligned, variant):
    shape = CONV_SHAPES[aligned]
    n, ci, co, w, h = shape
    inp, filt, bias = cx.harness("rand", shape)
    if aligned:
        lays = [l if l == D else (l[0] + "16", l[1]) for l in lays]

    def call(bi, bf, bb, bo):
        hb.filters.conv_layer_any_shape(bi, bf, bb, bo)
    (li, lf, lb), got, ran, (bi, _, _, _) = layout_call(hb, call, [inp, filt, bias], [lays[0], lays[1], D], (n, h, w, co),
                                                        np.float32, lays[2], variant)
    assert "conv_split_input_any" in ran, sorted(ran)
    assert conv_vec4(bi, ci) == aligned
    same(got, cx.run(hb, li, lf, lb), "against the dense call")
    close(got, oracle.conv_layer(li, lf, lb), 1e-6, str(lays))


# ---- row-sharded local_laplacian on bands in these layouts -----------------------------------------------------------

def _rank_main(rank, world, img, lay):
    """One rank of a loopback group: its band of `img` as input and output in layout `lay` (a broadcast input: row lo of
    the band read as every row, a dense output).  Returns (return code, error message, output band)."""
    import halide_b200
    from halide_b200.dist import band_rows
    l = halide_b200.load_library()
    rc = l.halide_b200_dist_init_loopback(rank, world)
    if rc:
        return rc, halide_b200.lib.last_error_message(), None
    try:
        c, h, w = img.shape
        lo, hi = band_rows(rank, world, h)
        band = img[:, lo:hi + 1, :]
        bi = Buf(halide_b200, band.shape, np.uint16, lay, "host", (0, lo, 0), band)
        bo = Buf(halide_b200, band.shape, np.uint16, "dense" if lay.startswith("bcast") else lay, "host", (0, lo, 0))
        rc = l.halide_b200_local_laplacian_sharded(bi.ptr, LEVELS, ctypes.c_float(ALPHA), ctypes.c_float(1.0), bo.ptr, 0, h)
        if rc:
            return rc, halide_b200.lib.last_error_message(), None
        return 0, "", bo.read()
    finally:
        l.halide_b200_dist_shutdown()


SHARD_LAYOUTS = ["flip_y", "flip_c", "pad", "xcy", "bcast_y"]


@pytest.mark.parametrize("level", [0, 2])
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("lay", SHARD_LAYOUTS)
def test_sharded_bands(hb, lay, world, level):
    """Bands whose halo rows are packed for the neighbours through a flipped, zero, padded or line-interleaved row
    stride; the gathered level chosen by size and forced to 2.  The bands put together equal the single-GPU filter bit for bit.
    Every case has a frame of its own: a pooled halo block left from an earlier call on the same frame would hide a pack
    that never ran."""
    from halide_b200.dist import band_rows
    img = u16_frame(FRAMES[world][0], 300 + 10 * world + level + 1000 * SHARD_LAYOUTS.index(lay))
    frame = img.copy()
    if lay == "bcast_y":  # (the frame the bands describe: each band's first row repeated)
        for r in range(world):
            lo, hi = band_rows(r, world, img.shape[1])
            frame[:, lo:hi + 1] = img[:, lo:lo + 1]
    want = _single(hb, frame)
    with _settings(level):
        futs = [_RANK_THREADS[r].submit(_rank_main, r, world, img, lay) for r in range(world)]
        res = [f.result(timeout=300) for f in futs]
    for r, (rc, msg, _) in enumerate(res):
        assert rc == 0, f"rank {r} of {world}: error {rc}: {msg}"
    same(np.concatenate([o for _, _, o in res], axis=1), want, f"{lay} over {world} ranks")


# ---- uploads and copies of broadcast buffers --------------------------------------------------------------------------

def test_broadcast_clip_uploads_one_frame(hb):
    """An 8-frame clip broadcast from one 3 x 540 x 960 frame (stride 0 over frames): the runtime copies the frame once,
    at most one host-to-device copy per frame-sized dense block instead of one 2-byte copy per sample, and the batched
    filter on the uploaded clip gives every frame the single-frame result."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    frame = u16_frame((3, 540, 960), 12)
    clip = np.broadcast_to(frame, (8,) + frame.shape)
    b = hb.HalideBuffer.from_numpy(clip)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        hb.lib.check(hb.capi.halide_copy_to_device(None, b.ptr, None))
        torch.cuda.synchronize()
    copies = [e.name for e in prof.events() if "memcpy" in e.name.lower() and "htod" in e.name.lower().replace(" ", "")]
    assert len(copies) == 1, (len(copies), copies[:4])  # the clip holds one dense frame (and a profiler that records
    # nothing fails too)
    out = np.zeros(clip.shape, np.uint16)
    bo = hb.HalideBuffer.from_numpy(out, host_dirty=False)
    hb.filters.local_laplacian_batch(b, LEVELS, ALPHA, 1.0, bo)
    bo.copy_to_host()
    want = np.zeros(frame.shape, np.uint16)
    hb.filters.local_laplacian(hb.HalideBuffer.from_numpy(frame), LEVELS, ALPHA, 1.0,
                               bw := hb.HalideBuffer.from_numpy(want, host_dirty=False))
    bw.copy_to_host()
    for k in range(clip.shape[0]):
        same(out[k], want, f"frame {k}")


@pytest.mark.parametrize("lay", ["bcast_y", "bcast_c", "bcast_n"])
@pytest.mark.parametrize("to_device", [True, False])
def test_buffer_copy_from_broadcast_replicates(hb, lay, to_device):
    """halide_buffer_copy from a broadcast host source into a dense destination, on the device or the host, writes every
    index of the broadcast dimension: only a dimension of stride 0 on both sides carries no data."""
    shape = (2, 3, H, W)
    src_shape, view_of = layout(shape, lay)
    mem = u16_frame(src_shape, 13)
    src = view_of(mem)[1]
    want = np.ascontiguousarray(src)
    bs = hb.HalideBuffer.from_numpy(src)
    dst = np.zeros(shape, np.uint16)
    bd = hb.HalideBuffer.from_numpy(dst, host_dirty=False)
    iface = hb.capi.halide_cuda_device_interface() if to_device else None
    hb.lib.check(hb.capi.halide_buffer_copy(None, bs.ptr, ctypes.c_void_p(iface), bd.ptr))
    if to_device:
        bd.copy_to_host()
    same(dst, want, "broadcast copy")
