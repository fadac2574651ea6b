"""GPU tests of halide_b200_local_laplacian_batch: every output frame of a batch must equal, bit for bit, the single-frame
local_laplacian call on that frame (the two share every kernel; a batch only adds the frame index), and small batches
equal the oracle frame by frame.  Each frame of a batch has its own seeded content and one frame is constant, so work
that lands in the wrong frame's slice shows up."""
import numpy as np
import pytest

from util import run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
ALPHA = 1.0 / 7.0


def make_batch(n, h, w, seed, c=3):
    """(n, c, h, w) uint16: frame k from seed 1000 * seed + k; frame 1 (when there is one) constant per channel."""
    a = np.stack([u16_frame((c, h, w), 1000 * seed + k) for k in range(n)])
    if n >= 2:
        for ch in range(c):
            a[1, ch] = (20000, 41000, 9000, 30000)[ch % 4]
    return a


def strided_copy(a, row_pad=0, frame_pad=0):
    """A view of `a`'s values whose rows are row_pad elements longer and whose frames are frame_pad elements further apart
    than dense."""
    n, c, h, w = a.shape
    pitch = w + row_pad
    fs = c * h * pitch + frame_pad
    flat = np.zeros(n * fs, np.uint16)
    v = np.lib.stride_tricks.as_strided(flat, shape=a.shape, strides=(2 * fs, 2 * h * pitch, 2 * pitch, 2))
    v[...] = a
    return v


def run_batch(hb, inp, levels, alpha, beta, out=None, in_mins=None, out_mins=None):
    if out is None:
        out = np.zeros(inp.shape, np.uint16)
    bi = hb.HalideBuffer.from_numpy(inp, in_mins)
    bo = hb.HalideBuffer.from_numpy(out, out_mins, host_dirty=False)
    hb.filters.local_laplacian_batch(bi, levels, alpha, beta, bo)
    assert bo.device_dirty
    bo.copy_to_host()
    return out


def assert_frames_equal(got, want, what=""):
    for k in range(got.shape[0]):
        bad = np.argwhere(got[k] != want[k])
        assert bad.size == 0, (f"{what} frame {k}: {len(bad)} mismatching samples, first at (c,y,x)={bad[0]}: "
                               f"got {got[k][tuple(bad[0])]} want {want[k][tuple(bad[0])]}")


def single_calls(hb, a, levels, alpha, beta, **kw):
    return np.stack([run_local_laplacian(hb, np.ascontiguousarray(a[k]), levels, alpha, beta, **kw) for k in range(a.shape[0])])


@pytest.mark.parametrize("n,w,h,levels,beta", [
    (1, 67, 91, 8, 1.0), (2, 67, 91, 8, 0.5), (3, 67, 91, 5, 1.0), (5, 67, 91, 8, 1.0),
    (3, 517, 333, 8, 1.0), (5, 517, 333, 5, 0.5), (2, 517, 333, 8, 0.5), (1, 517, 333, 8, 1.0),
])
def test_small_batches_match_single_calls_and_oracle(hb, oracle, n, w, h, levels, beta):
    """67 x 91 frames put level 2 into the cooperative coarse launch; 517 x 333 are odd sizes.  levels 8 takes the fast
    kernels, levels 5 the generic ones; beta 1 and 0.5 are the two BETA1 instantiations."""
    alpha = 1.0 / (levels - 1)
    a = make_batch(n, h, w, n * 31 + levels)
    got = run_batch(hb, a, levels, alpha, beta)
    assert_frames_equal(got, single_calls(hb, a, levels, alpha, beta), "single call")
    want = np.stack([oracle.local_laplacian(np.ascontiguousarray(a[k]), levels, alpha, beta) for k in range(n)])
    assert_frames_equal(got, want, "oracle")


@pytest.mark.parametrize("n,w,h,beta", [(1, 1920, 1080, 1.0), (3, 1920, 1080, 1.0), (2, 1920, 1080, 0.5),
                                        (2, 3840, 2160, 1.0)])
def test_video_frames_match_single_calls(hb, n, w, h, beta):
    a = make_batch(n, h, w, 7 + n)
    got = run_batch(hb, a, 8, ALPHA, beta)
    assert_frames_equal(got, single_calls(hb, a, 8, ALPHA, beta))


def test_mins_and_a_larger_input(hb, oracle):
    """Nonzero and negative mins in every dimension; the input is larger than the output in x, y, c and n, and the
    output takes frames 1..3 of its 5 frames (repeat_edge clamps at the input's own x / y / c bounds, frame by frame)."""
    h, w = 71, 97
    inp = make_batch(5, h + 9, w + 14, 3, c=4)
    in_mins, out_mins = (-5, 3, -1, -2), (-2, 5, 0, -1)
    out = np.zeros((3, 3, h, w), np.uint16)
    got = run_batch(hb, inp, 8, ALPHA, 1.0, out=out, in_mins=in_mins, out_mins=out_mins)
    kw = dict(out_shape=(3, h, w), in_mins=in_mins[:3], out_mins=out_mins[:3])
    frames = inp[1:4]
    assert_frames_equal(got, single_calls(hb, frames, 8, ALPHA, 1.0, **kw), "single call")
    want = np.stack([oracle.local_laplacian(np.ascontiguousarray(f), 8, ALPHA, 1.0, **kw) for f in frames])
    assert_frames_equal(got, want, "oracle")


@pytest.mark.parametrize("w,row_pad,frame_pad", [
    (256, 0, 0),    # frame stride a 16-byte multiple: the final kernel's 4-D TMA frame tile
    (250, 6, 0),    # padded rows, frame stride still a 16-byte multiple
    (256, 0, 2),    # frame stride even but no 16-byte multiple: aligned loads without TMA
    (256, 0, 1),    # odd frame stride: general addressing in the final kernel, unpaired loads in the level-1 kernel
    (250, 3, 5),    # odd row and frame strides
])
def test_row_and_frame_strides(hb, w, row_pad, frame_pad):
    h = 150
    a = make_batch(3, h, w, w + row_pad + frame_pad)
    want = single_calls(hb, a, 8, ALPHA, 1.0)
    inp = strided_copy(a, row_pad, frame_pad)
    out = strided_copy(np.zeros_like(a), row_pad + 2, frame_pad + 2)
    assert_frames_equal(run_batch(hb, inp, 8, ALPHA, 1.0, out=out), want)
    assert_frames_equal(run_batch(hb, inp, 8, ALPHA, 0.5), single_calls(hb, a, 8, ALPHA, 0.5), "beta 0.5")


@pytest.mark.parametrize("mask", [1, 2, 4, 8, 16, 64, 7, 1 | 8, 2 | 4, 16 | 64])
def test_force_generic_masks(hb, mask):
    """Every hook bit routes the batch through another kernel (generic down / up / final, no cooperative tail,
    general-layout final kernel, no TMA frame tile); each must keep the frames apart."""
    a = make_batch(3, 131, 204, mask)
    want = single_calls(hb, a, 8, ALPHA, 1.0)
    l = hb.load_library()
    try:
        l.halide_b200_ll_force_generic(mask)
        got = run_batch(hb, a, 8, ALPHA, 1.0)
    finally:
        l.halide_b200_ll_force_generic(0)
    assert_frames_equal(got, want, f"mask {mask}")


def test_torch_device_batch_on_the_current_stream(hb):
    """An (N, 3, H, W) uint16 clip already on the device, wrapped with from_torch, filtered on torch's current stream."""
    import ctypes

    import torch
    from halide_b200 import HalideBuffer, filters
    a = make_batch(4, 240, 320, 11)
    want = single_calls(hb, a, 8, ALPHA, 1.0)
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    stream = torch.cuda.Stream()
    try:
        with torch.cuda.stream(stream):
            t_in = torch.from_numpy(a.view(np.int16)).cuda().view(torch.uint16)
            t_out = torch.zeros_like(t_in)
            l.halide_b200_set_stream(ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
            bi, bo = HalideBuffer.from_torch(t_in), HalideBuffer.from_torch(t_out)
            filters.local_laplacian_batch(bi, 8, ALPHA, 1.0, bo)
            got = t_out.view(torch.int16).cpu().numpy().view(np.uint16)  # (ordered after the filter on the same stream)
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
    assert_frames_equal(got, want)


def test_consecutive_calls_with_different_frame_counts(hb):
    """Scratch and plan reuse between calls of one thread: 4 frames, then 2 of another size, then 4 again, then 1."""
    a4 = make_batch(4, 200, 264, 21)
    a2 = make_batch(2, 333, 517, 22)
    want4, want2 = single_calls(hb, a4, 8, ALPHA, 1.0), single_calls(hb, a2, 8, ALPHA, 1.0)
    assert_frames_equal(run_batch(hb, a4, 8, ALPHA, 1.0), want4, "first N=4")
    assert_frames_equal(run_batch(hb, a2, 8, ALPHA, 1.0), want2, "N=2")
    assert_frames_equal(run_batch(hb, a4, 8, ALPHA, 1.0), want4, "second N=4")
    assert_frames_equal(run_batch(hb, a4[2:3], 8, ALPHA, 1.0), want4[2:3], "N=1")
