"""local_laplacian off the 3-channel planar path, bit-exact against the oracle.

The filter's gray image reads absolute channels 0..2 clamped into the input's channel range (repeat_edge), while the
colour stage reads the unclamped input channel of each output channel (generator :84).  So output channel crops,
inputs with fewer than 3 channels or a channel min other than 0, four channels, and layouts whose channel stride is
smaller than their row stride each take kernel branches the 3-channel planar frames never reach: the final kernel's
general-layout path (ll_up2 with FINAL and not ALIGNED), the generic final kernel that runs for more than 3 output
channels, and the aligned / TMA frame tile with a tensor map over more than 3 channels."""
from contextlib import contextmanager

import numpy as np
import pytest

from test_dist_loopback_gpu import _run as run_sharded_ranks
from test_dist_loopback_gpu import _settings as shard_settings
from test_ll_batch_gpu import assert_frames_equal, make_batch, run_batch
from util import kernels_run, run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
LEVELS, ALPHA = 8, 1.0 / 7.0
# halide_b200_ll_force_generic bits: 1 = generic down kernels, 4 = generic final kernel, 16 = general-layout final
# kernel, 64 = no TMA frame tile in the final kernel
MASKS = [0, 1, 4, 16, 64]


@contextmanager
def force_generic(hb, mask):
    l = hb.load_library()
    l.halide_b200_ll_force_generic(mask)
    try:
        yield
    finally:
        l.halide_b200_ll_force_generic(0)


def assert_same(got, want, what=""):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"{what}: {len(bad)} mismatching samples, first at (c,y,x)={bad[0]}: "
                           f"got {got[tuple(bad[0])]} want {want[tuple(bad[0])]}")


def expected_kernels(mask, out_c):
    """Kernel names the launch sequence must contain (levels 8): the fast level-1 kernel unless bit 1 forces the generic
    one; the fast final kernel (which computes outGPyramid[1] itself) for up to 3 output channels unless bit 4 forces the
    generic final kernel."""
    down = "ll_level1_generic" if mask & 1 else "ll_level1"
    final = "ll_final" if (mask & 4) or out_c > 3 else "ll_final2"
    return down, final


def check(hb, oracle, img, out_shape, in_mins, out_mins, mask=0, beta=1.0, levels=LEVELS, alpha=ALPHA):
    want = oracle.local_laplacian(img, levels, alpha, beta, out_shape=out_shape, in_mins=in_mins, out_mins=out_mins)
    with force_generic(hb, mask), kernels_run(hb) as ran:
        got = run_local_laplacian(hb, img, levels, alpha, beta, out_shape=out_shape, in_mins=in_mins, out_mins=out_mins)
    assert_same(got, want, f"mask {mask} beta {beta}")
    down, final = expected_kernels(mask, out_shape[0])
    assert down in ran and final in ran, sorted(ran)
    assert ("ll_final2" in ran) == (final == "ll_final2"), sorted(ran)
    return ran


# (mask, beta): every hook bit at beta 1, and the default path at beta != 1 (the final kernel's BETA1 instantiations)
MASK_BETA = [(m, 1.0) for m in MASKS] + [(0, 0.6)]


@pytest.mark.parametrize("mask,beta", MASK_BETA)
@pytest.mark.parametrize("out_c,out_c0", [(1, 0), (1, 1), (1, 2), (2, 0), (2, 1)])
def test_output_channel_crops(hb, oracle, out_c, out_c0, mask, beta):
    """Output channels [out_c0, out_c0 + out_c) of a 3-channel input: fewer than 3 output channels, or an output that
    starts past channel 0, take the final kernel's general-layout path, whose colour stage reads input channel
    out_c0 + c and stores only c < C (or the generic final kernel under bit 4)."""
    img = u16_frame((3, 67, 96), 10 * out_c + out_c0)
    check(hb, oracle, img, (out_c, 67, 96), (0, 0, 0), (0, 0, out_c0), mask, beta)


@pytest.mark.parametrize("mask,beta", [(0, 1.0), (1, 1.0), (4, 1.0), (0, 0.6)])
@pytest.mark.parametrize("in_c,out_c,out_c0", [(1, 1, 0), (2, 2, 0), (2, 1, 1)])
def test_inputs_with_fewer_than_three_channels(hb, oracle, in_c, out_c, out_c0, mask, beta):
    """A 1- or 2-channel input: gray reads channel min(c, in_c - 1) for c = 0..2 in every kernel that recomputes it (the
    level-1 kernels and the final kernel), the colour stage reads the output's own channel."""
    img = u16_frame((in_c, 53, 74), 100 * in_c + out_c0)
    check(hb, oracle, img, (out_c, 53, 74), (0, 0, 0), (0, 0, out_c0), mask, beta)


@pytest.mark.parametrize("mask,beta", [(0, 1.0), (1, 1.0), (4, 1.0), (0, 0.6)])
@pytest.mark.parametrize("out_c,out_c0", [(3, 1), (1, 2)])
def test_input_channel_min_one(hb, oracle, out_c, out_c0, mask, beta):
    """Input channels [1, 4): gray reads absolute channels 1, 1, 2 (channel 0 clamps to the input's first channel); the
    colour stage reads input channel out_c0 + c - 1.  A 3-channel output at channel 1 is not the aligned layout (that
    needs both channel mins at 0), so it takes the general-layout path too."""
    img = u16_frame((3, 61, 88), 7 + out_c0)
    check(hb, oracle, img, (out_c, 61, 88), (0, 0, 1), (0, 0, out_c0), mask, beta)


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("mask", [0, 1])
def test_four_channel_input_and_output(hb, oracle, mask, beta):
    """Four output channels: the fast down-sweep (or the generic one under bit 1) followed by the generic final kernel
    and a level-1 up-sweep launch, since the fast final kernel covers at most 3 channels."""
    img = u16_frame((4, 70, 104), 44)
    check(hb, oracle, img, (4, 70, 104), (0, 0, 0), (0, 0, 0), mask, beta)


def tma_frame_tile(in_w, in_h, in_c, out_x0, in_x0=0):
    """The host's choice of the final kernel's TMA frame tile for a dense planar uint16 input at a 16-byte aligned
    base: row and channel strides in bytes must be 16-byte multiples and every tile's first column must start on one."""
    return (2 * in_w) % 16 == 0 and (2 * in_w * in_h) % 16 == 0 and (((out_x0 & ~1) - in_x0) & 7) == 0


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("mask", [0, 64, 16])
def test_four_channel_input_three_channel_output_tma(hb, oracle, mask, beta):
    """A 4-channel input with output channels [0, 3) and rows 16 bytes apart: the aligned layout test and the TMA map
    accept in_c >= 3, so the frame tile is fetched through a tensor map whose channel dimension is 4 (its box takes
    channels 0..2).  Bit 64 takes the aligned loads without TMA on the same frame, bit 16 the general-layout path."""
    h, w = 96, 136
    assert tma_frame_tile(w, h, 4, 0)
    img = u16_frame((4, h, w), 45)
    check(hb, oracle, img, (3, h, w), (0, 0, 0), (0, 0, 0), mask, beta)


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("out_x0", [6, 2, 5])
def test_four_channel_input_cropped_in_x(hb, oracle, out_x0, beta):
    """The same 4-channel input, output columns starting inside it: an even offset that is no multiple of 8 columns
    keeps the aligned path but not the TMA frame tile (its tiles would not start on 16 bytes); an odd offset leaves the
    aligned path for the general-layout one."""
    h, w = 96, 136
    assert not tma_frame_tile(w, h, 4, out_x0)
    img = u16_frame((4, h, w), 46 + out_x0)
    check(hb, oracle, img, (3, h - 10, w - 16), (0, 0, 0), (out_x0, 3, 0), 0, beta)


# ---- layouts that are not planar, on device-resident torch tensors -----------------------------------------------------

def interleaved_rows(h, w, row_pitch, values=None):
    """(3, h, w) uint16 in memory order (x, c, y): channel stride w, row stride row_pitch >= 3 w.  Returns the numpy
    base array and the (c, y, x) view of it."""
    base = np.zeros(h * row_pitch, np.uint16)
    view = np.lib.stride_tricks.as_strided(base, shape=(3, h, w), strides=(2 * w, 2 * row_pitch, 2))
    if values is not None:
        view[...] = values
    return base, view


@pytest.mark.parametrize("mask", [0, 64, 16])
@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("h,w,pad", [(80, 128, 0), (80, 128, 8), (57, 98, 3)])
def test_channel_stride_smaller_than_row_stride(hb, oracle, h, w, pad, mask, beta):
    """Input and output of memory order (x, c, y), strides (1, 3W + pad, W), wrapped as device buffers (no runtime
    copy).  W = 128 passes every even-stride check of the aligned layout test and, with rows 16 bytes apart, reaches the
    TMA frame tile with a tensor map whose channel stride is smaller than its row stride (if the driver refuses such a
    map, the aligned loads run instead); bits 64 and 16 force the aligned loads and the general-layout path.  The odd
    pitch of W = 98, pad 3 takes the general-layout path by itself.  The output's padding must stay untouched."""
    import torch
    from halide_b200 import HalideBuffer, filters
    pitch = 3 * w + pad
    src_base, img = interleaved_rows(h, w, pitch, u16_frame((3, h, w), h + w + pad))
    want = oracle.local_laplacian(img, LEVELS, ALPHA, beta)
    t_in_base = torch.from_numpy(src_base.view(np.int16)).cuda().view(torch.uint16)
    t_out_base = torch.zeros(h * pitch, dtype=torch.int16, device="cuda").view(torch.uint16)
    t_in = t_in_base.as_strided((3, h, w), (w, pitch, 1))
    t_out = t_out_base.as_strided((3, h, w), (w, pitch, 1))
    bi, bo = HalideBuffer.from_torch(t_in), HalideBuffer.from_torch(t_out)
    assert [d[2] for d in bi.shape()] == [1, pitch, w]
    with force_generic(hb, mask), kernels_run(hb) as ran:
        filters.local_laplacian(bi, LEVELS, ALPHA, beta, bo)
        bo.device_sync()
    torch.cuda.synchronize()
    out_base = t_out_base.view(torch.int16).cpu().numpy().view(np.uint16)
    got = np.lib.stride_tricks.as_strided(out_base, shape=(3, h, w), strides=(2 * w, 2 * pitch, 2))
    assert_same(np.ascontiguousarray(got), want, f"pitch {pitch} mask {mask}")
    if pad:
        assert not out_base.reshape(h, pitch)[:, 3 * w:].any(), "the filter wrote into the row padding"
    assert "ll_level1" in ran and "ll_final2" in ran, sorted(ran)
    del bi, bo


# ---- batches and row shards of 1 and 4 channels ---------------------------------------------------------------------

@pytest.mark.parametrize("c", [1, 4])
def test_batch_of_one_and_four_channels(hb, oracle, c):
    """halide_b200_local_laplacian_batch on (N, C, H, W) clips of 1 and 4 channels (the 4-channel one runs the generic
    final kernel with the frame index): every frame must equal its own single-frame oracle call."""
    n, h, w = 3, 58, 90
    a = make_batch(n, h, w, 60 + c, c=c)
    with kernels_run(hb) as ran:
        got = run_batch(hb, a, LEVELS, ALPHA, 1.0)
    want = np.stack([oracle.local_laplacian(np.ascontiguousarray(a[k]), LEVELS, ALPHA, 1.0) for k in range(n)])
    assert_frames_equal(got, want, f"{c} channels")
    assert ("ll_final" if c > 3 else "ll_final2") in ran, sorted(ran)


@pytest.mark.parametrize("c,world,shape", [(1, 2, (1, 517, 333)), (4, 3, (4, 601, 256))])
def test_row_sharded_one_and_four_channels(hb, oracle, c, world, shape):
    """halide_b200_local_laplacian_sharded on `world` rank threads of one GPU (in-process loopback group), for a 1- and
    a 4-channel frame: the input halo is exchanged per input channel and the level-1 kernel reads it by clamped channel
    index.  The bands put together must equal the oracle on the whole frame."""
    img = u16_frame(shape, 500 + c)
    want = oracle.local_laplacian(img, LEVELS, ALPHA, 1.0)
    with shard_settings():
        res = run_sharded_ranks(world, [(img, 1)])
    for r, (rc, msg, _) in enumerate(res):
        assert rc == 0, f"rank {r} of {world}: error {rc}: {msg}"
    got = np.concatenate([res[r][2][0] for r in range(world)], axis=1)
    assert_same(got, want, f"{c} channels over {world} ranks")
