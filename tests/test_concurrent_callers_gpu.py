"""Every filter entry point under concurrent callers and on a stream whose input is not ready yet (INTEGRATION.md §2,
Threads: calls are re-entrant, the stream is thread-local, scratch recycles through per-stream free lists, and the
library orders its work after the caller's stream), and the lifetime of local_laplacian's cached remap tables.

- JOBS: one closure-like job per entry point variant, each on a frame size of its own, together running every kernel
  the library launches.  The serial baseline runs each once and checks it against the oracle.
- Four threads, each on its own stream, run every job in their own order for three rounds: every result must be the
  baseline's bytes.
- On a torch stream: sentinel input, a sleep, the real input, a sentinel output, the call, a clone of the output, all
  enqueued before one synchronise: the clone must be the baseline's bytes.
- A remap table held (halide_b200_ll_lut_hold) survives evictions and is evicted once dropped; threads sweeping 160
  alphas get the serial results."""
import ctypes
import glob
import inspect
import os
import re
import threading
from dataclasses import dataclass, field

import numpy as np
import pytest

import conv_any_exact as cx
import conv_exact
import ll_bordered
from bilateral_grid_exact import dyadic
from halide_b200.image_io import convert
from test_camera_pipe_edges_gpu import raw_frame
from util import CP_M3200, CP_M7000, cp_params, f32_frame, kernels_run, u16_frame

pytestmark = pytest.mark.gpu
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "halide_b200", "csrc")
CP = cp_params({})
FLOAT_RTOL = 1e-4  # the float pipelines' tolerance against the oracle where they are not bit for bit (conv_layer)


# ---- jobs -----------------------------------------------------------------------------------------------------------

@dataclass
class In:
    """An input array (numpy, outermost-first); `view` maps the array (numpy or torch) to what the buffer describes."""
    array: np.ndarray
    view: object = None


@dataclass
class Out:
    """An output of this numpy shape and type, described through `view` like an In."""
    shape: tuple
    dtype: object
    view: object = None


@dataclass
class Job:
    name: str
    entry: str                # the function of halide_b200.filters
    args: list                # In, Out and scalars in the entry point's order
    want: object              # oracle -> the expected outputs, one per Out, as the Out arrays hold them
    rtol: float = None        # None: bit for bit
    kernels: set = field(default_factory=set)  # kernels this job alone must launch


def il(a):
    """A pixel-interleaved array ([n,] y, x, c) as the (x, y, c[, n]) buffer of it: c moved in front of y."""
    axes = (0, 3, 1, 2) if a.ndim == 4 else (2, 0, 1)
    return a.permute(*axes) if hasattr(a, "permute") else a.transpose(axes)


def planar(a):
    """Planar ([n,] c, y, x) copy of an interleaved numpy array."""
    return np.ascontiguousarray(il(a))


def u8_frame(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def ll_oracle(oracle, frames, levels, alpha, beta, pyramid_levels=8, u8=False):
    """The oracle on one planar frame or on each frame of a batch; 8-bit frames through to_u16 and to_u8."""
    def one(f):
        if u8:
            return convert(oracle.local_laplacian(convert(f, np.uint16), levels, alpha, beta), np.uint8)
        # (past 11 levels the literal evaluation's borders grow too large: the bordered one, test_ll_pyramid_levels.py)
        evaluate = ll_bordered.local_laplacian if pyramid_levels > 11 else oracle.local_laplacian
        return evaluate(f, levels, alpha, beta, pyramid_levels=pyramid_levels)
    return one(frames) if frames.ndim == 3 else np.stack([one(f) for f in frames])


def cp_oracle(oracle, raw, out_chw):
    return oracle.camera_pipe(raw, CP_M3200, CP_M7000, *CP, out_chw)


def make_jobs():
    jobs = []
    seed = iter(range(100, 1000))

    def add(*a, **kw):
        jobs.append(Job(*a, **kw))

    # halide_blur: pixel pairs 4-byte aligned on every row (even strides) take the quad kernel, odd strides the general one
    for name, (h, w), kern in [("blur_even", (70, 130), "blur3x3_u16_quad"), ("blur_odd", (61, 99), "blur3x3_u16")]:
        x = u16_frame((h, w), next(seed))
        add(name, "halide_blur", [In(x), Out((h - 2, w - 2), np.uint16)], lambda o, x=x: [o.blur(x)], kernels={kern})

    # local_laplacian, every job at an alpha of its own so that tables are built while other calls run
    def ll(name, entry, x, levels, alpha, beta, u8=False, interleaved=False, J=None, kernels=()):
        xv = il if interleaved else None
        scalars = [levels, alpha, beta] if J is None else [J, levels, alpha, beta]
        frames = planar(x) if interleaved else x
        add(name, entry, [In(x, xv)] + scalars + [Out(x.shape, x.dtype, xv)],
            lambda o: [(lambda r: np.ascontiguousarray(np.moveaxis(r, -3, -1)) if interleaved else r)(
                ll_oracle(o, frames, levels, alpha, beta, pyramid_levels=J or 8, u8=u8))],
            kernels=set(kernels))

    ll("ll8", "local_laplacian", u16_frame((3, 83, 127), next(seed)), 8, 0.1431, 1.0,
       kernels={"ll_level1", "ll_coarse_fused", "ll_final2"})
    ll("ll5_beta", "local_laplacian", u16_frame((3, 77, 141), next(seed)), 5, 0.2513, 0.5,
       kernels={"ll_level1_generic", "ll_final"})
    # a level too large for the fused tail gets launches of its own: ll_down_rows / ll_up2 at levels 8 (from level 3),
    # ll_down / ll_up at levels 5 (from level 2)
    ll("ll8_1440p", "local_laplacian", u16_frame((3, 1440, 2560), next(seed)), 8, 0.1419, 1.0,
       kernels={"ll_down_rows", "ll_up2"})
    ll("ll5_1080p", "local_laplacian", u16_frame((3, 1080, 1920), next(seed)), 5, 0.2477, 1.0,
       kernels={"ll_down", "ll_up"})
    ll("ll8_batch", "local_laplacian_batch", u16_frame((3, 3, 97, 131), next(seed)), 8, 0.1437, 1.0)
    ll("ll8_u8", "local_laplacian_u8", u8_frame((3, 89, 117), next(seed)), 8, 0.1423, 1.0, u8=True)
    ll("ll5_u8_batch", "local_laplacian_u8_batch", u8_frame((3, 3, 71, 103), next(seed)), 5, 0.2531, 0.5, u8=True)
    ll("ll8_interleaved", "local_laplacian_interleaved", u16_frame((91, 122, 3), next(seed)), 8, 0.1441, 1.0,
       interleaved=True)
    ll("ll8_interleaved_batch", "local_laplacian_interleaved_batch", u16_frame((3, 63, 86, 3), next(seed)), 8, 0.1447,
       0.5, interleaved=True)
    ll("ll8_u8_interleaved", "local_laplacian_u8_interleaved", u8_frame((79, 134, 3), next(seed)), 8, 0.1411, 1.0,
       u8=True, interleaved=True)
    ll("ll5_u8_interleaved_batch", "local_laplacian_u8_interleaved_batch", u8_frame((3, 58, 93, 3), next(seed)), 5,
       0.2549, 1.0, u8=True, interleaved=True)
    ll("ll_J1", "local_laplacian_pyramid_levels", u16_frame((3, 69, 113), next(seed)), 8, 0.1453, 1.0, J=1,
       kernels={"ll_tone"})
    ll("ll_J2", "local_laplacian_pyramid_levels", u16_frame((3, 74, 109), next(seed)), 8, 0.1459, 1.0, J=2)
    ll("ll_J14", "local_laplacian_pyramid_levels", u16_frame((3, 150, 190), next(seed)), 8, 0.1463, 1.0, J=14)

    # stencil_chain, and 7 stencils (the last launch fuses fewer stages than the others)
    x = u16_frame((90, 140), next(seed))
    add("stencil_chain", "stencil_chain", [In(x), Out(x.shape, np.uint16)], lambda o, x=x: [o.stencil_chain(x)])
    x = u16_frame((101, 77), next(seed))
    add("stencil_chain_7", "stencil_chain_stencils", [In(x), 7, Out(x.shape, np.uint16)],
        lambda o, x=x: [o.stencil_chain(x, stencils=7)])

    # bilateral_grid: bit for bit on dyadic content at s_sigma 8, on any content with the any-S kernels; the 8-bit form's
    # bytes are checked against the float filter's by the baseline (its bins are not exact sums on v / 255)
    x = dyadic((123, 211), next(seed))
    add("bilateral_grid", "bilateral_grid", [In(x), 0.1, Out(x.shape, np.float32)],
        lambda o, x=x: [o.bilateral_grid(x, 0.1)], kernels={"bg_hist_blurz", "bg_blur_xy", "bg_slice"})
    x = f32_frame((97, 143), next(seed))
    add("bilateral_grid_s3", "bilateral_grid_s_sigma", [In(x), 3, 0.1, Out(x.shape, np.float32)],
        lambda o, x=x: [o.bilateral_grid(x, 0.1, s_sigma=3)], kernels={"bg_hist_blurz_s", "bg_slice_s"})
    x = u8_frame((111, 167), next(seed))
    add("bilateral_grid_u8", "bilateral_grid_u8", [In(x), 0.1, Out(x.shape, np.uint8)], None)  # (check_bg_u8)

    # nl_means: the register-window kernel at 3/7, the generic one at 5/9; bit for bit
    x = f32_frame((3, 67, 95), next(seed))
    add("nl_means_3_7", "nl_means", [In(x), 3, 7, 0.12, Out(x.shape, np.float32)],
        lambda o, x=x: [o.nl_means(x, 3, 7, 0.12)], kernels={"nl_means_window"})
    x = f32_frame((3, 59, 83), next(seed))
    add("nl_means_5_9", "nl_means", [In(x), 5, 9, 0.3, Out(x.shape, np.float32)],
        lambda o, x=x: [o.nl_means(x, 5, 9, 0.3)], kernels={"nl_means"})
    x = u8_frame((3, 73, 101), next(seed))
    add("nl_means_u8", "nl_means_u8", [In(x), 3, 7, 0.12, Out(x.shape, np.uint8)],
        lambda o, x=x: [convert(o.nl_means(convert(x, np.float32), 3, 7, 0.12), np.uint8)])

    # camera_pipe: one frame and bursts of 3, planar and interleaved; the matrices are inputs too
    mats = [In(CP_M3200.copy()), In(CP_M7000.copy())]
    for name, entry, (h, w), n, inter in [("camera_pipe", "camera_pipe", (62, 96), 0, False),
                                          ("camera_pipe_batch", "camera_pipe_batch", (54, 72), 3, False),
                                          ("camera_pipe_interleaved", "camera_pipe_interleaved", (66, 88), 0, True),
                                          ("camera_pipe_interleaved_batch", "camera_pipe_interleaved_batch", (50, 80), 3,
                                           True)]:
        s = next(seed)
        raw = raw_frame(h + 30, w + 40, s) if n == 0 else np.stack([raw_frame(h + 30, w + 40, s + k) for k in range(n)])
        frames = [raw] if n == 0 else list(raw)
        out_shape = ((h, w, 3) if inter else (3, h, w)) if n == 0 else ((n, h, w, 3) if inter else (n, 3, h, w))

        def want(o, frames=frames, h=h, w=w, n=n, inter=inter):
            r = [cp_oracle(o, f, (3, h, w)) for f in frames]
            r = [np.ascontiguousarray(f.transpose(1, 2, 0)) if inter else f for f in r]
            return [r[0] if n == 0 else np.stack(r)]
        add(name, entry, [In(raw)] + mats + list(CP) + [Out(out_shape, np.uint8, il if inter else None)], want,
            kernels={"camera_pipe_il" if inter else "camera_pipe", "cp_tables"})

    # conv_layer at its fixed shape, conv_layer_any_shape at a plain shape and at one that folds
    d = conv_exact.harness("rand")
    add("conv_layer", "conv_layer", [In(a) for a in d] + [Out(conv_exact.OUT_SHAPE, np.float32)],
        lambda o, d=d: [o.conv_layer(*d)], rtol=FLOAT_RTOL, kernels={"conv_layer_tc"})
    for shape in [(2, 37, 75, 29, 17), (1, 160, 136, 9, 5)]:
        d = cx.harness("rand", shape)
        add(f"conv_any_{'x'.join(map(str, shape))}", "conv_layer_any_shape",
            [In(a) for a in d] + [Out(cx.shapes_of(shape)[3], np.float32)], lambda o, d=d: [o.conv_layer(*d)],
            rtol=FLOAT_RTOL)
    return jobs


JOBS = make_jobs()
assert len({j.name for j in JOBS}) == len(JOBS)
assert len({j.args[0].array.shape for j in JOBS if j.entry != "conv_layer"}) == len(JOBS) - 1, "one frame size per job"
assert cx.folds(160) > 0 and cx.folds(37) == 0


def run_host(hb, job):
    """The job on numpy host buffers (copied by the runtime, read back with copy_to_host) on the calling thread's stream;
    its buffers are dropped here, on that thread."""
    bufs, outs = [], []
    for a in job.args:
        if isinstance(a, In):
            bufs.append(hb.HalideBuffer.from_numpy(a.view(a.array) if a.view else a.array))
        elif isinstance(a, Out):
            base = np.zeros(a.shape, a.dtype)
            bo = hb.HalideBuffer.from_numpy(a.view(base) if a.view else base, host_dirty=False)
            bufs.append(bo)
            outs.append((base, bo))
        else:
            bufs.append(a)
    getattr(hb.filters, job.entry)(*bufs)
    for _, bo in outs:
        bo.copy_to_host()
    results = [base for base, _ in outs]
    del bufs, outs, bo
    return results


def same_bytes(got, want):
    return got.shape == want.shape and np.array_equal(np.ascontiguousarray(got).view(np.uint8),
                                                      np.ascontiguousarray(want).view(np.uint8))


def launch_names():
    """Every kernel name the library's sources launch under (HB_LAUNCH, and count_launch for the cooperative launch),
    the conv_layer_tc tile variants as one."""
    names = set()
    for path in glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")):
        with open(path) as f:
            for line in f:
                if re.search(r"\bHB_LAUNCH\(|count_launch\(\"", line):
                    names.update(re.findall(r'"([a-z0-9_]+)"', line))
    return {tile_as_one(n) for n in names}


def tile_as_one(name):
    return "conv_layer_tc_n*" if name.startswith("conv_layer_tc_n") else name


# ---- serial baseline --------------------------------------------------------------------------------------------------

def check_bg_u8(hb, oracle, job, got):
    """test_bg_nl_u8_gpu.py's bar: the bytes of to_u8(bilateral_grid(to_f32(x))) on the GPU, and the oracle's composition
    wherever the two float results agree, never more than 1 away elsewhere (bg_hist_blurz's re-association is exact
    only where every partial bin sum is, which v / 255 does not guarantee)."""
    x, r_sigma = job.args[0].array, job.args[1]
    f = run_host(hb, Job("float", "bilateral_grid", [In(convert(x, np.float32)), r_sigma, Out(x.shape, np.float32)],
                         None))[0]
    want_f = oracle.bilateral_grid(convert(x, np.float32), r_sigma)
    want = convert(want_f, np.uint8)
    failures = []
    if not same_bytes(got, convert(f, np.uint8)):
        failures.append(f"{job.name}: differs from to_u8(bilateral_grid(to_f32(x)))")
    if not same_bytes(got[f == want_f], want[f == want_f]) or np.abs(got.astype(np.int16) - want).max() > 1:
        failures.append(f"{job.name}: differs from the oracle's composition")
    return failures


@pytest.fixture(scope="module")
def baseline(hb, oracle):
    """{job name: outputs} of one serial run of every job on the default stream, each checked against the oracle; asserts
    that the jobs together launch every kernel of the library but the self-test."""
    l = hb.load_library()
    l.halide_b200_set_stream(None)
    assert l.halide_b200_ll_last_own_level(2560, 1440, 8) >= 3, "ll8_1440p would not launch ll_down_rows"
    assert l.halide_b200_ll_last_own_level(1920, 1080, 8) >= 2, "ll5_1080p would not launch ll_down"
    results, ran_all, failures = {}, set(), []
    for job in JOBS:
        with kernels_run(hb) as ran:
            got = run_host(hb, job)
        ran_all |= {tile_as_one(k) for k in ran}
        if not job.kernels <= set(ran):
            failures.append(f"{job.name}: launched {sorted(ran)}, missing {sorted(job.kernels - set(ran))}")
        if job.entry == "bilateral_grid_u8":
            failures += check_bg_u8(hb, oracle, job, got[0])
        else:
            for g, w in zip(got, job.want(oracle), strict=True):
                if job.rtol is None:
                    ok = same_bytes(g, w)
                else:
                    ok = np.isfinite(g).all() and (np.abs(g - w) / np.maximum(np.abs(w), 1e-6)).max() <= job.rtol
                if not ok:
                    failures.append(f"{job.name}: differs from the oracle" +
                                    (f" at {int((g != w).sum())} of {g.size} samples" if g.shape == w.shape else ""))
        results[job.name] = got
    assert not failures, "\n".join(failures)
    missing = launch_names() - {"ll_selftest"} - ran_all
    assert not missing, f"kernels no job launched: {sorted(missing)}"
    return results


def test_jobs_cover_every_entry_point():
    from halide_b200 import filters
    public = {n for n, f in inspect.getmembers(filters, inspect.isfunction) if f.__module__ == filters.__name__ and
              not n.startswith("_")}
    assert len(public) == 23 and public == {j.entry for j in JOBS}, sorted(public ^ {j.entry for j in JOBS})


def test_serial_baseline_matches_the_oracle(baseline):
    assert set(baseline) == {j.name for j in JOBS}


# ---- concurrent callers -----------------------------------------------------------------------------------------------

def on_own_streams(hb, n, work):
    """Runs work(i) on n threads, each bound to a stream of its own for the duration; returns the exceptions raised."""
    l = hb.load_library()
    errors = []

    def thread(i):
        s = l.halide_b200_stream_create()
        try:
            assert s, "halide_b200_stream_create failed"
            l.halide_b200_set_stream(s)
            work(i)
        except BaseException as e:
            errors.append(e)
        finally:
            if s:
                l.halide_b200_set_stream(None)
                l.halide_b200_stream_destroy(s)

    threads = [threading.Thread(target=thread, args=(i,)) for i in range(n)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    return errors


def test_concurrent_callers_get_the_serial_bytes(hb, baseline):
    """Four threads, one stream each, every job in an order of the thread's own for three rounds, so that scratch blocks
    recycle through each stream's free list between different entry points while the other threads' calls run."""
    mismatches = []

    def work(i):
        rng = np.random.default_rng(1000 + i)
        for rnd in range(3):
            for k in rng.permutation(len(JOBS)):
                job = JOBS[k]
                got = run_host(hb, job)
                for o, (g, w) in enumerate(zip(got, baseline[job.name], strict=True)):
                    if not same_bytes(g, w):
                        mismatches.append(f"thread {i} round {rnd}: {job.name} output {o}")

    errors = on_own_streams(hb, 4, work)
    assert not errors, errors
    assert not mismatches, "\n".join(mismatches)


# ---- stream ordering --------------------------------------------------------------------------------------------------

SLEEP_CYCLES = 50_000_000  # ~30 ms at the H100's clocks: far longer than the enqueueing of one call


def torch_storage(a):
    """A device tensor holding numpy array a, uint16 stored as int16 (torch has few uint16 kernels)."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()


def sentinel_fill(t):
    import torch
    t.fill_(float("nan") if t.dtype == torch.float32 else (0xA5 if t.dtype == torch.uint8 else 0x5A5A))


def as_filter_type(t, dtype):
    import torch
    return t.view(torch.uint16) if dtype == np.uint16 else t


@pytest.mark.parametrize("job", JOBS, ids=lambda j: j.name)
def test_calls_wait_for_the_callers_stream(hb, baseline, job):
    """On a torch stream passed to the library, enqueued back to back with no host wait: the inputs (the camera_pipe
    matrices and the conv filter and bias included) filled with a sentinel, a sleep, the real inputs copied in, the
    outputs filled with a sentinel, the call, a clone of the outputs.  A copy, launch or table build of the call that did
    not wait for the caller's stream would read sentinel input or have its output overwritten by the sentinel fill."""
    import torch
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    stream = torch.cuda.Stream()
    real = [torch_storage(a.array) for a in job.args if isinstance(a, In)]
    torch.cuda.synchronize()
    try:
        l.halide_b200_set_stream(ctypes.c_void_p(stream.cuda_stream))
        with torch.cuda.stream(stream):
            ins = [torch.empty_like(r) for r in real]
            outs = [torch_storage(np.zeros(a.shape, a.dtype)) for a in job.args if isinstance(a, Out)]
            for t in ins:
                sentinel_fill(t)
            torch.cuda._sleep(SLEEP_CYCLES)
            for t, r in zip(ins, real):
                t.copy_(r)
            for t in outs:
                sentinel_fill(t)
            bufs, it_in, it_out = [], iter(ins), iter(outs)
            for a in job.args:
                if isinstance(a, (In, Out)):
                    t = as_filter_type(next(it_in if isinstance(a, In) else it_out), np.dtype(a.array.dtype if isinstance(a, In) else a.dtype))
                    bufs.append(hb.HalideBuffer.from_torch(a.view(t) if a.view else t))
                else:
                    bufs.append(a)
            getattr(hb.filters, job.entry)(*bufs)
            clones = [t.clone() for t in outs]
        stream.synchronize()
        del bufs
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
    for o, (c, w) in enumerate(zip(clones, baseline[job.name], strict=True)):
        got = c.cpu().numpy().view(w.dtype)
        assert same_bytes(got, w), f"output {o}: {int((got != w).sum())} of {w.size} samples differ from the serial call"


# ---- remap table lifetime ---------------------------------------------------------------------------------------------

def fresh_alphas(n, base):
    """n distinct float32 alphas no other test uses (from base, 2^-20 apart)."""
    return [float(np.float32(base + k * 2.0 ** -20)) for k in range(n)]


def ll_call(hb, x, levels, alpha):
    out = np.zeros_like(x)
    bi, bo = hb.HalideBuffer.from_numpy(x), hb.HalideBuffer.from_numpy(out, host_dirty=False)
    hb.filters.local_laplacian(bi, levels, alpha, 1.0, bo)
    bo.copy_to_host()
    del bi, bo
    return out


def lut_hold(hb, levels, alpha, hold):
    return hb.load_library().halide_b200_ll_lut_hold(ctypes.c_int32(levels), ctypes.c_float(alpha), ctypes.c_int32(hold))


def test_held_table_survives_eviction(hb, oracle):
    """Held, table (8, a0) outlives 70 new alphas (at least one eviction of the 64-table cache) and is reused; dropped, it
    goes at the next eviction, so the cache stays bounded."""
    x = u16_frame((3, 40, 56), 77)
    a0 = float(np.float32(0.3719))
    sweep = fresh_alphas(140, 0.38)
    assert lut_hold(hb, 8, a0, 1) == 0
    try:
        for a in sweep[:70]:
            ll_call(hb, x, 8, a)
        with kernels_run(hb) as ran:
            got = ll_call(hb, x, 8, a0)
        assert "ll_lut" not in ran, sorted(ran)
        assert same_bytes(got, oracle.local_laplacian(x, 8, a0, 1.0))
    finally:
        assert lut_hold(hb, 8, a0, 0) == 0
    assert lut_hold(hb, 8, a0, 0) != 0, "a table that is not held was dropped"
    for a in sweep[70:]:
        ll_call(hb, x, 8, a)
    with kernels_run(hb) as ran:
        again = ll_call(hb, x, 8, a0)
    assert ran.get("ll_lut", (0,))[0] == 1, sorted(ran)
    assert same_bytes(again, got)


def test_threads_sweeping_alphas_get_the_serial_results(hb, oracle):
    """Four threads (one at levels 5), 40 alphas each, interleaved across the threads: 160 tables, more than two
    evictions, built and evicted while the other threads' calls run.  Every result is the serial call's."""
    alphas = fresh_alphas(160, 0.41)
    plan = [(8 if i else 5, u16_frame((3, 48 + 8 * i, 72 + 6 * i), 300 + i), alphas[i::4]) for i in range(4)]
    serial = [[ll_call(hb, x, levels, a) for a in mine] for levels, x, mine in plan]
    for i in (0, 1):
        levels, x, mine = plan[i]
        assert same_bytes(serial[i][0], oracle.local_laplacian(x, levels, mine[0], 1.0))
    mismatches = []

    def work(i):
        levels, x, mine = plan[i]
        for k, a in enumerate(mine):
            if not same_bytes(ll_call(hb, x, levels, a), serial[i][k]):
                mismatches.append(f"thread {i} levels {levels} alpha {a}")

    errors = on_own_streams(hb, 4, work)
    assert not errors, errors
    assert not mismatches, "\n".join(mismatches)
