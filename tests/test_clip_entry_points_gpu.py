"""The clip entry points (halide_b200.blur_video, stencil_chain_video, bilateral_grid_video and nl_means_video) held to
the bar test_concurrent_callers_gpu.py and test_layouts_gpu.py set for the one-frame entry points of
halide_b200.filters:

- CLIP_JOBS: one job per public function of the four modules, each on a frame size of its own, 3 to 5 frames, an odd
  width and an input whose frames (or, for a one-frame interleaved call, whose x / y range) are offset from the
  output's.  heavy_jobs(): clips whose frames run in groups sharing one scratch allocation, or one frame at a time.
- The serial baseline runs every job once on the default stream and checks it frame by frame against the oracle.
- On a torch stream: sentinel input, a sleep, the real input, a sentinel output, the call, a clone, all enqueued before
  one synchronise (and a broadcast input made with expand): the clone must be the baseline's bytes, and the sleep must
  still be running when the call and the clone have been enqueued.
- Four threads, each on its own stream, run the one-frame jobs of test_concurrent_callers_gpu.py and the clip jobs in
  their own order for three rounds: every result must be the serial run's bytes.
- Every clip entry point on padded, flipped, broadcast, row-interleaved (memory [y, n, x]) and, for nl_means,
  line-interleaved or pixel-pitch-4 buffers, on the host and wrapped on the device, inside a sentinel canvas: every
  frame equals the one-frame entry point on a dense copy of its input frame.  An interleaved buffer with a negative or
  zero row or frame stride is refused with -8, and nothing is written."""
import ctypes
import functools
import importlib
import inspect
import time
from dataclasses import dataclass

import numpy as np
import pytest

from bilateral_grid_exact import KERNELS_8, KERNELS_S, dyadic, noise
from halide_b200.image_io import convert
from test_bilateral_grid_batch_gpu import frames_per_group as bg_frames_per_group
from test_blur_stencil_chain_batch_gpu import frames_per_group as sc_frames_per_group
from test_concurrent_callers_gpu import (JOBS, SLEEP_CYCLES, In, Job, Out, as_filter_type, check_bg_u8, fresh_alphas, il,
                                         ll_call, on_own_streams, planar, same_bytes, sentinel_fill, torch_storage,
                                         u8_frame)
from test_layouts_gpu import SENTINEL, Buf, dense_call, layout, same
from util import f32_frame, kernels_run, u16_frame

gpu = pytest.mark.gpu
CLIP_MODULES = ("blur_video", "stencil_chain_video", "bilateral_grid_video", "nl_means_video")
R_FINE = float(np.float32(1.0) / np.float32(128))  # 130 intensity planes: grids large enough to fill the budget
# The delayed-stream sleep: SLEEP_CYCLES lasts 25 ms on an H100 80GB HBM3 (700 W), and a clip call's first device
# allocations on a new stream (its scratch, and the clone's) have taken up to 54 ms of host time there, so the sleep is
# eight times as long, for the call to be enqueued well before it ends.
CLIP_SLEEP_CYCLES = 8 * SLEEP_CYCLES


# ---- jobs -----------------------------------------------------------------------------------------------------------

@dataclass
class ClipIn(In):
    mins: tuple = None  # Halide order (x, y, [c,] n)


@dataclass
class ClipOut(Out):
    mins: tuple = None


@dataclass
class ClipJob(Job):
    first: int = 0        # the index of the input frame output frame 0 reads
    launches: dict = None  # {kernel: launches} the call must make (the heavy jobs)


def call_site(entry):
    """The Python function of a job's entry: "module.function" in halide_b200, or a function of halide_b200.filters."""
    module, _, name = entry.rpartition(".")
    return getattr(importlib.import_module("halide_b200." + (module or "filters")), name)


def per_frame(one, x, out_n, first):
    """want() of a clip job: one(oracle, input frame) for the out_n input frames from index `first`, stacked."""
    return lambda o: [np.stack([one(o, x[first + k]) for k in range(out_n)])]


def hwc(r):
    """A planar (3, h, w) result as the (h, w, 3) frame of an interleaved output array."""
    return np.ascontiguousarray(np.moveaxis(r, 0, -1))


def nl_u8(o, f, p, s, sigma, *shape_mins):
    """nl_means_u8's composition on a planar uint8 frame: to_u8(nl_means(to_f32(f)))."""
    return convert(o.nl_means(convert(f, np.float32), p, s, sigma, *shape_mins), np.uint8)


def make_clip_jobs():
    jobs = []
    seed = iter(range(2000, 3000))

    def add(name, entry, x, scalars, out_shape, want, in_mins=None, out_mins=None, view=None, first=0, kernels=()):
        jobs.append(ClipJob(name, entry, [ClipIn(x, view, in_mins)] + list(scalars) +
                            [ClipOut(out_shape, x.dtype, view, out_mins)], want, kernels=set(kernels), first=first))

    # blur: input frames [-1, 4), output frames [0, 4) at x / y mins (-3, 5)
    x = u16_frame((5, 45, 79), next(seed))
    add("blur_batch", "blur_video.blur_batch", x, [], (4, 43, 77),
        per_frame(lambda o, f: o.blur(f, (43, 77), (-3, 5), (-3, 5)), x, 4, 1), (-3, 5, -1), (-3, 5, 0), first=1)

    # stencil_chain: 32 stages at mins that make repeat_edge reach past the input; 13 stages (4 launches, 2 planes)
    x = u16_frame((4, 53, 75), next(seed))
    add("stencil_chain_batch", "stencil_chain_video.stencil_chain_batch", x, [], (3, 51, 73),
        per_frame(lambda o, f: o.stencil_chain(f, (51, 73), (4, -7), (1, -9)), x, 3, 1), (4, -7, 1), (1, -9, 2),
        first=1, kernels={"stencil_chain_window"})
    x = u16_frame((5, 57, 91), next(seed))
    add("stencil_chain_stencils_batch", "stencil_chain_video.stencil_chain_stencils_batch", x, [13], (4, 57, 91),
        per_frame(lambda o, f: o.stencil_chain(f, stencils=13), x, 4, 1), (0, 0, -1), first=1,
        kernels={"stencil_chain_window"})

    # bilateral_grid: bit for bit on dyadic content at S = 8, on any content at S = 5; the 8-bit form per frame by
    # check_bg_u8
    x = np.stack([dyadic((63, 109), next(seed)) for _ in range(4)])
    add("bilateral_grid_batch", "bilateral_grid_video.bilateral_grid_batch", x, [0.1], (3, 63, 109),
        per_frame(lambda o, f: o.bilateral_grid(f, 0.1), x, 3, 1), None, (0, 0, 1), first=1, kernels=KERNELS_8)
    x = noise((5, 71, 93), next(seed))
    add("bilateral_grid_s_sigma_batch", "bilateral_grid_video.bilateral_grid_s_sigma_batch", x, [5, 0.1], (3, 71, 93),
        per_frame(lambda o, f: o.bilateral_grid(f, 0.1, s_sigma=5), x, 3, 2), (0, 0, 3), (0, 0, 5), first=2,
        kernels=KERNELS_S)
    x = u8_frame((4, 67, 121), next(seed))
    add("bilateral_grid_u8_batch", "bilateral_grid_video.bilateral_grid_u8_batch", x, [0.1], (3, 67, 121), None,
        None, (0, 0, 1), first=1, kernels=KERNELS_8)

    # nl_means: the register-window kernel at 3/7, the generic one at 5/9, float and 8-bit, planar and interleaved;
    # the one-frame interleaved calls read an RGBA input (its alpha is never read) and a crop of it or of their output
    x = f32_frame((5, 3, 39, 61), next(seed))
    add("nl_means_batch", "nl_means_video.nl_means_batch", x, [3, 7, 0.12], (4, 3, 39, 61),
        per_frame(lambda o, f: o.nl_means(f, 3, 7, 0.12), x, 4, 1), (0, 0, 0, -1), first=1, kernels={"nl_means_window"})
    x = u8_frame((4, 3, 35, 67), next(seed))
    add("nl_means_u8_batch", "nl_means_video.nl_means_u8_batch", x, [5, 9, 0.3], (3, 3, 35, 67),
        per_frame(lambda o, f: nl_u8(o, f, 5, 9, 0.3), x, 3, 1), (0, 0, 0, 2), (0, 0, 0, 3), first=1,
        kernels={"nl_means"})
    x = f32_frame((53, 87, 4), next(seed))
    add("nl_means_interleaved", "nl_means_video.nl_means_interleaved", x, [3, 7, 0.12], (47, 81, 3),
        lambda o, x=x: [hwc(o.nl_means(planar(x)[:3], 3, 7, 0.12, (3, 47, 81), (-2, -3, 0)))], (-2, -3, 0), view=il,
        kernels={"nl_means_window"})
    x = f32_frame((4, 33, 59, 3), next(seed))
    add("nl_means_interleaved_batch", "nl_means_video.nl_means_interleaved_batch", x, [5, 9, 0.3], (3, 33, 59, 3),
        per_frame(lambda o, f: hwc(o.nl_means(planar(f), 5, 9, 0.3)), x, 3, 1), (0, 0, 0, -1), view=il, first=1,
        kernels={"nl_means"})
    x = u8_frame((41, 73, 4), next(seed))
    add("nl_means_u8_interleaved", "nl_means_video.nl_means_u8_interleaved", x, [5, 9, 0.3], (37, 69, 3),
        lambda o, x=x: [hwc(nl_u8(o, planar(x)[:3], 5, 9, 0.3, (3, 37, 69), None, (2, 2, 0)))], None, (2, 2, 0),
        view=il, kernels={"nl_means"})
    x = u8_frame((5, 29, 55, 3), next(seed))
    add("nl_means_u8_interleaved_batch", "nl_means_video.nl_means_u8_interleaved_batch", x, [3, 7, 0.12],
        (4, 29, 55, 3), per_frame(lambda o, f: hwc(nl_u8(o, planar(f), 3, 7, 0.12)), x, 4, 1), (0, 0, 0, 0),
        (0, 0, 0, 1), view=il, first=1, kernels={"nl_means_window"})
    return jobs


@functools.cache
def heavy_jobs():
    """Clips whose frames do not fit one group: built on first use (about 230 MB of frames)."""
    jobs = []
    # stencil_chain at S = 9 (3 launches, 2 scratch planes): 7 frames a group, 8 frames run as 2 groups on one allocation
    h, w, n, s = 2161, 3839, 8, 9
    g = sc_frames_per_group(h, w, n, s)
    assert 1 < g < n, g
    x = u16_frame((n + 1, h, w), 4001)
    jobs.append(ClipJob("stencil_chain_groups", "stencil_chain_video.stencil_chain_stencils_batch",
                        [ClipIn(x, None, (0, 0, -1)), s, ClipOut((n, h, w), np.uint16)],
                        per_frame(lambda o, f, s=s: o.stencil_chain(f, stencils=s), x, n, 1), first=1,
                        launches={"stencil_chain_window": -(-s // 4) * -(-n // g)}))
    # bilateral_grid at S = 9 and 130 intensity planes: 4 frames a group, 5 frames run as 2 groups on one pair of grids
    h, w, n, s = 1079, 1921, 5, 9
    g = bg_frames_per_group(h, w, n, R_FINE, s)
    assert 1 < g < n, g
    x = noise((n + 1, h, w), 4002)
    jobs.append(ClipJob("bilateral_grid_groups", "bilateral_grid_video.bilateral_grid_s_sigma_batch",
                        [ClipIn(x, None, (0, 0, -1)), s, R_FINE, ClipOut((n, h, w), np.float32)],
                        per_frame(lambda o, f, s=s: o.bilateral_grid(f, R_FINE, s_sigma=s), x, n, 1), first=1,
                        launches={k: -(-n // g) for k in KERNELS_S}))
    # bilateral_grid at S = 6: fewer than kMinGroup frames fit the budget, so the 3 frames run one at a time
    h, w, n, s = 1081, 1917, 3, 6
    assert bg_frames_per_group(h, w, n, R_FINE, s) == 1
    x = noise((n + 1, h, w), 4003)
    jobs.append(ClipJob("bilateral_grid_one_by_one", "bilateral_grid_video.bilateral_grid_s_sigma_batch",
                        [ClipIn(x, None, (0, 0, -1)), s, R_FINE, ClipOut((n, h, w), np.float32)],
                        per_frame(lambda o, f, s=s: o.bilateral_grid(f, R_FINE, s_sigma=s), x, n, 1), first=1,
                        launches={k: n for k in KERNELS_S}))
    return jobs


HEAVY = ["stencil_chain_groups", "bilateral_grid_groups", "bilateral_grid_one_by_one"]
CLIP_JOBS = make_clip_jobs()


def frame_sizes(job):
    """Every (h, w) a job's arrays could be read as: each pair of adjacent axes of its inputs and outputs."""
    shapes = [a.array.shape for a in job.args if isinstance(a, In)] + [a.shape for a in job.args if isinstance(a, Out)]
    return {s[i:i + 2] for s in shapes for i in range(len(s) - 1)}


def out_frame_size(job):
    out = next(a for a in job.args if isinstance(a, Out))
    return out.shape[-3:-1] if out.view is il else out.shape[-2:]


assert len({j.name for j in CLIP_JOBS} | {j.name for j in JOBS}) == len(CLIP_JOBS) + len(JOBS)
assert len({out_frame_size(j) for j in CLIP_JOBS}) == len(CLIP_JOBS), "one frame size per clip job"
assert not {out_frame_size(j) for j in CLIP_JOBS} & set().union(*map(frame_sizes, JOBS)), "a frame size of JOBS"
assert all(out_frame_size(j)[1] % 2 for j in CLIP_JOBS), "an odd width per clip job"


def heavy(name):
    return next(j for j in heavy_jobs() if j.name == name)


def run_host(hb, job):
    """The job on numpy host buffers at its mins (copied by the runtime, read back with copy_to_host) on the calling
    thread's stream; a job of test_concurrent_callers_gpu.py runs as it does there."""
    bufs, outs = [], []
    for a in job.args:
        if isinstance(a, In):
            bufs.append(hb.HalideBuffer.from_numpy(a.view(a.array) if a.view else a.array, getattr(a, "mins", None)))
        elif isinstance(a, Out):
            base = np.zeros(a.shape, a.dtype)
            bo = hb.HalideBuffer.from_numpy(a.view(base) if a.view else base, getattr(a, "mins", None), host_dirty=False)
            bufs.append(bo)
            outs.append((base, bo))
        else:
            bufs.append(a)
    call_site(job.entry)(*bufs)
    for _, bo in outs:
        bo.copy_to_host()
    results = [base for base, _ in outs]
    del bufs, outs, bo
    return results


def test_clip_jobs_cover_every_clip_entry_point():
    """Every public function of the four clip modules is a job here, so a new clip entry point has to join."""
    public = set()
    for m in CLIP_MODULES:
        mod = importlib.import_module("halide_b200." + m)
        public |= {f"{m}.{n}" for n, f in inspect.getmembers(mod, inspect.isfunction)
                   if f.__module__ == mod.__name__ and not n.startswith("_")}
    assert len(public) == 12 and public == {j.entry for j in CLIP_JOBS}, sorted(public ^ {j.entry for j in CLIP_JOBS})


# ---- serial baseline --------------------------------------------------------------------------------------------------

def check_against_oracle(hb, oracle, job, got):
    """Failures of a clip job's outputs against the oracle: bit for bit, the 8-bit bilateral_grid frame by frame at
    check_bg_u8's bar."""
    if job.want is None:
        x, r_sigma = job.args[0].array, job.args[1]
        failures = []
        for k, g in enumerate(got[0]):
            f = x[job.first + k]
            failures += check_bg_u8(hb, oracle, Job(f"{job.name} frame {k}", "bilateral_grid_u8",
                                                    [In(f), r_sigma, Out(f.shape, np.uint8)], None), g)
        return failures
    failures = []
    for g, w in zip(got, job.want(oracle), strict=True):
        if not same_bytes(g, w):
            failures.append(f"{job.name}: differs from the oracle" +
                            (f" at {int((g != w).sum())} of {g.size} samples" if g.shape == w.shape else ""))
    return failures


@pytest.fixture(scope="module")
def baseline(hb, oracle):
    """{job name: outputs} of one serial run of every clip job, the heavy ones included, on the default stream, each
    checked against the oracle and for the kernels (heavy: the launch counts) its path must take."""
    hb.load_library().halide_b200_set_stream(None)
    results, failures = {}, []
    for job in CLIP_JOBS + heavy_jobs():
        with kernels_run(hb) as ran:
            got = run_host(hb, job)
        if not job.kernels <= set(ran):
            failures.append(f"{job.name}: launched {sorted(ran)}, missing {sorted(job.kernels - set(ran))}")
        if job.launches is not None and {k: c for k, (c, _) in ran.items()} != job.launches:
            failures.append(f"{job.name}: launched {ran}, want {job.launches}")
        failures += check_against_oracle(hb, oracle, job, got)
        results[job.name] = got
    assert not failures, "\n".join(failures)
    return results


@pytest.fixture(scope="module")
def frame_baseline(hb):
    """{job name: outputs} of one serial run of every job of test_concurrent_callers_gpu.py (that file checks them
    against the oracle).  On teardown the remap tables of their alphas are evicted (65 calls at new alphas: the library
    drops every unheld table once 64 are cached), so that a later module's calls at those alphas build their own, as
    that file's baseline asserts."""
    hb.load_library().halide_b200_set_stream(None)
    yield {job.name: run_host(hb, job) for job in JOBS}
    x = u16_frame((3, 16, 24), 47)
    for a in fresh_alphas(65, 0.47):
        ll_call(hb, x, 8, a)


@gpu
def test_serial_baseline_matches_the_oracle(baseline):
    assert set(baseline) == {j.name for j in CLIP_JOBS} | set(HEAVY)


# ---- stream ordering --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def sleep_ms(hb):
    """What torch.cuda._sleep(CLIP_SLEEP_CYCLES) lasts on this GPU, in ms (CUDA events; the second of two runs)."""
    import torch
    for _ in range(2):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        torch.cuda._sleep(CLIP_SLEEP_CYCLES)
        end.record()
        end.synchronize()
    return start.elapsed_time(end)


def broadcast(job):
    """The job with its input one frame (the frame output frame 0 reads) expanded over all of the input's frames (a
    frame stride of 0, as torch's expand and numpy's broadcast_to make)."""
    a = job.args[0]
    n = a.array.shape[0]

    def view(t):
        v = t.expand(n, *t.shape[1:]) if hasattr(t, "expand") else np.broadcast_to(t, (n,) + t.shape[1:])
        return a.view(v) if a.view else v
    one = a.array[job.first:job.first + 1]
    return ClipJob(job.name + "_bcast", job.entry, [ClipIn(one, view, a.mins)] + job.args[1:], None, first=0)


def delayed_call(hb, job):
    """test_concurrent_callers_gpu.py's test_calls_wait_for_the_callers_stream on the job's inputs as torch device
    tensors at the job's mins, with a sleep of CLIP_SLEEP_CYCLES: (the clones of the outputs, the host seconds from the
    call to the clones, whether the sleep was still running when the clones were enqueued)."""
    import torch
    l = hb.load_library()
    prev = l.halide_b200_get_stream()
    stream = torch.cuda.Stream()
    real = [torch_storage(a.array) for a in job.args if isinstance(a, In)]
    # (device blocks cached by earlier calls, the library's and torch's, released first: an allocation that found the
    # device full would release them itself, with a device-wide synchronise that waits out the sleep)
    hb.capi.halide_cuda_release_unused_device_allocations(None)
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    try:
        l.halide_b200_set_stream(ctypes.c_void_p(stream.cuda_stream))
        with torch.cuda.stream(stream):
            ins = [torch.empty_like(r) for r in real]
            outs = [torch_storage(np.zeros(a.shape, a.dtype)) for a in job.args if isinstance(a, Out)]
            for t in ins:
                sentinel_fill(t)
            torch.cuda._sleep(CLIP_SLEEP_CYCLES)
            slept = torch.cuda.Event()
            slept.record(stream)
            for t, r in zip(ins, real):
                t.copy_(r)
            for t in outs:
                sentinel_fill(t)
            bufs, it_in, it_out = [], iter(ins), iter(outs)
            for a in job.args:
                if isinstance(a, (In, Out)):
                    is_in = isinstance(a, In)
                    t = as_filter_type(next(it_in if is_in else it_out), np.dtype(a.array.dtype if is_in else a.dtype))
                    bufs.append(hb.HalideBuffer.from_torch(a.view(t) if a.view else t, a.mins))
                else:
                    bufs.append(a)
            t0 = time.perf_counter()
            call_site(job.entry)(*bufs)
            clones = [t.clone() for t in outs]
            enqueue = time.perf_counter() - t0
            sleeping = not slept.query()
        stream.synchronize()
        del bufs
    finally:
        l.halide_b200_set_stream(ctypes.c_void_p(prev))
    dtypes = [np.dtype(a.dtype) for a in job.args if isinstance(a, Out)]
    return [c.cpu().numpy().view(d) for c, d in zip(clones, dtypes)], enqueue, sleeping


def check_delayed(hb, job, want, sleep_ms):
    got, enqueue, sleeping = delayed_call(hb, job)
    for o, (g, w) in enumerate(zip(got, want, strict=True)):
        assert same_bytes(g, w), f"output {o}: {int((g != w).sum())} of {w.size} samples differ from the serial call"
    # (a call enqueued only once the sleep had ended would pass whether or not it waits for the caller's stream)
    assert sleeping, f"the sleep ({sleep_ms:.1f} ms) had ended when the call was enqueued ({enqueue * 1e3:.1f} ms)"


@gpu
@pytest.mark.parametrize("name", [j.name for j in CLIP_JOBS] + HEAVY)
def test_calls_wait_for_the_callers_stream(hb, baseline, sleep_ms, name):
    """A copy, launch or scratch reuse of the call that did not wait for the caller's stream would read sentinel input
    or have its output overwritten by the sentinel fill.  The heavy jobs reuse one scratch allocation across groups or
    frames within the call."""
    job = next((j for j in CLIP_JOBS if j.name == name), None) or heavy(name)
    check_delayed(hb, job, baseline[name], sleep_ms)


@gpu
@pytest.mark.parametrize("name", [j.name for j in CLIP_JOBS if j.entry.endswith("_batch") and j.args[0].view is None])
def test_broadcast_clips_wait_for_the_callers_stream(hb, sleep_ms, name):
    """The planar clip jobs, on one input frame expanded over the input's frames: every output frame is the same, and
    the delayed call gives the serial call's bytes.  (An interleaved clip's frame stride must be positive.)"""
    job = broadcast(next(j for j in CLIP_JOBS if j.name == name))
    hb.load_library().halide_b200_set_stream(None)
    want = run_host(hb, job)
    assert all(same_bytes(f, want[0][0]) for f in want[0]), "the frames of a broadcast clip differ"
    check_delayed(hb, job, want, sleep_ms)


# ---- concurrent callers -----------------------------------------------------------------------------------------------

@gpu
def test_concurrent_callers_get_the_serial_bytes(hb, baseline, frame_baseline):
    """Four threads, one stream each, every one-frame and clip job in an order of the thread's own for three rounds, so
    that the clip calls' scratch blocks recycle through each stream's free list between the other entry points' while
    the other threads' calls run."""
    jobs = JOBS + CLIP_JOBS
    want = {**frame_baseline, **baseline}
    mismatches = []

    def work(i):
        rng = np.random.default_rng(3000 + i)
        for rnd in range(3):
            for k in rng.permutation(len(jobs)):
                job = jobs[k]
                for o, (g, w) in enumerate(zip(run_host(hb, job), want[job.name], strict=True)):
                    if not same_bytes(g, w):
                        mismatches.append(f"thread {i} round {rnd}: {job.name} output {o}")

    errors = on_own_streams(hb, 4, work)
    assert not errors, errors
    assert not mismatches, "\n".join(mismatches)


# ---- stride layouts ---------------------------------------------------------------------------------------------------

class Lay:
    """A layout of this file's own for test_layouts_gpu.layout: the logical axes in memory order (outermost first),
    `pad` extra samples on memory axes, logical axes flipped, and a logical axis broadcast."""

    def __init__(self, name, order, pad=None, flip=(), bcast=None):
        self.name, self.order, self.pad, self.flip, self.bcast = name, order, pad or {}, flip, bcast

    def __repr__(self):
        return self.name

    def __call__(self, shape):
        extent = [1 if a == self.bcast else shape[a] for a in self.order]
        mshape = tuple(e + self.pad.get(i, 0) for i, e in enumerate(extent))
        back = tuple(np.argsort(self.order))

        def view_of(m):
            v = m[tuple(slice(0, e) for e in extent)].transpose(back)
            for a in self.flip:
                v = np.flip(v, a)
            return v, (v if self.bcast is None else np.broadcast_to(v, shape))
        return mshape, view_of


def rows_n(nd):
    """Row-interleaved frames: memory [y, n, x] ([c, y, n, x] for a planar 4-D clip), frame stride = the row pitch, row
    stride = N x pitch."""
    return Lay("rows_n", (1, 0, 2) if nd == 3 else (1, 2, 0, 3))


def interleaved(name, nd):
    """A pixel-interleaved layout of a planar ([n,] c, y, x) clip: memory [n, y, x, c] (il), rows padded by a pixel
    (il_pad), a pixel pitch of 4 with rows padded (il4_pad) or flipped (il4_flip_y), flipped or broadcast frames
    (il_flip_n, il_bcast_n), or row-interleaved frames, memory [y, n, x, c] (il_rows_n)."""
    o = (0, 2, 3, 1) if nd == 4 else (1, 2, 0)
    return {"il": Lay(name, o), "il_pad": Lay(name, o, {nd - 2: 1}), "il4_pad": Lay(name, o, {nd - 2: 1, nd - 1: 1}),
            "il4_flip_y": Lay(name, o, {nd - 1: 1}, (nd - 2,)),
            "il_flip_n": Lay(name, o, flip=(0,)), "il_bcast_n": Lay(name, o, bcast=0),
            "il_rows_n": Lay(name, (2, 0, 3, 1))}[name]


def lay_of(name, nd):
    """A layout name of this section as test_layouts_gpu.layout takes it, for a clip of nd logical axes."""
    if name.startswith("il"):
        return interleaved(name, nd)
    if name == "rows_n":
        return rows_n(nd)
    return {"flip_n": ("flip", -nd), "bcast_n": ("bcast", -nd)}.get(name, name)


@dataclass
class Spec:
    """A clip entry point on a small clip: its one-frame counterpart of halide_b200.filters (planar), the logical
    (planar) input and output shapes, the layouts of each side, the oracle on one planar frame, and `oracle_pair`,
    the layouts also compared with the oracle."""
    entry: str
    one: str
    in_shape: tuple
    out_shape: tuple
    dtype: object
    scalars: tuple
    in_lays: list
    out_lays: list
    oracle: object
    oracle_pair: tuple
    data: object = None
    seed: int = 0


N3, H3, W3 = 3, 37, 53
U16 = ["pad", "flip_y", "flip_y_odd", "flip_n", "rows_n"]
F32 = ["pad", "flip_y", "flip_n", "rows_n"]
IL_BATCH = ["il", "il_pad", "il4_pad", "il_rows_n", "il4_flip_y", "il_flip_n"]
IL_ONE = ["il_pad", "il4_pad", "il4_flip_y"]
# An interleaved buffer's row and frame strides must be positive (filters._INTERLEAVED_LAYOUT): these are refused with
# -8, before anything is written.
REFUSED = {"il4_flip_y", "il_flip_n", "il_bcast_n"}


def make_specs():
    c3, c4 = (N3, H3, W3), (N3, 3, H3, W3)
    u8 = lambda shape, seed: u8_frame(shape, seed)  # noqa: E731
    specs = {
        "blur_batch": Spec("blur_video.blur_batch", "halide_blur", (N3, H3 + 2, 56), (N3, H3, 54), np.uint16, (),
                           U16 + ["bcast_n"], U16, lambda o, f: o.blur(f), ("rows_n", "dense"), u16_frame),
        "stencil_chain_batch": Spec("stencil_chain_video.stencil_chain_batch", "stencil_chain", c3, c3, np.uint16, (),
                                    U16 + ["bcast_n"], U16, lambda o, f: o.stencil_chain(f), ("dense", "rows_n"),
                                    u16_frame),
        "stencil_chain_stencils_batch": Spec("stencil_chain_video.stencil_chain_stencils_batch",
                                             "stencil_chain_stencils", c3, c3, np.uint16, (5,), U16 + ["bcast_n"], U16,
                                             lambda o, f: o.stencil_chain(f, stencils=5), ("rows_n", "flip_y_odd"),
                                             u16_frame),
        "bilateral_grid_batch": Spec("bilateral_grid_video.bilateral_grid_batch", "bilateral_grid", c3, c3, np.float32,
                                     (0.1,), F32 + ["bcast_n"], F32, lambda o, f: o.bilateral_grid(f, 0.1),
                                     ("rows_n", "dense"), dyadic),
        "bilateral_grid_s_sigma_batch": Spec("bilateral_grid_video.bilateral_grid_s_sigma_batch",
                                             "bilateral_grid_s_sigma", c3, c3, np.float32, (3, 0.1), F32 + ["bcast_n"],
                                             F32, lambda o, f: o.bilateral_grid(f, 0.1, s_sigma=3), ("dense", "rows_n"),
                                             noise),
        "bilateral_grid_u8_batch": Spec("bilateral_grid_video.bilateral_grid_u8_batch", "bilateral_grid_u8", c3, c3,
                                        np.uint8, (0.1,), F32 + ["bcast_n"], F32, None, ("rows_n", "flip_n"), u8),
        "nl_means_batch": Spec("nl_means_video.nl_means_batch", "nl_means", c4, c4, np.float32, (3, 7, 0.12),
                               F32 + ["xcy", "bcast_n"], F32 + ["xcy"], lambda o, f: o.nl_means(f, 3, 7, 0.12),
                               ("xcy", "rows_n"), f32_frame),
        "nl_means_u8_batch": Spec("nl_means_video.nl_means_u8_batch", "nl_means_u8", c4, c4, np.uint8, (5, 9, 0.3),
                                  F32 + ["xcy", "bcast_n"], F32 + ["xcy"], lambda o, f: nl_u8(o, f, 5, 9, 0.3),
                                  ("rows_n", "xcy"), u8),
        "nl_means_interleaved_batch": Spec("nl_means_video.nl_means_interleaved_batch", "nl_means", c4, c4, np.float32,
                                           (5, 9, 0.3), IL_BATCH + ["il_bcast_n"], IL_BATCH,
                                           lambda o, f: o.nl_means(f, 5, 9, 0.3), ("il_rows_n", "il4_pad"),
                                           f32_frame),
        "nl_means_u8_interleaved_batch": Spec("nl_means_video.nl_means_u8_interleaved_batch", "nl_means_u8", c4, c4,
                                              np.uint8, (3, 7, 0.12), IL_BATCH + ["il_bcast_n"], IL_BATCH,
                                              lambda o, f: nl_u8(o, f, 3, 7, 0.12), ("il4_pad", "il_rows_n"), u8),
        "nl_means_interleaved": Spec("nl_means_video.nl_means_interleaved", "nl_means", c4[1:], c4[1:], np.float32,
                                     (3, 7, 0.12), IL_ONE, IL_ONE, lambda o, f: o.nl_means(f, 3, 7, 0.12),
                                     ("il4_pad", "il4_pad"), f32_frame),
        "nl_means_u8_interleaved": Spec("nl_means_video.nl_means_u8_interleaved", "nl_means_u8", c4[1:], c4[1:],
                                        np.uint8, (5, 9, 0.3), IL_ONE, IL_ONE, lambda o, f: nl_u8(o, f, 5, 9, 0.3),
                                        ("il_pad", "il4_pad"), u8),
    }
    for k, (name, s) in enumerate(specs.items()):
        assert s.entry.endswith("." + name)
        s.seed = 5000 + k
    return specs


SPECS = make_specs()
assert {s.entry for s in SPECS.values()} == {j.entry for j in CLIP_JOBS}


def layout_cases():
    """Each input layout with a dense (il: pitch 3) output, each output layout with a dense input, and every oracle pair."""
    cases = []
    for name, s in SPECS.items():
        d = "il" if s.in_lays[0].startswith("il") else "dense"
        pairs = [(l, d) for l in s.in_lays] + [(d, l) for l in s.out_lays if l != d] + [s.oracle_pair]
        cases += [(name, i, o) for i, o in dict.fromkeys(pairs)]
    return cases


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def blur_pair_ok(bi, bo):
    """blur.cu: both bases 4-byte aligned and every row and frame stride even -> the pair kernel (input and output at
    mins 0, so the input's first read is its element at the mins)."""
    return (((bi.buf.buf.device | bo.buf.buf.device) & 3) == 0 and
            all(s % 2 == 0 for s in bi.strides()[1:3] + bo.strides()[1:3]))


@gpu
@pytest.mark.parametrize("variant", ["host", "device"])
@pytest.mark.parametrize("name,in_lay,out_lay", layout_cases())
def test_clip_layouts(hb, oracle, name, in_lay, out_lay, variant):
    """The clip entry point on its input in `in_lay` into an output in `out_lay` inside a sentinel canvas (Buf.read: the
    bytes outside the output's view, an RGBA output's alpha among them, keep the sentinel); every frame against the
    one-frame entry point on a dense copy of its input frame, and against the oracle on the spec's oracle pair."""
    s = SPECS[name]
    nd = len(s.in_shape)
    data = s.data(s.in_shape, s.seed)
    bi = Buf(hb, s.in_shape, s.dtype, lay_of(in_lay, nd), variant, data=data)
    bo = Buf(hb, s.out_shape, s.dtype, lay_of(out_lay, nd), variant)
    if {in_lay, out_lay} & REFUSED:
        with pytest.raises(hb.HalideError, match="for an interleaved buffer") as e:
            call_site(s.entry)(bi.buf, *s.scalars, bo.buf)
        assert e.value.code == -8
        mem = bo.mem if variant == "host" else bo.t.cpu().numpy()
        assert (mem.view(np.uint8) == SENTINEL).all(), "a refused call wrote its output"
        return
    with kernels_run(hb) as ran:
        call_site(s.entry)(bi.buf, *s.scalars, bo.buf)
        got = bo.read()
    logical = bi.logical
    batch = s.entry.endswith("_batch")
    frames, outs = (logical, got) if batch else (logical[None], got[None])
    one = call_site(s.one)
    for k, (f, g) in enumerate(zip(frames, outs, strict=True)):
        want = dense_call(hb, lambda b_in, b_out: one(b_in, *s.scalars, b_out), [f], g.shape, s.dtype)
        same(bits(g), bits(want), f"{in_lay} -> {out_lay} ({variant}) frame {k}: against the one-frame entry point")
    if (in_lay, out_lay) == s.oracle_pair:
        for k, (f, g) in enumerate(zip(frames, outs)):
            if s.oracle is None:
                job = Job(f"{name} frame {k}", "bilateral_grid_u8", [In(f), s.scalars[0], Out(f.shape, np.uint8)], None)
                failures = check_bg_u8(hb, oracle, job, g)
                assert not failures, failures
            else:
                same(bits(g), bits(s.oracle(oracle, f)), f"{in_lay} -> {out_lay} frame {k}: against the oracle")
    if name == "blur_batch":
        pair = blur_pair_ok(bi, bo)
        assert set(ran) == {"blur3x3_u16_quad" if pair else "blur3x3_u16"}, (sorted(ran), bi.strides(), bo.strides())
        if variant == "device":  # (aligned bases; every pitch and frame stride even but flip_y_odd's)
            assert pair == ("flip_y_odd" not in (in_lay, out_lay)), (in_lay, out_lay)


def test_same_reports_swapped_frames():
    """same() reports a clip whose frames n and n + 1 are swapped, on synthetic arrays."""
    want = np.arange(4 * 5 * 7, dtype=np.uint16).reshape(4, 5, 7)
    got = want[[0, 2, 1, 3]]
    with pytest.raises(AssertionError, match=r"70 of 140 samples differ, first at .*: got 70 want 35"):
        same(got, want, "swapped frames")
    same(want.copy(), want, "equal")
