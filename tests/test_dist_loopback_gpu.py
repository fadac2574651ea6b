"""The row-sharded local_laplacian on ONE GPU: `world` host threads each join an in-process loopback group
(halide_b200_dist_init_loopback) and call halide_b200_local_laplacian_sharded on their band of the frame.  Every line
of the sharded path runs — band all-gather, input-halo exchange, levels 1-2 split into an interior launch and two edge
launches, the gathered level — and so do the kernels' halo-row addressing.  The bands put together must equal the
single-GPU filter on the whole frame bit for bit.  (The NCCL transport across devices is test_dist_gpu.py's.)

The rank threads stay on the library's default stream, the legacy stream that all threads share: the ranks' kernels
never run at the same time, and the cooperative coarse launch is never co-scheduled with another rank's kernel.
Rank r always runs on the same thread, which keeps its own halo stream and band plan from call to call."""
import concurrent.futures
import ctypes
import os
import subprocess
import sys
from contextlib import contextmanager

import numpy as np
import pytest

from test_local_laplacian_gpu import _region_vs_oracle
from util import run_local_laplacian, u16_frame

pytestmark = pytest.mark.gpu
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
LEVELS, ALPHA = 8, 1.0 / 7.0
GENERIC_ERROR, CONSTRAINT_VIOLATED = -1, -8   # halide_error_code_t
# one thread per rank for the whole module: a rank thread's halo stream and events live as long as the thread
_RANK_THREADS = [concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix=f"rank{r}") for r in range(8)]

# Per rank count: a frame whose rows do not divide by the rank count and whose odd width makes the halo rows' pitch
# odd (the level-1 kernel's unaligned path), and one whose rows divide and are 16-byte multiples (the final kernel's
# TMA path on every band).  Both are tall enough for every gathered level 2..7.
FRAMES = {2: [(3, 517, 333), (3, 640, 256)], 3: [(3, 601, 333), (3, 768, 200)], 4: [(3, 902, 261), (3, 1024, 200)],
          8: [(3, 1931, 203), (3, 2048, 136)]}


def _lib():
    import halide_b200
    return halide_b200.load_library()


def _band_rows(rank, world, h):
    from halide_b200.dist import band_rows
    return band_rows(rank, world, h)


def _rank_main(rank, world, jobs, beta, x0):
    """One rank: join the group, run `calls` sharded calls on its band of each (frame, calls) job, leave.  Returns
    (return code, error message, [output band of every call])."""
    import halide_b200
    from halide_b200 import HalideBuffer
    l = _lib()
    rc = l.halide_b200_dist_init_loopback(rank, world)
    if rc:
        return rc, halide_b200.lib.last_error_message(), []
    outs = []
    try:
        for img, calls in jobs:
            h = img.shape[1]
            lo, hi = _band_rows(rank, world, h)
            bi = HalideBuffer.from_numpy(np.ascontiguousarray(img[:, lo:hi + 1, :]), (x0, lo, 0))
            for _ in range(calls):  # (the input stays on the device from the first call on)
                # the output's device copy starts as a pattern the filter must overwrite everywhere
                out = np.full((img.shape[0], hi - lo + 1, img.shape[2]), 0xA5A5, np.uint16)
                bo = HalideBuffer.from_numpy(out, (x0, lo, 0))
                halide_b200.lib.check(l.halide_copy_to_device(None, bo.ptr, None))
                rc = l.halide_b200_local_laplacian_sharded(bi.ptr, LEVELS, ctypes.c_float(ALPHA), ctypes.c_float(beta), bo.ptr,
                                                           0, h)
                if rc:
                    return rc, halide_b200.lib.last_error_message(), outs
                out[:] = 0
                bo.copy_to_host()
                outs.append(out)
        return 0, "", outs
    finally:
        l.halide_b200_dist_shutdown()


def _run(world, jobs, beta=1.0, x0=0, timeout=300):
    futs = [_RANK_THREADS[r].submit(_rank_main, r, world, jobs, beta, x0) for r in range(world)]
    return [f.result(timeout=timeout) for f in futs]


@contextmanager
def _settings(level=0, force_generic=0):
    """Process-wide: the gathered level (0: chosen by size) and the generic-kernel mask, for every rank thread."""
    l = _lib()
    l.halide_b200_ll_shard_coarse_level(level)
    l.halide_b200_ll_force_generic(force_generic)
    try:
        yield
    finally:
        l.halide_b200_ll_shard_coarse_level(0)
        l.halide_b200_ll_force_generic(0)


def _single(hb, img, beta=1.0, x0=0):
    return run_local_laplacian(hb, img, LEVELS, ALPHA, beta, in_mins=(x0, 0, 0), out_mins=(x0, 0, 0))


def _sharded(world, jobs, wants, beta=1.0, x0=0, level=0, force_generic=0):
    """Run `jobs` on `world` rank threads; every call's bands put together must equal the job's entry of `wants`.
    Returns the frame of the last call."""
    with _settings(level, force_generic):
        res = _run(world, jobs, beta, x0)
    for r, (rc, msg, _) in enumerate(res):
        assert rc == 0, f"rank {r} of {world}: error {rc}: {msg}"
    k = 0
    for (img, calls), want in zip(jobs, wants):
        for c in range(calls):
            got = np.concatenate([res[r][2][k] for r in range(world)], axis=1)
            bad = np.argwhere(got != want)
            assert bad.size == 0, f"frame {img.shape}, call {c}: {len(bad)} mismatching samples, first at {bad[0]}"
            k += 1
    return got


def _check(hb, world, img, beta=1.0, x0=0, level=0, force_generic=0, calls=1):
    return _sharded(world, [(img, calls)], [_single(hb, img, beta, x0)], beta, x0, level, force_generic)


# ---- bit parity with the single-GPU filter -------------------------------------------------------------------------

@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("level", [0, 2, 3, 4, 5, 6, 7])
@pytest.mark.parametrize("world,shape", [(w, s) for w, frames in FRAMES.items() for s in frames])
def test_bands_match_single_gpu(hb, world, shape, level, beta):
    """Every rank count, both frame layouts, the gathered level chosen by size and each forced level, both beta
    variants of the kernels."""
    _check(hb, world, u16_frame(shape, world * 100 + level), beta, level=level)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_band_seams_match_oracle(hb, oracle, world):
    """The rows around every band seam, against the CPU oracle run on the crop that determines them."""
    shape = FRAMES[world][0]
    img = u16_frame(shape, 40 + world)
    got = _check(hb, world, img)
    for r in range(1, world):
        seam = _band_rows(r, world, shape[1])[0]
        for x0 in (0, shape[2] - 128):
            _region_vs_oracle(oracle, img, got, seam - 64, x0)


@pytest.mark.parametrize("beta", [1.0, 0.6])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_input_x_min_one(hb, world, beta):
    """Frames whose columns start at x = 1: the pyramid's column parity and the level-1 kernel's unaligned loads."""
    _check(hb, world, u16_frame(FRAMES[world][0], 50 + world), beta, x0=1)


@pytest.mark.parametrize("mask", [1, 2, 4, 8])
@pytest.mark.parametrize("world", [3, 4])
def test_generic_kernel_paths(hb, world, mask):
    """halide_b200_ll_force_generic on the bands: 1 = generic down-sweep (level 1 in one launch that reads the halo
    rows), 2 = generic up-sweep, 4 = generic final kernel, 8 = no fused coarse launch."""
    _check(hb, world, u16_frame(FRAMES[world][0], 60 + mask), force_generic=mask)


@pytest.mark.parametrize("world", [3, 8])
def test_repeated_calls_then_new_geometry(hb, world):
    """Three calls per geometry, a second geometry, then the first again, on the same rank threads: the band plan is
    re-gathered on every change and pooled scratch is reused across calls."""
    a, b = u16_frame(FRAMES[world][0], 70), u16_frame(FRAMES[world][1], 71)
    _sharded(world, [(a, 3), (b, 3), (a, 1)], [_single(hb, a), _single(hb, b), _single(hb, a)])


def test_new_group_gathers_again(hb):
    """A frame over 8 ranks, another over 4 (threads 0-3 only), the first over 8 again: threads 4-7 still hold the
    first frame's band plan, but every member of a new group must take part in its band all-gather."""
    a, b = u16_frame(FRAMES[8][0], 72), u16_frame(FRAMES[4][0], 73)
    want_a = _single(hb, a)
    _sharded(8, [(a, 1)], [want_a])
    _sharded(4, [(b, 1)], [_single(hb, b)])
    _sharded(8, [(a, 1)], [want_a])


# ---- the split of levels 1-2 into interior and edge launches -------------------------------------------------------

def _level12_split(w, h, world, rank, level=0):
    """The spans run_local_laplacian_sharded gives its level-1/2 launches on `rank` (restated from the band geometry
    probe): None when the band has no interior level-1 rows, else the interior level-1 rows and the level-2 rows of the
    interior (c2), top and bottom launches."""
    from halide_b200 import dist
    jr = level or dist.shard_plan_level(w, h, world)
    lo, hi = _band_rows(rank, world, h)
    lv, _ = dist.band_geometry(w, h, lo, hi, rank == 0, rank == world - 1, jr)
    cy = lv[1]["d"]
    cy2 = lv[2]["own"] if jr == 2 else lv[2]["d"]
    i_lo, i_hi = max(cy[0], (lo + 2) >> 1), min(cy[1], (hi - 2) >> 1)
    if i_lo > i_hi:
        return None
    c2 = (max(cy2[0], (i_lo + 2) >> 1), min(cy2[1], (i_hi - 2) >> 1))
    top2 = (cy2[0], min(cy2[1], c2[0] - 1))
    bot2 = (max(c2[1], top2[1]) + 1, cy2[1])
    return {"interior": (i_lo, i_hi), "c2": c2, "top2": top2, "bot2": bot2}


def _empty(span):
    return span[0] > span[1]


def _find(pred, start):
    n = start
    while not pred(n):
        n += 1
    return n


@pytest.mark.parametrize("case", ["no_interior_rows", "empty_c2", "middle_rank_edges"])
def test_level12_split_branches(hb, oracle, case):
    """Frames that reach each branch of the split: a band too thin for interior level-1 rows (one launch after the
    halo), an interior launch with no level-2 rows of its own, and middle ranks whose top and bottom launches both
    build level-2 rows.  Checked against the single-GPU filter and the oracle."""
    w = 1000
    if case == "no_interior_rows":
        world, h = 2, 4
        assert any(_level12_split(w, h, world, r) is None for r in range(world))
    elif case == "empty_c2":
        world, h = 2, 9
        splits = [_level12_split(w, h, world, r) for r in range(world)]
        assert all(s is not None for s in splits) and any(_empty(s["c2"]) for s in splits)
    else:
        world = 4

        def edges(n):
            s = [_level12_split(w, n, world, r) for r in (1, 2)]
            return all(x is not None and not _empty(x["c2"]) and not _empty(x["top2"]) and not _empty(x["bot2"]) for x in s)
        h = _find(edges, 60)
    img = u16_frame((3, h, w), h)
    got = _check(hb, world, img, 0.6)
    assert np.array_equal(got, oracle.local_laplacian(img, LEVELS, ALPHA, 0.6))


def test_overlap_splits_level1(hb):
    """With the halo exchange on its own stream, levels 1-2 take more than one launch per rank call (the path the
    split tests mean to reach is the one that runs)."""
    assert os.environ.get("HALIDE_B200_SHARD_OVERLAP", "1") != "0"
    world, img = 3, u16_frame(FRAMES[3][0], 80)
    want = _single(hb, img)
    lib = hb.lib
    lib.profile_reset()
    lib.profile(True)
    try:
        _sharded(world, [(img, 2)], [want])
        report = lib.profile_report()
    finally:
        lib.profile(False)
        lib.profile_reset()
    assert report["ll_level1"][0] > 2 * world, report


def _one_stream_main():
    """Run in a subprocess with HALIDE_B200_SHARD_OVERLAP=0 (read once per process): the halo exchange on the compute
    stream, level 1 in one launch per call."""
    import halide_b200
    lib = halide_b200.lib
    for world in (2, 3, 8):
        for beta in (1.0, 0.6):
            img = u16_frame(FRAMES[world][0], 90 + world)
            want = _single(halide_b200, img, beta)
            lib.profile_reset()
            lib.profile(True)
            _sharded(world, [(img, 2)], [want], beta)
            report = lib.profile_report()
            lib.profile(False)
            assert report["ll_level1"][0] == 2 * world, report
    print("one-stream path OK")


def test_one_stream_path():
    env = dict(os.environ, HALIDE_B200_SHARD_OVERLAP="0", PYTHONPATH=os.pathsep.join([ROOT, TESTS]))
    out = subprocess.run([sys.executable, "-c", "import test_dist_loopback_gpu as t; t._one_stream_main()"], cwd=TESTS, env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "one-stream path OK" in out.stdout


# ---- bench.py's frame -----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def frame_16k(hb):
    img = np.random.default_rng(16).integers(0, 1 << 16, (3, 16384, 16384), dtype=np.uint16)
    return img, _single(hb, img)


@pytest.mark.parametrize("world", [8, 2])
def test_bench_frame_matches_single_gpu(frame_16k, world):
    """bench.py's workload (16384 x 16384 x 3, levels 8, alpha 1/7, beta 1) over 8 and 2 ranks."""
    img, want = frame_16k
    _sharded(world, [(img, 1)], [want])


# ---- bands too thin to shard -----------------------------------------------------------------------------------------

def _refuses_alone(w, h, world, level):
    """Per rank: would it refuse the frame judging only its own band, as each rank did before the refusal became
    collective?  (Its level 1..jr owns no row, or its input halo or a neighbour's reaches beyond the adjacent band.)"""
    from halide_b200 import dist
    jr = level or dist.shard_plan_level(w, h, world)
    bands = [_band_rows(q, world, h) for q in range(world)]
    geo = [dist.band_geometry(w, h, lo, hi, q == 0, q == world - 1, jr) for q, (lo, hi) in enumerate(bands)]
    rows = lambda q: bands[q][1] - bands[q][0] + 1 if 0 <= q < world else 0
    above = lambda q: bands[q][0] - geo[q][1][0]
    below = lambda q: geo[q][1][1] - bands[q][1]
    out = []
    for q in range(world):
        no_row = any(_empty(geo[q][0][j]["own"]) for j in range(1, min(jr, 7) + 1))
        halo = above(q) > rows(q - 1) or below(q) > rows(q + 1) or (q > 0 and below(q - 1) > rows(q)) or \
            (q < world - 1 and above(q + 1) > rows(q))
        out.append(no_row or halo)
    return out


@pytest.mark.parametrize("world,level,h_from", [(8, 0, 35), (4, 0, 17), (3, 5, 40), (4, 7, 100), (8, 3, 40)])
def test_thin_bands_refused_by_every_rank(hb, world, level, h_from):
    """Frames on which some ranks' own bands are fine and others' are too thin: every rank must refuse with
    constraint_violated before any exchange (a rank refusing alone left its neighbours waiting for it), and the group
    must then run a valid frame."""
    w = 1000
    h = _find(lambda n: any(_refuses_alone(w, n, world, level)) and not all(_refuses_alone(w, n, world, level)), h_from)
    if level == 0:
        assert h == h_from
    with _settings(level):
        res = _run(world, [(u16_frame((3, h, w), h), 1)])
    assert [rc for rc, _, _ in res] == [CONSTRAINT_VIOLATED] * world, [(r, rc, msg) for r, (rc, msg, _) in enumerate(res)]
    _check(hb, world, u16_frame(FRAMES[world][0], 99), level=level)
