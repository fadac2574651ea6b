"""Row-sharded multi-GPU execution: one process per GPU (torchrun).

local_laplacian: `RowSharder` joins the library's communicator and calls halide_b200_local_laplacian_sharded: one
NCCL exchange of input halo rows with the row neighbours (every pyramid row a band needs beyond itself is recomputed
from them), one all-to-all gather of a coarse pyramid level, the coarser levels replicated
(halide_b200/csrc/local_laplacian.cu, ll_geom.h, hb_dist.cu; DESIGN.md §7).  torch.distributed is only the control
plane there (broadcast of the NCCL unique id, barriers in bench.py).

The five filters that depend on other bands only through a halo of input rows are sharded by host logic at the end of
this file (`InputHaloSharder`): a torch.distributed point-to-point row exchange, then the ordinary single-GPU filter.
"""
import ctypes
import os

from .lib import lib, check


def band_rows(rank, world, frame_h):
    """Rows [lo, hi] of the frame owned by `rank`: contiguous, top to bottom, balanced."""
    base, rem = divmod(frame_h, world)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0) - 1
    return lo, hi


def band_geometry(frame_w, frame_h, lo, hi, first, last, jr):
    """Per-level rows of a band with pyramid level `jr` gathered (host-only probe of ll_geom.h: ShardLevel): a list of
    8 dicts {own, d, u, S} of inclusive (lo, hi) pairs — rows owned in the gather partition, Gaussian-side rows
    computed and held, outGPyramid rows needed, the level's stored rows on the whole frame — and the input rows read."""
    out = (ctypes.c_int32 * 66)()
    check(lib.halide_b200_ll_band_geometry(frame_w, frame_h, lo, hi, int(first), int(last), int(jr), out))
    levels = []
    for j in range(8):
        o = out[j * 8:(j + 1) * 8]
        levels.append({"own": (o[0], o[1]), "d": (o[2], o[3]), "u": (o[4], o[5]), "S": (o[6], o[7])})
    return levels, (out[64], out[65])


def shard_plan_level(frame_w, frame_h, world):
    """The pyramid level halide_b200_local_laplacian_sharded gathers all-to-all for this frame and rank count."""
    return int(lib.halide_b200_ll_shard_plan_level(frame_w, frame_h, world))


_initialised = False


def init_from_torch_distributed():
    """Join the library's NCCL communicator using torch.distributed as the control plane."""
    global _initialised
    if _initialised:
        return
    import torch
    import torch.distributed as td
    rank, world = td.get_rank(), td.get_world_size()
    buf = ctypes.create_string_buffer(128)
    if rank == 0:
        check(lib.halide_b200_dist_unique_id(buf))
    if td.get_backend() == "nccl":
        t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).cuda()
        td.broadcast(t, 0)
        raw = bytes(t.cpu().numpy().tobytes())
    else:
        obj = [buf.raw]
        td.broadcast_object_list(obj, 0)
        raw = obj[0]
    check(lib.halide_b200_dist_init(rank, world, raw))
    _initialised = True


class RowSharder:
    """Each rank holds a band of W x band_h rows of a frame of W x (band_h * world) rows."""

    def __init__(self, rank, world, width, band_h):
        self.rank, self.world, self.width, self.band_h = rank, world, width, band_h
        self.frame_h = band_h * world
        self.lo, self.hi = band_rows(rank, world, self.frame_h)
        init_from_torch_distributed()
        lvl = os.environ.get("HALIDE_B200_SHARD_COARSE_LEVEL")  # experiment knob; see halide_b200_ll_shard_coarse_level
        if lvl is not None:
            lib.halide_b200_ll_shard_coarse_level(int(lvl))

    def set_band_mins(self, buf):
        """Put a band buffer (rows 0..band_h-1 locally) at its rows of the frame."""
        buf.dims[1].min = self.lo

    def local_laplacian(self, in_band, levels, alpha, beta, out_band):
        self.set_band_mins(in_band)
        self.set_band_mins(out_band)
        return check(lib.halide_b200_local_laplacian_sharded(in_band.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                             ctypes.c_float(beta), out_band.ptr, ctypes.c_int32(0),
                                                             ctypes.c_int32(self.frame_h)))


# ---- row sharding of the filters whose only cross-band dependence is a halo of INPUT rows --------------------------
# (SURVEY.md §8e: blur, nl_means, stencil_chain, bilateral_grid, camera_pipe.)  Each rank owns a contiguous band of
# the frame's rows, fetches the few input rows its output band additionally reads from whichever ranks own them (one
# batch of point-to-point messages, torch.distributed as plumbing: NCCL between GPUs, gloo in the CPU tests), and then
# calls the ordinary single-GPU filter on the extended input with both buffers placed at their rows of the frame
# (halide_buffer_t mins) — no kernel knows about the sharding.  For the filters that clamp at the input buffer's edge
# (repeat_edge) the extended buffer ends exactly at the frame edge on the first / last rank and at least a full stencil
# footprint beyond the band elsewhere, so the clamp only ever acts where it would on the whole frame.

def default_in_own(rank, world, out_rows, in_frame_rows):
    """Input rows owned by `rank` when the output rows are split by band_rows: the same row numbers, with the input
    frame's leading rows given to rank 0 and its trailing rows to the last rank (inputs are taller than outputs for
    blur and camera_pipe)."""
    lo, hi = out_rows
    if rank == 0:
        lo = in_frame_rows[0]
    if rank == world - 1:
        hi = in_frame_rows[1]
    return lo, hi


def halo_rows(name, **params):
    """(rows above, rows below) of the input that an output band of filter `name` reads beyond its own row numbers."""
    if name == "halide_blur":
        return 0, 2                                     # in(x..x+2, y..y+2), halide_blur_generator.cpp:31-40
    if name == "nl_means":
        r = params["search_area"] // 2 + params["patch_size"] // 2   # nl_means_generator.cpp:26-60
        return r, r
    if name == "stencil_chain":
        return 2 * params.get("stencils", 32), 2 * params.get("stencils", 32)   # 5x5 stencil per stage
    if name == "bilateral_grid":
        # grid cells yi-2 .. yi+3 (blury +-2, slice yi / yi+1) of S rows each, cell origin offset by -S/2: at most
        # 3S - 1 + S/2 rows above and 4S - 1 - S/2 below (S = s_sigma, 8 unless given)
        s = params.get("s_sigma", 8)
        return 4 * s, 4 * s
    raise ValueError(f"no halo rule for {name}")


def exchange_rows(band, own, need, rank, world, row_dim=-2):
    """Collective.  `band` holds this rank's rows own=(a, b) (inclusive, frame coordinates) along `row_dim`; returns a
    tensor holding rows need=(lo, hi), assembled from this rank's rows and the rows other ranks own.  Every rank must
    call it; rows nobody owns raise."""
    import torch
    import torch.distributed as td
    row_dim = row_dim % band.dim()
    meta = torch.tensor([own[0], own[1], need[0], need[1]], dtype=torch.int64, device=band.device)
    gathered = [torch.empty_like(meta) for _ in range(world)]
    td.all_gather(gathered, meta)
    table = [tuple(int(v) for v in m.tolist()) for m in gathered]
    shape = list(band.shape)
    shape[row_dim] = need[1] - need[0] + 1
    out = torch.empty(shape, dtype=band.dtype, device=band.device)
    covered = torch.zeros(shape[row_dim], dtype=torch.bool)

    def wire(t):  # NCCL has no 16-bit integer types (and gloo no uint16): ship contiguous tensors as bytes
        return t.view(torch.uint8) if t.dtype in (torch.uint16, torch.int16) else t

    lo, hi = max(need[0], own[0]), min(need[1], own[1])
    if lo <= hi:
        out.narrow(row_dim, lo - need[0], hi - lo + 1).copy_(band.narrow(row_dim, lo - own[0], hi - lo + 1))
        covered[lo - need[0]:hi - need[0] + 1] = True
    ops, keep = [], []
    for q in range(world):
        if q == rank:
            continue
        q_own_lo, q_own_hi, q_need_lo, q_need_hi = table[q]
        s_lo, s_hi = max(q_need_lo, own[0]), min(q_need_hi, own[1])       # rows q wants from me
        if s_lo <= s_hi:
            t = band.narrow(row_dim, s_lo - own[0], s_hi - s_lo + 1).contiguous()
            keep.append(t)
            ops.append(td.P2POp(td.isend, wire(t), q))
        r_lo, r_hi = max(need[0], q_own_lo), min(need[1], q_own_hi)       # rows I want from q
        if r_lo <= r_hi:
            rs = list(band.shape)
            rs[row_dim] = r_hi - r_lo + 1
            buf = torch.empty(rs, dtype=band.dtype, device=band.device)
            keep.append((r_lo, r_hi, buf))
            ops.append(td.P2POp(td.irecv, wire(buf), q))
    if ops:
        for req in td.batch_isend_irecv(ops):
            req.wait()
    for item in keep:
        if isinstance(item, tuple):
            r_lo, r_hi, buf = item
            out.narrow(row_dim, r_lo - need[0], r_hi - r_lo + 1).copy_(buf)
            covered[r_lo - need[0]:r_hi - need[0] + 1] = True
    if not bool(covered.all()):
        raise RuntimeError(f"rank {rank}: rows {need} are not all owned by some rank (table {table})")
    return out


def run_input_halo_sharded(call, in_band, in_own, in_frame_rows, out_band, out_rows, halo, rank, world, row_dim=-2):
    """One sharded call: fetch the halo rows, then call(extended_input, first_row_of_it, out_band, first_out_row).
    `halo` = (rows above out_rows[0], rows below out_rows[1]) read from the input; clipped to the input frame."""
    need = (max(in_frame_rows[0], out_rows[0] - halo[0]), min(in_frame_rows[1], out_rows[1] + halo[1]))
    ext = exchange_rows(in_band, in_own, need, rank, world, row_dim)
    call(ext, need[0], out_band, out_rows[0])
    return need


class InputHaloSharder:
    """The five input-halo filters on one band per rank (device tensors, NCCL).  Output rows are split by
    band_rows; pass each rank's input rows as given by default_in_own."""

    def __init__(self, rank, world):
        self.rank, self.world = rank, world

    def _buf(self, t, row0, ndim_rows_from_end=2):
        from .buffer import HalideBuffer
        mins = [0] * t.dim()
        mins[1] = row0  # halide dims are innermost-first: (x, y[, c])
        return HalideBuffer.from_torch(t, mins=tuple(mins))

    def _run(self, name, invoke, in_band, in_frame_h, out_band, out_frame_h, **params):
        out_rows = band_rows(self.rank, self.world, out_frame_h)
        in_own = default_in_own(self.rank, self.world, out_rows, (0, in_frame_h - 1))

        def call(ext, ext_row0, out_t, out_row0):
            invoke(self._buf(ext, ext_row0), self._buf(out_t, out_row0))

        return run_input_halo_sharded(call, in_band, in_own, (0, in_frame_h - 1), out_band, out_rows,
                                      halo_rows(name, **params), self.rank, self.world)

    def halide_blur(self, in_band, out_band, out_frame_h):
        from . import filters
        return self._run("halide_blur", lambda bi, bo: filters.halide_blur(bi, bo), in_band, out_frame_h + 2, out_band,
                         out_frame_h)

    def nl_means(self, in_band, patch_size, search_area, sigma, out_band, frame_h):
        from . import filters
        return self._run("nl_means", lambda bi, bo: filters.nl_means(bi, patch_size, search_area, sigma, bo), in_band,
                         frame_h, out_band, frame_h, patch_size=patch_size, search_area=search_area)

    def stencil_chain(self, in_band, out_band, frame_h, stencils=32):
        from . import filters
        if stencils == 32:
            invoke = lambda bi, bo: filters.stencil_chain(bi, bo)  # noqa: E731
        else:
            invoke = lambda bi, bo: filters.stencil_chain_stencils(bi, stencils, bo)  # noqa: E731
        return self._run("stencil_chain", invoke, in_band, frame_h, out_band, frame_h, stencils=stencils)

    def bilateral_grid(self, in_band, r_sigma, out_band, frame_h, s_sigma=8):
        from . import filters
        if s_sigma == 8:
            invoke = lambda bi, bo: filters.bilateral_grid(bi, r_sigma, bo)  # noqa: E731
        else:
            invoke = lambda bi, bo: filters.bilateral_grid_s_sigma(bi, s_sigma, r_sigma, bo)  # noqa: E731
        return self._run("bilateral_grid", invoke, in_band, frame_h, out_band, frame_h, s_sigma=s_sigma)

    def camera_pipe(self, raw_band, raw_frame_h, m3200, m7000, color_temp, gamma, contrast, sharpen_strength, black, white,
                    out_band, out_frame_h):
        """raw_band: uint16 [rows, W_raw]; out_band: uint8 [3, rows, W_out]; m3200 / m7000: float32 [3, 4] tensors."""
        from . import filters
        from .buffer import HalideBuffer
        out_rows = band_rows(self.rank, self.world, out_frame_h)
        in_own = default_in_own(self.rank, self.world, out_rows, (0, raw_frame_h - 1))
        b32, b70 = HalideBuffer.from_torch(m3200), HalideBuffer.from_torch(m7000)
        args = (color_temp, gamma, contrast, sharpen_strength, black, white)
        need = camera_pipe_need_rows(self._buf(out_band, out_rows[0]), b32, b70, args)

        def call(ext, ext_row0, out_t, out_row0):
            filters.camera_pipe(self._buf(ext, ext_row0), b32, b70, *args, self._buf(out_t, out_row0))

        ext = exchange_rows(raw_band, in_own, need, self.rank, self.world)
        call(ext, need[0], out_band, out_rows[0])
        return need


def camera_pipe_need_rows(out_buf, b32, b70, args):
    """Raw rows the output region described by `out_buf` reads: asked from the filter itself in bounds-query mode (the
    input is shifted by (16, 12) and never clamped, camera_pipe_generator.cpp:407-412; host-only, no CUDA call)."""
    import numpy as np
    from . import filters
    from .buffer import HalideBuffer
    q = HalideBuffer.bounds_query(np.uint16, 2)
    filters.camera_pipe(q, b32, b70, *args, out_buf)
    (_x0, _w, _), (y0, h, _) = q.shape()
    return y0, y0 + h - 1
