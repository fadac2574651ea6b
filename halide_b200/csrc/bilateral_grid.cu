// bilateral_grid.cu — bilateral_grid(input, r_sigma, output) for sm_90a (s_sigma = 8), and
// halide_b200_bilateral_grid_s_sigma for any cell size (its kernels follow bg_slice below).
//
// Reference algorithm: apps/bilateral_grid/bilateral_grid_generator.cpp:17-67
//   histogram(x,y,zi,c) += mux(c,{val,1}) over the 8x8 pixels of cell (x,y) (offset -4), zi = int(val/r_sigma + 0.5)
//   blurz/blurx/blury: unnormalised 1-4-6-4-1 along z, x, y
//   output = trilinear slice of blury at (x/8, y/8, val/r_sigma), channel 0 / channel 1
// Float pipeline against oracle/oracle_bilateral_grid.cpp: the kernels perform the oracle's float operations in its order
// (each bin summed rows, then columns; the same blur5 association; the lerp nest x -> y -> z; an IEEE divide; no
// contraction: --fmad=false here, -ffp-contract=off there), and the input clamp maps NaN to 1 as Halide's select-based
// min / max do (hl::clamp01).  So the any-S kernels are bit-exact on any input.  The one re-association is bg_hist_blurz
// (S = 8): lanes 2c and 2c+1 each sum four columns of a cell and their sums are then added, which gives the oracle's bits
// wherever every partial sum of a bin is exact (a uint16 frame / 65536: at most 64 terms of 16 bits), and stays within
// 1e-4 relative on arbitrary float data (all terms are non-negative: no cancellation).
// (tests/test_bilateral_grid_exact_gpu.py holds both bit for bit; tests/test_bilateral_grid_gpu.py S = 8 on noise.)
//
// HBM-bound: 8 algorithmic B/px (4 in + 4 out).  Three kernels:
//   bg_hist_blurz   reads the frame once with coalesced float4 loads; each lane scatters its 4
//                   columns x 8 rows into lane-private shared-memory bins (no atomics, no
//                   conflicts: bin-major layout), the two lanes of a cell then emit blurz.
//   bg_blur_xy      blurx then blury fused: each thread owns one (cell column, z, channel) and walks
//                   down the grid rows with a 5-row register window of blurx values.
//   bg_slice        one block per 120 x 8 pixels (one row of grid cells): the 16 x 2 x nz cells it interpolates between
//                   are staged in shared memory with a plane stride of 32 cells (bank = cell, whatever the plane);
//                   4 pixels per thread (float4 in / float4 out), 8 shared 8-byte corner loads per pixel.
// Grid layout in HBM: [cell_y][cell_x][z][2] f32 — the (z, z+1) x (value, weight) quad a pixel
// needs at one corner is 16 contiguous bytes.
#include <algorithm>

#include "hb_common.h"
#include "hl_math.cuh"

namespace {

constexpr int S = 8;  // s_sigma GeneratorParam of the shipped app (generator :8)

struct BGParams {
    const float *in;  // element at input mins
    int64_t in_sy;
    int in_x0, in_y0, in_w, in_h;
    float *out;  // element at output mins
    int64_t out_sy;
    int out_x0, out_y0, W, H;
    float inv_r;
    int zmax;      // largest histogram bin
    int nz;        // blurred grid planes: z in [0, zmax+1]
    int gx0, gy0;  // first grid cell stored (absolute cell coordinates)
    int gw, gh;    // stored cells
    float *grid_a, *grid_b;  // [gh][gw][nz][2]
};

// ---- K1: histogram + blurz --------------------------------------------------------------------------
// One warp handles 16 horizontally adjacent cells (128 px): lane l covers columns 4l..4l+3 of the
// strip for all 8 rows of the cell row.  Bins live in shared memory as [bin][channel][thread].
__global__ void __launch_bounds__(128) bg_hist_blurz_kernel(BGParams p) {
    extern __shared__ float s_bins[];  // (zmax+1) * 2 * 128
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nb = p.zmax + 1;
    for (int b = 0; b < nb * 2; b++) s_bins[b * 128 + tid] = 0.f;
    const int cell_row = blockIdx.y;                       // index into stored rows
    const int cell_col0 = (blockIdx.x * 4 + warp) * 16;    // first stored cell column of this warp
    const int gy = p.gy0 + cell_row;
    const int px0 = (p.gx0 + cell_col0) * S - S / 2 + 4 * lane;  // absolute x of this lane's first pixel
    const bool interior_x = (px0 >= p.in_x0) && (px0 + 3 <= p.in_x0 + p.in_w - 1);
#pragma unroll
    for (int ry = 0; ry < S; ry++) {
        int y = hl::clampi(gy * S + ry - S / 2, p.in_y0, p.in_y0 + p.in_h - 1) - p.in_y0;
        const float *row = p.in + (int64_t)y * p.in_sy;
        float v[4];
        if (interior_x && ((reinterpret_cast<uintptr_t>(row + (px0 - p.in_x0)) & 15) == 0)) {
            float4 t = __ldg(reinterpret_cast<const float4 *>(row + (px0 - p.in_x0)));
            v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
            for (int i = 0; i < 4; i++) {
                int x = hl::clampi(px0 + i, p.in_x0, p.in_x0 + p.in_w - 1) - p.in_x0;
                v[i] = __ldg(row + x);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            float val = hl::clamp01(v[i]);
            int zi = (int)__fadd_rn(__fmul_rn(val, p.inv_r), 0.5f);
            zi = min(zi, p.zmax);
            s_bins[(zi * 2) * 128 + tid] += val;
            s_bins[(zi * 2 + 1) * 128 + tid] += 1.0f;
        }
    }
    __syncwarp();
    // lanes 2c, 2c+1 hold the two halves of cell c: even lane emits channel 0, odd lane channel 1
    const int cell = cell_col0 + (lane >> 1);
    if (cell >= p.gw) return;
    const int ch = lane & 1;
    const int ta = tid & ~1, tb = ta + 1;
    auto h = [&](int z) -> float {
        if (z < 0 || z > p.zmax) return 0.f;
        return s_bins[(z * 2 + ch) * 128 + ta] + s_bins[(z * 2 + ch) * 128 + tb];
    };
    float *g = p.grid_a + ((size_t)cell_row * p.gw + cell) * p.nz * 2 + ch;
    float hm2 = 0.f, hm1 = 0.f, h0 = h(0), h1 = h(1), h2 = h(2);
    for (int z = 0; z < p.nz; z++) {
        // blurz = h(z-2) + 4 h(z-1) + 6 h(z) + 4 h(z+1) + h(z+2) (generator :33-37)
        g[z * 2] = (((hm2 + hm1 * 4.0f) + h0 * 6.0f) + h1 * 4.0f) + h2;
        hm2 = hm1; hm1 = h0; h0 = h1; h1 = h2; h2 = h(z + 3);
    }
}

// ---- K2: blurx + blury on the grid -------------------------------------------------------------------
// blury is only needed on the interior (stored region shrunk by 2 cells on every side); the result is
// written over the same extent with the border cells left untouched (never read by the slice).
__global__ void __launch_bounds__(256) bg_blur_xy_kernel(BGParams p, int rows_per_block) {
    const int V = p.nz * 2;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;  // (cell_x - 2) * V + v
    const int cx = t / V + 2;
    if (cx >= p.gw - 2) return;
    const int v = t - (cx - 2) * V;
    const int y_begin = 2 + blockIdx.y * rows_per_block;
    const int y_end = min(y_begin + rows_per_block, p.gh - 2);
    if (y_begin >= y_end) return;
    // x-blur of one grid row at this thread's (cell, value): five loads, combined in the generator's order.  The loads of
    // two rows are issued together (ten in flight per thread): with one row per iteration the kernel sat on its own load
    // latency.
    struct Taps {
        float t[5];
    };
    auto load_taps = [&](int cy) -> Taps {
        const float *r = p.grid_a + ((size_t)cy * p.gw + cx) * V + v;
        Taps k;
        k.t[0] = __ldg(r - 2 * V); k.t[1] = __ldg(r - V); k.t[2] = __ldg(r); k.t[3] = __ldg(r + V); k.t[4] = __ldg(r + 2 * V);
        return k;
    };
    auto blurx = [](const Taps &k) -> float {
        return (((k.t[0] + k.t[1] * 4.0f) + k.t[2] * 6.0f) + k.t[3] * 4.0f) + k.t[4];
    };
    float a, b, c, d;
    {
        const Taps k0 = load_taps(y_begin - 2), k1 = load_taps(y_begin - 1), k2 = load_taps(y_begin), k3 = load_taps(y_begin + 1);
        a = blurx(k0); b = blurx(k1); c = blurx(k2); d = blurx(k3);
    }
    for (int cy = y_begin; cy < y_end; cy += 2) {
        const bool two = cy + 1 < y_end;
        const Taps k0 = load_taps(cy + 2);
        const Taps k1 = load_taps(two ? cy + 3 : cy + 2);  // (rows up to y_end + 1 <= gh - 1 exist: the grid keeps a 2-cell border)
        float e = blurx(k0);
        p.grid_b[((size_t)cy * p.gw + cx) * V + v] = (((a + b * 4.0f) + c * 6.0f) + d * 4.0f) + e;
        a = b; b = c; c = d; d = e;
        if (two) {
            e = blurx(k1);
            p.grid_b[((size_t)(cy + 1) * p.gw + cx) * V + v] = (((a + b * 4.0f) + c * 6.0f) + d * 4.0f) + e;
            a = b; b = c; c = d; d = e;
        }
    }
}

// ---- K3: trilinear slice + normalise -----------------------------------------------------------------
// One block = 128 x 8 pixels = one row of grid cells: the 17 x 2 cells (x nz planes x 2 channels) its pixels interpolate
// between are staged once into shared memory as [z][cell row][24] float2, so that a corner fetch is one 8-byte shared
// load.  Lane l of a warp owns the 4 pixels of cell (l & 15) at offset 4 * (l >> 4): the 16 lanes of a half-warp — the
// unit an 8-byte shared load is served in — then read 16 DIFFERENT cells, and with a plane stride of 48 entries
// (= 0 mod 16 bank pairs) the bank of a fetch depends on the cell only, never on the data-dependent plane zi: no
// conflicts whatever the image.  (Lanes 2c and 2c+1 sharing cell c would make every fetch a two-way conflict on a noisy
// image, where the two lanes' planes zi differ.)
constexpr int kSliceW = 128, kSliceCells = 17, kSlicePitch = 24;

__global__ void __launch_bounds__(256) bg_slice_kernel(BGParams p) {
    extern __shared__ float2 s_grid[];  // [nz][2][kSlicePitch]
    const int lane = threadIdx.x, row = threadIdx.y, tid = row * 32 + lane;
    const int X0 = (p.out_x0 & ~(S - 1)) + blockIdx.x * kSliceW, Y0 = (p.out_y0 & ~(S - 1)) + blockIdx.y * S;
    const int cx0 = (X0 >> 3) - p.gx0, cy0 = (Y0 >> 3) - p.gy0;  // first stored cell of the tile
    {
        const float2 *g = reinterpret_cast<const float2 *>(p.grid_b);
        for (int it = tid; it < 2 * kSliceCells * p.nz; it += 256) {
            // (cell fastest: consecutive lanes store to consecutive banks; the planes of a cell are contiguous in HBM, so
            // the later planes of a cell hit the line the first one brought into L1)
            const int z = it / (2 * kSliceCells), cell = it - z * (2 * kSliceCells);
            const int cr = cell >= kSliceCells ? 1 : 0, cc = cell - cr * kSliceCells;
            const int cx = min(cx0 + cc, p.gw - 1), cy = min(cy0 + cr, p.gh - 1);
            s_grid[(z * 2 + cr) * kSlicePitch + cc] = __ldg(g + ((size_t)cy * p.gw + cx) * p.nz + z);
        }
    }
    __syncthreads();
    const int y = Y0 + row, x = X0 + 8 * (lane & 15) + 4 * (lane >> 4);
    if (y < p.out_y0 || y >= p.out_y0 + p.H || x + 3 < p.out_x0 || x >= p.out_x0 + p.W) return;
    const float *ip = p.in + (int64_t)(y - p.in_y0) * p.in_sy + (x - p.in_x0);
    float *op = p.out + (int64_t)(y - p.out_y0) * p.out_sy + (x - p.out_x0);
    const float2 *c00 = s_grid + (lane & 15);  // cell (xi, yi) of this thread's four pixels; xi + 1: +1, yi + 1: +kSlicePitch
    const float yf = __fmul_rn((float)(y & (S - 1)), 0.125f);
    auto px = [&](float raw, int xx) -> float {
        const float val = hl::clamp01(raw);
        const float zv = __fmul_rn(val, p.inv_r);
        int zi = (int)zv;
        const float zf = __fsub_rn(zv, (float)zi);
        zi = min(zi, p.nz - 2);
        const float xf = __fmul_rn((float)(xx & (S - 1)), 0.125f);
        const float2 *c = c00 + zi * (2 * kSlicePitch);
        const float2 a0 = c[0], b0 = c[1], d0 = c[kSlicePitch], e0 = c[kSlicePitch + 1];
        const float2 a1 = c[2 * kSlicePitch], b1 = c[2 * kSlicePitch + 1], d1 = c[3 * kSlicePitch], e1 = c[3 * kSlicePitch + 1];
        // lerp nest x -> y -> z exactly as generator :59-64
        const float v0 = hl::lerpf(hl::lerpf(hl::lerpf(a0.x, b0.x, xf), hl::lerpf(d0.x, e0.x, xf), yf),
                                   hl::lerpf(hl::lerpf(a1.x, b1.x, xf), hl::lerpf(d1.x, e1.x, xf), yf), zf);
        const float v1 = hl::lerpf(hl::lerpf(hl::lerpf(a0.y, b0.y, xf), hl::lerpf(d0.y, e0.y, xf), yf),
                                   hl::lerpf(hl::lerpf(a1.y, b1.y, xf), hl::lerpf(d1.y, e1.y, xf), yf), zf);
        return __fdiv_rn(v0, v1);
    };
    const bool full = x >= p.out_x0 && x + 3 < p.out_x0 + p.W;
    if (full && ((reinterpret_cast<uintptr_t>(ip) | reinterpret_cast<uintptr_t>(op)) & 15) == 0) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(ip));
        float4 o;
        o.x = px(v.x, x);
        o.y = px(v.y, x + 1);
        o.z = px(v.z, x + 2);
        o.w = px(v.w, x + 3);
        *reinterpret_cast<float4 *>(op) = o;
    } else {
        for (int i = 0; i < 4; i++) {
            if (x + i >= p.out_x0 && x + i < p.out_x0 + p.W) op[i] = px(__ldg(ip + i), x + i);
        }
    }
}

// ==== any cell size: halide_b200_bilateral_grid_s_sigma ==============================================================
// bg_blur_xy only sees the grid and runs unchanged; the histogram and slice kernels below take S at run time.

// floor(n / S) = (n * mag) >> kMagShift with mag = ceil(2^kMagShift / S), exact for 0 <= n and n * S < 2^kMagShift:
// n * mag / 2^k = n / S + n * e / (S * 2^k) with 0 <= e < S, and that error stays below 1 / S (the least distance from
// n / S up to the next integer) when n * e < 2^k.  The slice applies it to offsets n < S + 1024 <= 1152 (its tallest
// tile is 4 passes of 256 rows, its widest 128 columns) and the histogram to column offsets n < kHistCols = 4096, with
// S <= 128: n * S <= 2^19, and n * mag < 4096 * 2^20 fits in 32 bits.
constexpr int kMagShift = 20;

struct BGSParams {
    int S;          // cell size in pixels, 1..128
    float inv_s;    // fold(1 / S): the reciprocal in double rounded to float (hl::recip_const of the oracle)
    uint32_t mag;   // ceil(2^kMagShift / S)
    int cpb, cslots;  // histogram: cells per block, cell slots (nb threads each; a slot takes every cslots-th cell)
    int rows_chunk;   // histogram: rows staged at a time
    int cell_stride;  // histogram: float2 per staged cell (odd)
    int tx, th;     // slice tile: tx threads (4 px each) across, th pixel rows
    int ncx, ncy;   // slice tile: staged cells per row, staged cell rows
    int plane;      // slice tile: float2 entries per staged plane (odd)
};

__device__ __forceinline__ int floor_div_dev(int a, int b) {  // b > 0; per block, never per pixel
    const int q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

// ---- histogram + blurz for any S ---------------------------------------------------------------------------------
// Bin b of a cell is the sequential float sum, in the generator's order (rows, then columns: the RDom's r.x innermost),
// of the cell's pixels that fall into b; pixels of other bins never touch it.  So a thread per (cell, bin) that walks the
// cell's pixels in that order and adds those of its bin forms exactly the generator's sum, and a cell's S x S pixels are
// shared out over nb threads.  (The weight channel adds 1.0f per pixel: exact integers, in any order.)
// Block = 256 threads over cpb = cslots * k horizontally adjacent cells of one cell row: thread t < cslots * nb owns bin
// t % nb of cells t / nb + j * cslots.  Rows are staged rows_chunk at a time, all cpb * S columns of the block read with
// coalesced loads, each pixel as (clamped value, bin) in one float2, cell-major with an odd cell stride: lanes of one cell
// read one address, lanes of adjacent cells different banks.  Running sums live in shared memory as [cell][bin], each
// entry owned by one thread.  blurz then runs over (cell, z) items, so consecutive threads store consecutive float2 of the
// grid (the block's cells are contiguous there).  (The minimum-blocks hint: without it ptxas held this kernel to 32
// registers and spilled.)
__global__ void __launch_bounds__(256, 1) bg_hist_blurz_s_kernel(BGParams p, BGSParams q) {
    extern __shared__ float2 s_hist[];  // [cpb][nb] running sums, then [cpb][cell_stride] staged pixels
    const int tid = threadIdx.x, S = q.S, nb = p.zmax + 1, cpb = q.cpb;
    float2 *s_pix = s_hist + cpb * nb;
    for (int i = tid; i < cpb * nb; i += 256) s_hist[i] = make_float2(0.f, 0.f);
    const int cell_row = blockIdx.x, c0 = blockIdx.y * cpb;
    const int ncell = min(cpb, p.gw - c0);  // stored cells of this block
    const int gy = p.gy0 + cell_row;
    const int xb = (p.gx0 + c0) * S - S / 2;  // absolute x of the block's first pixel column
    const int xlo = p.in_x0, xhi = p.in_x0 + p.in_w - 1;
    const int cols = ncell * S, cs = q.cell_stride;
    const int b = tid % nb, slot = tid / nb;
    for (int r0 = 0; r0 < S; r0 += q.rows_chunk) {
        const int nr = min(q.rows_chunk, S - r0);
        __syncthreads();  // the previous chunk is consumed (first chunk: the sums are cleared)
        for (int r = 0; r < nr; r++) {
            const int y = hl::clampi(gy * S + r0 + r - S / 2, p.in_y0, p.in_y0 + p.in_h - 1) - p.in_y0;
            const float *row = p.in + (int64_t)y * p.in_sy;
            for (int c = tid; c < cols; c += 256) {
                const float val = hl::clamp01(__ldg(row + (hl::clampi(xb + c, xlo, xhi) - xlo)));
                int zi = (int)__fadd_rn(__fmul_rn(val, p.inv_r), 0.5f);
                zi = min(zi, p.zmax);
                const int cell = (int)(((uint32_t)c * q.mag) >> kMagShift);
                s_pix[cell * cs + r * S + (c - cell * S)] = make_float2(val, __int_as_float(zi));
            }
        }
        __syncthreads();
        if (slot < q.cslots) {
            for (int cell = slot; cell < ncell; cell += q.cslots) {
                const float2 *px = s_pix + cell * cs;
                float2 acc = s_hist[cell * nb + b];
                for (int i = 0; i < nr * S; i++) {
                    const float2 e = px[i];
                    if (__float_as_int(e.y) == b) {
                        acc.x += e.x;
                        acc.y += 1.0f;
                    }
                }
                s_hist[cell * nb + b] = acc;
            }
        }
    }
    __syncthreads();
    float2 *g = reinterpret_cast<float2 *>(p.grid_a) + ((size_t)cell_row * p.gw + c0) * p.nz;
    for (int it = tid; it < ncell * p.nz; it += 256) {
        const int cell = it / p.nz, z = it - cell * p.nz;
        const float2 *hc = s_hist + cell * nb;
        float2 t[5];  // h(z-2) .. h(z+2), zero outside the bins
#pragma unroll
        for (int d = 0; d < 5; d++) {
            const int zz = z - 2 + d;
            t[d] = (zz < 0 || zz > p.zmax) ? make_float2(0.f, 0.f) : hc[zz];
        }
        const float2 hm2 = t[0], hm1 = t[1], h0 = t[2], h1 = t[3], h2 = t[4];
        // blurz = h(z-2) + 4 h(z-1) + 6 h(z) + 4 h(z+1) + h(z+2) (generator :33-37)
        g[it] = make_float2((((hm2.x + hm1.x * 4.0f) + h0.x * 6.0f) + h1.x * 4.0f) + h2.x,
                            (((hm2.y + hm1.y * 4.0f) + h0.y * 6.0f) + h1.y * 4.0f) + h2.y);
    }
}

// Histogram block shape for cell size S, nb bins and a grid of gw x gh cells: as many cell slots as 256 threads hold
// (at most 4096 / S columns' worth), k cells per slot so a block reads at least 256 columns, running sums within 64 KB,
// and fewer slots when the frame would not give two blocks per SM; staged rows fill up to 4096 pixels.
constexpr int kHistCols = 4096;

void choose_hist_block(BGSParams &q, int nb, int gw, int gh) {
    const int S = q.S;
    int cslots = std::max(1, std::min(256 / nb, kHistCols / S));
    const int64_t min_blocks = 2 * (int64_t)hb::sm_count();
    while (cslots > 1 && (int64_t)gh * ((gw + cslots - 1) / cslots) < min_blocks) cslots = (cslots + 1) / 2;
    int k = std::max(1, (256 + cslots * S - 1) / (cslots * S));
    while (k > 1 && (cslots * k * S > kHistCols || (size_t)cslots * k * nb * sizeof(float2) > 64 * 1024)) k--;
    q.cslots = cslots;
    q.cpb = cslots * k;
    q.rows_chunk = std::max(1, std::min(S, kHistCols / (q.cpb * S)));
    q.cell_stride = (q.rows_chunk * S) | 1;
}

size_t hist_s_bytes(const BGSParams &q, int nb) {
    return ((size_t)q.cpb * nb + (size_t)q.cpb * q.cell_stride) * sizeof(float2);
}

// ---- trilinear slice + normalise for any S -----------------------------------------------------------------------
// One block = 256 threads over a tile of 4 * tx x th pixels; the ncx x ncy cells (x nz planes x 2 channels) its pixels
// interpolate between are staged once in shared memory as [z][cell row][cell column] float2.  Thread (c, r) owns the 4
// pixels at tile column 4c and rows r, r + 256 / tx, ...: float4 in / float4 out where aligned.  Cell index and
// fraction come from the offset within the tile (floor division by S via a magic multiplier, see kMagShift), never from
// a per-pixel division.  Bank conflicts: lanes whose corners fall in one cell read one address when their planes agree
// (a broadcast) and, with an odd plane stride, different banks when the planes differ by less than 16; lanes in
// different cells can still collide when the data puts them on different planes.
__global__ void __launch_bounds__(256) bg_slice_s_kernel(BGParams p, BGSParams q) {
    extern __shared__ float2 s_cells[];  // [nz][plane], plane >= ncy * ncx
    const int tid = threadIdx.x, S = q.S;
    const int X0 = (p.out_x0 & ~3) + blockIdx.y * (4 * q.tx), Y0 = p.out_y0 + blockIdx.x * q.th;
    const int cxl = floor_div_dev(X0, S), cyl = floor_div_dev(Y0, S);  // first cell of the tile (absolute)
    const int rx0 = X0 - cxl * S, ry0 = Y0 - cyl * S;                   // tile origin within that cell, [0, S)
    {
        const float2 *g = reinterpret_cast<const float2 *>(p.grid_b);
        const int ncells = q.ncx * q.ncy;
        // plane fastest: a cell's planes are contiguous in HBM, and an odd plane stride spreads them over the banks
        for (int it = tid; it < ncells * p.nz; it += 256) {
            const int cell = it / p.nz, z = it - cell * p.nz;
            const int cr = cell / q.ncx, cc = cell - cr * q.ncx;
            const int cx = min(max(cxl + cc - p.gx0, 0), p.gw - 1), cy = min(max(cyl + cr - p.gy0, 0), p.gh - 1);
            s_cells[z * q.plane + cell] = __ldg(g + ((size_t)cy * p.gw + cx) * p.nz + z);
        }
    }
    __syncthreads();
    const int c = tid % q.tx, rows_pass = 256 / q.tx;
    const int x = X0 + 4 * c;
    if (x + 3 < p.out_x0 || x >= p.out_x0 + p.W) return;
    int xi[4];
    float xf[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t n = (uint32_t)(rx0 + 4 * c + i);
        xi[i] = (int)((n * q.mag) >> kMagShift);  // cell column within the tile
        xf[i] = __fmul_rn((float)((int)n - xi[i] * S), q.inv_s);
    }
    for (int r = tid / q.tx; r < q.th; r += rows_pass) {
        const int y = Y0 + r;
        if (y >= p.out_y0 + p.H) break;
        const uint32_t n = (uint32_t)(ry0 + r);
        const int yi = (int)((n * q.mag) >> kMagShift);
        const float yf = __fmul_rn((float)((int)n - yi * S), q.inv_s);
        const float2 *crow = s_cells + yi * q.ncx;  // cell row yi of plane 0
        const float *ip = p.in + (int64_t)(y - p.in_y0) * p.in_sy + (x - p.in_x0);
        float *op = p.out + (int64_t)(y - p.out_y0) * p.out_sy + (x - p.out_x0);
        auto px = [&](float raw, int i) -> float {
            const float val = hl::clamp01(raw);
            const float zv = __fmul_rn(val, p.inv_r);
            int zi = (int)zv;
            const float zf = __fsub_rn(zv, (float)zi);
            zi = min(zi, p.nz - 2);
            const float2 *e = crow + zi * q.plane + xi[i];
            const int P = q.plane, R = q.ncx;
            const float2 a0 = e[0], b0 = e[1], d0 = e[R], e0 = e[R + 1];
            const float2 a1 = e[P], b1 = e[P + 1], d1 = e[P + R], e1 = e[P + R + 1];
            // lerp nest x -> y -> z exactly as generator :59-64
            const float v0 = hl::lerpf(hl::lerpf(hl::lerpf(a0.x, b0.x, xf[i]), hl::lerpf(d0.x, e0.x, xf[i]), yf),
                                       hl::lerpf(hl::lerpf(a1.x, b1.x, xf[i]), hl::lerpf(d1.x, e1.x, xf[i]), yf), zf);
            const float v1 = hl::lerpf(hl::lerpf(hl::lerpf(a0.y, b0.y, xf[i]), hl::lerpf(d0.y, e0.y, xf[i]), yf),
                                       hl::lerpf(hl::lerpf(a1.y, b1.y, xf[i]), hl::lerpf(d1.y, e1.y, xf[i]), yf), zf);
            return __fdiv_rn(v0, v1);
        };
        const bool full = x >= p.out_x0 && x + 3 < p.out_x0 + p.W;
        if (full && ((reinterpret_cast<uintptr_t>(ip) | reinterpret_cast<uintptr_t>(op)) & 15) == 0) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(ip));
            float4 o;
            o.x = px(v.x, 0);
            o.y = px(v.y, 1);
            o.z = px(v.z, 2);
            o.w = px(v.w, 3);
            *reinterpret_cast<float4 *>(op) = o;
        } else {
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if (x + i >= p.out_x0 && x + i < p.out_x0 + p.W) op[i] = px(__ldg(ip + i), i);
            }
        }
    }
}

// Slice tile for cell size S and nz planes: the widest, tallest tile (up to four row passes) whose staged cells fit
// kSliceBudget bytes, so that two blocks share an SM; failing that, the single-pass tile with the most pixels (busy
// threads) that fits the opt-in maximum (S = 1 with 200 bins).  A tile of 4 x 1 pixels (5 x 2 cells) always fits.
constexpr int kSliceBudget = 112 * 1024, kSliceMaxSmem = 227 * 1024;

size_t slice_s_bytes(const BGSParams &q, int nz) {
    return (size_t)q.plane * nz * sizeof(float2);
}

void choose_slice_tile(BGSParams &q, int nz) {
    auto set = [&](int tx, int th) {
        q.tx = tx; q.th = th;
        q.ncx = (4 * tx - 1 + q.S - 1) / q.S + 2;  // floor((X0 + 4tx - 1) / S) - floor(X0 / S) + 2 at most
        q.ncy = (th - 1 + q.S - 1) / q.S + 2;
        q.plane = (q.ncx * q.ncy) | 1;
        return slice_s_bytes(q, nz);
    };
    for (int passes = 4; passes >= 1; passes >>= 1) {
        for (int tx = 32; tx >= 1; tx >>= 1) {
            if (set(tx, passes * (256 / tx)) <= (size_t)kSliceBudget) return;
        }
    }
    int best_tx = 1, best_th = 1;  // else the single-pass tile covering the most pixels within the opt-in maximum
    for (int tx = 32; tx >= 1; tx >>= 1) {
        for (int th = 256 / tx; th >= 1; th--) {
            if (set(tx, th) <= (size_t)kSliceMaxSmem) {
                if (tx * th > best_tx * best_th) best_tx = tx, best_th = th;
                break;
            }
        }
    }
    set(best_tx, best_th);
}

int64_t est_i[2][2] = {{0, 1536}, {0, 2560}};
const int64_t *const est_ptrs[4] = {&est_i[0][0], &est_i[0][1], &est_i[1][0], &est_i[1][1]};
const halide_scalar_value_t sv_rsigma = hb::scalar_f32(0.1f);
const halide_filter_argument_t kArgs[3] = {
    {"input", halide_argument_kind_input_buffer, 2, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
    {"r_sigma", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv_rsigma, nullptr},
    {"bilateral_grid", halide_argument_kind_output_buffer, 2, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
};

inline int fdiv(int a, int b) {  // floor division, b > 0
    int q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

// bilateral_grid with cell size s_sigma (the generator's GeneratorParam): the shipped S runs bg_hist_blurz, bg_blur_xy
// and bg_slice; every other cell size runs bg_hist_blurz_s, bg_blur_xy and bg_slice_s.
int run_bilateral_grid(halide_buffer_t *input, int s_sigma, float r_sigma, halide_buffer_t *output) {
    int r;
    hb::Arg args[2] = {{input, kArgs[0]}, {output, kArgs[2]}};
    if ((r = hb::check_args(args, 2))) return r;
    // the slice reads input(x,y) unclamped (generator :50): the input must cover the output region
    const hb::Region need[2] = {hb::region_of(output, true), hb::region_of(output, false)};
    if (hb::answer_bounds_query(args, need, 2)) return 0;
    if ((r = hb::check_shapes(args, 2)) || (r = hb::check_required(args, need, 2))) return r;
    const int W = output->dim[0].extent, H = output->dim[1].extent;
    if (W <= 0 || H <= 0) return 0;
    if (s_sigma < 1 || s_sigma > 128) {
        return hb::fail(s_sigma < 1 ? halide_error_code_param_too_small : halide_error_code_param_too_large,
                        "Parameter s_sigma is %d but must be in [1, 128]", (int)s_sigma);
    }
    if (!(r_sigma > 0.0f)) {
        return hb::fail(halide_error_code_param_too_small, "Parameter r_sigma is %g but must be positive", (double)r_sigma);
    }
    BGParams p;
    p.inv_r = 1.0f / r_sigma;
    p.zmax = (int)(1.0f * p.inv_r + 0.5f);
    p.nz = p.zmax + 2;
    const size_t bins_bytes = (size_t)(p.zmax + 1) * 2 * 128 * sizeof(float);
    if (bins_bytes > 200 * 1024) {
        return hb::fail(halide_error_code_param_too_small,
                        "Parameter r_sigma is %g: more than %d intensity bins are not supported by this build",
                        (double)r_sigma, (int)(200 * 1024 / (2 * 128 * sizeof(float))));
    }
    if ((r = hb::acquire(args, 2))) return r;

    const int ox = output->dim[0].min, oy = output->dim[1].min;
    p.in = (const float *)args[0].dev;
    p.in_sy = input->dim[1].stride;
    p.in_x0 = input->dim[0].min; p.in_y0 = input->dim[1].min;
    p.in_w = input->dim[0].extent; p.in_h = input->dim[1].extent;
    p.out = (float *)args[1].dev;
    p.out_sy = output->dim[1].stride;
    p.out_x0 = ox; p.out_y0 = oy; p.W = W; p.H = H;
    // cells the slice touches are xi..xi+1; blury/blurx add 2 cells on every side
    p.gx0 = fdiv(ox, s_sigma) - 2;
    p.gy0 = fdiv(oy, s_sigma) - 2;
    p.gw = fdiv(ox + W - 1, s_sigma) + 1 + 2 - p.gx0 + 1;
    p.gh = fdiv(oy + H - 1, s_sigma) + 1 + 2 - p.gy0 + 1;
    hb::Scratch scratch;
    const size_t gelems = (size_t)p.gw * p.gh * p.nz * 2;
    p.grid_a = scratch.get<float>(gelems);
    p.grid_b = scratch.get<float>(gelems);
    if (!p.grid_a || !p.grid_b) return hb::fail(halide_error_code_device_malloc_failed, "bilateral_grid: scratch allocation failed");

    cudaStream_t s = hb::stream();
    {
        hb::CallTimer timer(s);
        BGSParams q;  // (the any-S kernels' shapes)
        if (s_sigma == S) {
            hb::allow_smem(bg_hist_blurz_kernel, bins_bytes);
            dim3 g1((p.gw + 63) / 64, p.gh);
            HB_LAUNCH("bg_hist_blurz", bg_hist_blurz_kernel, g1, 128, bins_bytes, s, p);
        } else {
            q.S = s_sigma;
            q.inv_s = (float)(1.0 / (double)s_sigma);
            q.mag = (uint32_t)(((1u << kMagShift) + s_sigma - 1) / s_sigma);
            choose_slice_tile(q, p.nz);
            choose_hist_block(q, p.zmax + 1, p.gw, p.gh);
            const size_t hist_bytes = hist_s_bytes(q, p.zmax + 1);
            hb::allow_smem(bg_hist_blurz_s_kernel, hist_bytes);
            dim3 g1(p.gh, (p.gw + q.cpb - 1) / q.cpb);
            HB_LAUNCH("bg_hist_blurz_s", bg_hist_blurz_s_kernel, g1, 256, hist_bytes, s, p, q);
        }
        const int V = p.nz * 2;
        const int cols = (p.gw - 4) * V;
        const int64_t min_blocks = (int64_t)hb::sm_count() * 4;
        int rows = 16;
        while (rows > 2 && (int64_t)((cols + 255) / 256) * ((p.gh - 4 + rows - 1) / rows) < min_blocks) rows >>= 1;
        dim3 g2((cols + 255) / 256, (p.gh - 4 + rows - 1) / rows);
        HB_LAUNCH("bg_blur_xy", bg_blur_xy_kernel, g2, 256, 0, s, p, rows);
        if (s_sigma == S) {
            const int tx0 = ox & ~(S - 1), ty0 = oy & ~(S - 1);
            dim3 g3((ox + W - tx0 + kSliceW - 1) / kSliceW, (oy + H - ty0 + S - 1) / S);
            const size_t slice_smem = (size_t)p.nz * 2 * kSlicePitch * sizeof(float2);
            hb::allow_smem(bg_slice_kernel, slice_smem);
            HB_LAUNCH("bg_slice", bg_slice_kernel, g3, dim3(32, 8), slice_smem, s, p);
        } else {
            const int tw = 4 * q.tx, tx0 = ox & ~3;
            dim3 g3((H + q.th - 1) / q.th, (ox + W - tx0 + tw - 1) / tw);
            const size_t slice_smem = slice_s_bytes(q, p.nz);
            hb::allow_smem(bg_slice_s_kernel, slice_smem);
            HB_LAUNCH("bg_slice_s", bg_slice_s_kernel, g3, 256, slice_smem, s, p, q);
        }
    }
    return hb::finish(args, 2, "bilateral_grid launch");
}

}  // namespace

extern "C" int bilateral_grid(halide_buffer_t *input, float r_sigma, halide_buffer_t *output) {
    return run_bilateral_grid(input, S, r_sigma, output);
}
HB_EXPORT_FILTER(bilateral_grid, kArgs)
HB_EXPORT_AUTO_SCHEDULE(bilateral_grid, kArgs)

// bilateral_grid with the s_sigma GeneratorParam as a run-time argument, in [1, 128].  S = 8 runs bilateral_grid's own
// kernels (bit for bit).  Buffer rules, error codes and the bounds query are bilateral_grid's.
extern "C" int halide_b200_bilateral_grid_s_sigma(halide_buffer_t *input, int32_t s_sigma, float r_sigma,
                                                  halide_buffer_t *output) {
    return run_bilateral_grid(input, s_sigma, r_sigma, output);
}
