// nl_means.cu — nl_means(input, patch_size, search_area, sigma, output) for sm_90a.
//
// Reference algorithm: apps/nl_means/nl_means_generator.cpp:24-63
//   d(x,y,dx,dy)  = sum_c (I(x,y,c) - I(x+dx,y+dy,c))^2            (clamped coordinates, c = 0..2)
//   blur_d        = box sum of d over the patch (y then x)
//   w             = fast_exp(blur_d * (-1 / (sigma^2 * patch^2)))
//   out_c         = clamp( sum_{dy,dx} w * I_c(x+dx,y+dy) / sum_{dy,dx} w , 0, 1 )
// Float pipeline, bit-exact against oracle/oracle_nl_means.cpp: both kernels perform its float operations in its order
// (d over channels 0..2, the box sums y then x, ascending, search rows outer and dx inner, the same fast_exp, an IEEE
// divide) and the library builds with --fmad=false (tests/test_nl_means_exact_gpu.py).
//
// Compute-bound (~1.5 kflop/px at patch 3 / search 7 against 24 algorithmic B/px): the frame is
// read once into a shared-memory tile with its (search/2 + patch/2) apron, then for each search row
// dy three phases run per block with the whole dx row batched between barriers:
//   A  d for all dx over the tile grown by the patch apron          -> smem D[dx][y][x]
//   B  vertical patch sums                                          -> smem V[dx][y][x]
//   C  horizontal patch sums, fast_exp, accumulate 4 running sums in registers (2 px per thread)
// halide_b200_nl_means_u8 runs the same kernels on uint8 frames: they take the frame's element type T as a template
// parameter and convert while they fill the float tile sI (hl::frame_to_f32) and in the final store (hl::frame_from_f32);
// the phases in between are the float path's.
//
// The batch and interleaved entry points run the same kernels too, with two more template parameters: IL (the frames are
// pixel-interleaved: the tile fill reads them in memory order and the final store writes a pixel's channels side by side)
// and FR (the grid's blocks walk the frames of a 4-D buffer, frame n = blockIdx.z, + gridDim.z, ...).  Only the fill of
// sI and the final store differ, and both kernels share them (fill_tile, store_rows); the phases, and so every float
// operation, are the planar one-frame kernels'.  Each kernel is one template; its parameter block is NLParamsOf<IL, FR>.
#include <algorithm>
#include <type_traits>

#include "hb_common.h"
#include "hl_math.cuh"

namespace {

constexpr int TX = 32, TY = 16;  // output tile per block; 256 threads, 2 rows per thread

struct NLParams {
    const float *in;  // element at input mins (a uint8_t frame's for the <uint8_t> kernels; a batch's: of the input frame
                      // that output frame 0 reads)
    int64_t in_sy, in_sc;
    int in_x0, in_y0, in_c0, in_w, in_h, in_c;
    float *out;       // (the same)
    int64_t out_sy, out_sc;
    int out_x0, out_y0, W, H;
    int p, s, p_lo, s_lo;  // patch/search extents and their first offsets (-(n/2))
    float inv_sigma_sq;
    int nd;                // dx offsets batched per pass
    int iw, ih;            // input tile extent (TX + p + s - 2, TY + p + s - 2)
    int dw, dh;            // D tile extent (TX + p - 1, TY + p - 1)
};
// The parameters of the IL and FR kernels: NLParams and, after it, the frame strides and pixel pitches.  (A separate
// type, so that the planar one-frame kernels keep their parameter block byte for byte: any field appended to it changes
// their code.)
struct NLVideoParams : NLParams {
    int64_t in_sn, out_sn;  // frame strides (FR kernels)
    int in_px, out_px;      // pixel pitches (IL kernels, whose channel strides in_sc / out_sc are 1)
    int N;                  // frames (FR kernels)
};
template<bool IL, bool FR>
using NLParamsOf = std::conditional_t<IL || FR, NLVideoParams, NLParams>;

// Frame n's input (the element at the input's x/y/c mins) and output (at the output's mins), formed where they are used;
// the one-frame kernels (FR false) read q.in and q.out there as they always did.
template<typename T, bool FR, typename Q>
__device__ __forceinline__ const T *frame_in(const Q &q, int n) {
    if constexpr (FR) return reinterpret_cast<const T *>(q.in) + n * q.in_sn;
    else return reinterpret_cast<const T *>(q.in);
}
template<typename T, bool FR, typename Q>
__device__ __forceinline__ T *frame_out(const Q &q, int n) {
    if constexpr (FR) return reinterpret_cast<T *>(q.out) + n * q.out_sn;
    else return reinterpret_cast<T *>(q.out);
}
template<bool FR, typename Q>
__device__ __forceinline__ int frames(const Q &q) {
    if constexpr (FR) return q.N;
    else return 1;
}

// The tile fill of both kernels: sI[c][v][u], three planes of npix = ih * iw floats, tile (u, v) at absolute
// (ax0 + u, ay0 + v), from frame n with every coordinate clamped to the input.  The window kernel passes constant
// extents, the generic kernel q.iw and q.ih: by reference, so that its planar fill reads them from the parameters at
// each use instead of holding them in registers across the loop (by value, its frame-walking instance compiles to
// other code).
// The IL fill's warp loads take the tile's samples in memory order, channel innermost (32 consecutive samples of a pixel
// row per load), and a warp shuffle hands each lane the three channels of one pixel, so that each store writes 32
// consecutive floats of one plane: storing the loaded samples directly would put the three channels of a pixel into one
// bank (npix is a multiple of 32 at patch 3 / search 7).
template<typename T, bool IL, bool FR, typename Q>
__device__ __forceinline__ void fill_tile(float *sI, const Q &q, int n, int tid, int ax0, int ay0, const int &iw,
                                          const int &ih) {
    if constexpr (IL) {
        const T *in = frame_in<T, FR>(q, n);
        const int npix = ih * iw, lane = tid & 31;
        for (int p0 = (tid >> 5) * 32; p0 < npix; p0 += 256) {  // (warp-uniform: every lane takes the shuffles)
            float smp[3];  // samples 3 * p0 + 32 * k + lane of the tile, pixel (that / 3), channel (that % 3)
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const int j = 3 * p0 + 32 * k + lane, pix = j / 3, c = j - 3 * pix;
                smp[k] = 0.f;
                if (pix < npix) {
                    const int v = pix / iw, u = pix - v * iw;
                    const int x = hl::clampi(ax0 + u, q.in_x0, q.in_x0 + q.in_w - 1) - q.in_x0;
                    const int y = hl::clampi(ay0 + v, q.in_y0, q.in_y0 + q.in_h - 1) - q.in_y0;
                    const int cc = hl::clampi(c, q.in_c0, q.in_c0 + q.in_c - 1) - q.in_c0;
                    smp[k] = hl::frame_to_f32(__ldg(in + (int64_t)y * q.in_sy + (int64_t)x * q.in_px + cc));
                }
            }
#pragma unroll
            for (int c = 0; c < 3; c++) {
                // Lane p takes sample 3p + c, held in smp[(3p + c) / 32] of lane (3p + c) % 32.  This lane holds it for
                // the one p with 3p + c == lane (mod 32), p = 11 (lane - c) mod 32 (3 * 11 == 1 mod 32), and sends that
                // register.
                const int p = ((lane - c) * 11) & 31, k = (3 * p + c) >> 5;
                const float send = k == 0 ? smp[0] : (k == 1 ? smp[1] : smp[2]);
                const float got = __shfl_sync(0xffffffffu, send, (3 * lane + c) & 31);
                if (p0 + lane < npix) sI[c * npix + p0 + lane] = got;
            }
        }
    } else {
        for (int t = tid; t < 3 * ih * iw; t += 256) {
            const int c = t / (ih * iw), rem = t - c * ih * iw;
            const int v = rem / iw, u = rem - v * iw;
            const int x = hl::clampi(ax0 + u, q.in_x0, q.in_x0 + q.in_w - 1) - q.in_x0;
            const int y = hl::clampi(ay0 + v, q.in_y0, q.in_y0 + q.in_h - 1) - q.in_y0;
            const int cc = hl::clampi(c, q.in_c0, q.in_c0 + q.in_c - 1) - q.in_c0;
            sI[t] = hl::frame_to_f32(__ldg(frame_in<T, FR>(q, n) + (int64_t)cc * q.in_sc + (int64_t)y * q.in_sy + x));
        }
    }
}

// The final store of both kernels: a thread's two output pixels of frame n (column tx, rows ty and ty + 8 of the block's
// tile), each the four running sums acc[r] normalised and clamped.
template<typename T, bool IL, bool FR, typename Q>
__device__ __forceinline__ void store_rows(const Q &q, int n, const float (&acc)[2][4], int tx, int ty) {
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int lx = blockIdx.x * TX + tx, ly = blockIdx.y * TY + ty + 8 * r;
        if (lx < q.W && ly < q.H) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                // (NaN -> 1: every weight is NaN when sigma^2 * patch^2 underflows and -1 / it is -inf)
                const float v = hl::clamp01(__fdiv_rn(acc[r][c], acc[r][3]));
                T *out = frame_out<T, FR>(q, n);
                if constexpr (IL) out[(int64_t)ly * q.out_sy + (int64_t)lx * q.out_px + c] = hl::frame_from_f32<T>(v);
                else out[(int64_t)c * q.out_sc + (int64_t)ly * q.out_sy + lx] = hl::frame_from_f32<T>(v);
            }
        }
    }
}

// nl_means_kernel on frame n.
template<typename T, bool IL, bool FR, typename Q>
__device__ __forceinline__ void nl_means_frame(const Q &q, int n) {
    extern __shared__ float smem[];
    float *sI = smem;                              // [3][ih][iw]
    float *sD = sI + 3 * q.ih * q.iw;              // [nd][dh][dw]
    float *sV = sD + q.nd * q.dh * q.dw;           // [nd][TY][dw]
    const int tid = FR ? hl::frame_tid() : (int)threadIdx.x;
    const int X0 = q.out_x0 + blockIdx.x * TX, Y0 = q.out_y0 + blockIdx.y * TY;
    // tile coordinate (u,v) <-> absolute (X0 + p_lo + s_lo + u, Y0 + p_lo + s_lo + v)
    const int ax0 = X0 + q.p_lo + q.s_lo, ay0 = Y0 + q.p_lo + q.s_lo;
    fill_tile<T, IL, FR>(sI, q, n, tid, ax0, ay0, q.iw, q.ih);
    __syncthreads();
    const int plane = q.ih * q.iw;
    const int tx = tid & 31, ty = tid >> 5;  // rows ty and ty + 8
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    const int off_s = -q.s_lo;               // tile offset of search offset 0
    for (int dyi = 0; dyi < q.s; dyi++) {
        for (int dx0 = 0; dx0 < q.s; dx0 += q.nd) {
            const int nd = min(q.nd, q.s - dx0);
            // ---- phase A: D[j][v][u] = d(X0 + p_lo + u, Y0 + p_lo + v, dx, dy), dx = s_lo + dx0 + j
            for (int t = tid; t < q.dh * q.dw; t += 256) {
                int v = t / q.dw, u = t - v * q.dw;
                const float *a = sI + (v + off_s) * q.iw + (u + off_s);
                const float *b = sI + (v + dyi) * q.iw + (u + dx0);
                const float a0 = a[0], a1 = a[plane], a2 = a[2 * plane];
                for (int j = 0; j < nd; j++) {
                    float e0 = a0 - b[j], e1 = a1 - b[plane + j], e2 = a2 - b[2 * plane + j];
                    sD[j * q.dh * q.dw + t] = ((0.0f + e0 * e0) + e1 * e1) + e2 * e2;
                }
            }
            __syncthreads();
            // ---- phase B: V[j][y][u] = sum_{t<p} D[j][y + t][u]
            for (int t = tid; t < TY * q.dw; t += 256) {
                int y = t / q.dw, u = t - y * q.dw;
                for (int j = 0; j < nd; j++) {
                    const float *d = sD + (j * q.dh + y) * q.dw + u;
                    float sum = 0.f;
                    for (int k = 0; k < q.p; k++) sum += d[k * q.dw];
                    sV[j * TY * q.dw + t] = sum;
                }
            }
            __syncthreads();
            // ---- phase C: horizontal sums, weights, accumulation
            for (int j = 0; j < nd; j++) {
#pragma unroll
                for (int r = 0; r < 2; r++) {
                    int y = ty + 8 * r;
                    const float *vrow = sV + (j * TY + y) * q.dw + tx;
                    float bd = 0.f;
                    for (int k = 0; k < q.p; k++) bd += vrow[k];
                    float w = hl::fast_exp(bd * q.inv_sigma_sq);
                    const float *nb = sI + (y - q.p_lo + dyi) * q.iw + (tx - q.p_lo + dx0 + j);
                    acc[r][0] += w * nb[0];
                    acc[r][1] += w * nb[plane];
                    acc[r][2] += w * nb[2 * plane];
                    acc[r][3] += w;
                }
            }
            // phase A of the next pass overwrites sD only (phase C reads sV and sI): one barrier is
            // enough between C and the next B, and the A->B barrier above provides it.
        }
    }
    store_rows<T, IL, FR>(q, n, acc, tx, ty);
}
// (The planar one-frame instances call the frame body directly: through the one-iteration frame loop they compile to
// longer code.)
template<typename T, bool IL, bool FR>
__global__ void __launch_bounds__(256) nl_means_kernel(NLParamsOf<IL, FR> q) {
    if constexpr (!IL && !FR) {
        nl_means_frame<T, false, false>(q, 0);
    } else {
        for (int n = FR ? blockIdx.z : 0; n < frames<FR>(q); n += FR ? gridDim.z : 1) {
            if (n != (int)blockIdx.z) __syncthreads();  // the previous frame's last phase C may still read sI
            nl_means_frame<T, IL, FR>(q, n);
        }
    }
}

// ---- register-window version for compile-time patch / search sizes ------------------------------------------------
// The kernel above is generic in patch and search size: every tile coordinate costs an integer division by a run-time
// extent, d goes through shared memory twice (D, then V) and the loops cannot unroll — ~165 instructions per pixel and
// search offset.  With P and S fixed at compile time:
//   phase 1: a thread owns one column u of one search offset dx and walks down the tile's TY + P - 1 rows; d of the new
//            row comes from six shared loads (three channels of the centre and of the shifted tile), the vertical patch
//            sum is the explicit ascending sum over a register window ((0 + d0) + d1) + ... — the reference's order —
//            and only V is written to shared memory;
//   phase 2: as before (horizontal patch sum, fast_exp, four running sums per pixel, two rows per thread), unrolled.
// All S offsets of a search row are batched between two barriers.  Same float operations in the same order as the
// generic kernel (results are bit-identical to it; tests/test_nl_means_gpu.py runs both against the oracle).
// (A frame's last search row ends in a barrier after its last read of sI and sV: the next frame's fill needs no other.)
template<typename T, int P, int S, bool IL, bool FR, typename Q>
__device__ __forceinline__ void nl_means_window_frame(const Q &q, int n) {
    constexpr int IW = TX + P + S - 2, IH = TY + P + S - 2, DW = TX + P - 1, DH = TY + P - 1, PLANE = IH * IW;
    constexpr int PLO = -(P / 2), SLO = -(S / 2), OFFS = -SLO;
    extern __shared__ float smem[];
    float *sI = smem;             // [3][IH][IW]
    float *sV = sI + 3 * PLANE;   // [S][TY][DW]
    const int tid = FR ? hl::frame_tid() : (int)threadIdx.x;
    const int X0 = q.out_x0 + blockIdx.x * TX, Y0 = q.out_y0 + blockIdx.y * TY;
    const int ax0 = X0 + PLO + SLO, ay0 = Y0 + PLO + SLO;  // tile (u, v) <-> absolute (ax0 + u, ay0 + v)
    fill_tile<T, IL, FR>(sI, q, n, tid, ax0, ay0, IW, IH);
    __syncthreads();
    const int tx = tid & 31, ty = tid >> 5;  // rows ty and ty + 8
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    for (int dyi = 0; dyi < S; dyi++) {
        // ---- phase 1: V[j][y][u] = sum_{k<P} d(u, y + k) for search offset (SLO + j, SLO + dyi)
        for (int it = tid; it < DW * S; it += 256) {
            const int j = it / DW, u = it - j * DW;
            const float *a = sI + OFFS * IW + (u + OFFS);   // centre pixel of d: tile row v + OFFS
            const float *b = sI + dyi * IW + (u + j);       // shifted pixel:     tile row v + dyi
            float *vout = sV + j * TY * DW + u;
            float win[P];
#pragma unroll
            for (int v = 0; v < DH; v++) {
                const float e0 = a[v * IW] - b[v * IW], e1 = a[PLANE + v * IW] - b[PLANE + v * IW],
                            e2 = a[2 * PLANE + v * IW] - b[2 * PLANE + v * IW];
                win[v % P] = ((0.0f + e0 * e0) + e1 * e1) + e2 * e2;
                if (v >= P - 1) {
                    float sum = 0.f;
#pragma unroll
                    for (int k = 0; k < P; k++) sum += win[(v - (P - 1) + k) % P];  // rows y .. y + P - 1, ascending
                    vout[(v - (P - 1)) * DW] = sum;
                }
            }
        }
        __syncthreads();
        // ---- phase 2: horizontal sums, weights, accumulation
#pragma unroll
        for (int j = 0; j < S; j++) {
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const int y = ty + 8 * r;
                const float *vrow = sV + (j * TY + y) * DW + tx;
                float bd = 0.f;
#pragma unroll
                for (int k = 0; k < P; k++) bd += vrow[k];
                const float w = hl::fast_exp(bd * q.inv_sigma_sq);
                const float *nb = sI + (y - PLO + dyi) * IW + (tx - PLO + j);
                acc[r][0] += w * nb[0];
                acc[r][1] += w * nb[PLANE];
                acc[r][2] += w * nb[2 * PLANE];
                acc[r][3] += w;
            }
        }
        __syncthreads();  // (the next search row's phase 1 overwrites sV)
    }
    store_rows<T, IL, FR>(q, n, acc, tx, ty);
}
// The uint8 IL kernels are held to 8 blocks per SM, which the planar kernels reach with 32 registers: left to itself the
// compiler gives them 40, room for 6 blocks, and the interleaved call at 3/7 takes 1.08x the planar one's time at 4K
// instead of 1.06x.  The same bound on the other kernels, which take 32 registers anyway, slows them by 2-3 %; for them
// the minimum of 0 blocks leaves the compiler free, as the one-argument form does.
template<typename T, int P, int S, bool IL, bool FR>
__global__ void __launch_bounds__(256, IL && sizeof(T) == 1 ? 8 : 0) nl_means_window_kernel(NLParamsOf<IL, FR> q) {
    if constexpr (!IL && !FR) {
        nl_means_window_frame<T, P, S, false, false>(q, 0);
    } else {
        for (int n = FR ? blockIdx.z : 0; n < frames<FR>(q); n += FR ? gridDim.z : 1) {
            nl_means_window_frame<T, P, S, IL, FR>(q, n);
        }
    }
}
template<int P, int S>
constexpr size_t nl_window_smem() {
    return (size_t)(3 * (TY + P + S - 2) * (TX + P + S - 2) + S * TY * (TX + P - 1)) * sizeof(float);
}

int g_variant = 0;  // test hook (halide_b200_nl_means_variant): 1 = generic kernel for every patch / search size

int64_t est_i[3][2] = {{0, 1536}, {0, 2560}, {0, 3}};
const int64_t *const est_ptrs[6] = {&est_i[0][0], &est_i[0][1], &est_i[1][0], &est_i[1][1], &est_i[2][0], &est_i[2][1]};
const halide_scalar_value_t sv_patch = hb::scalar_i32(7), sv_search = hb::scalar_i32(7), sv_sigma = hb::scalar_f32(0.12f);
const halide_filter_argument_t kArgs[5] = {
    {"input", halide_argument_kind_input_buffer, 3, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
    {"patch_size", halide_argument_kind_input_scalar, 0, {halide_type_int, 32, 0}, nullptr, nullptr, nullptr, &sv_patch, nullptr},
    {"search_area", halide_argument_kind_input_scalar, 0, {halide_type_int, 32, 0}, nullptr, nullptr, nullptr, &sv_search, nullptr},
    {"sigma", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv_sigma, nullptr},
    {"non_local_means", halide_argument_kind_output_buffer, 3, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
};
// halide_b200_nl_means_u8: the same buffers in uint8.
const halide_filter_argument_t kU8Args[2] = {hb::variant(kArgs[0], 0, hb::kU8), hb::variant(kArgs[4], 0, hb::kU8)};
// The batch entry points: the same buffers with a fourth dimension, the frame index n (float32, then uint8).  The
// interleaved entry points use these records and the ones above with hb::Arg::interleaved set.
const halide_filter_argument_t kBatchArgs[2] = {hb::variant(kArgs[0], 1), hb::variant(kArgs[4], 1)};
const halide_filter_argument_t kU8BatchArgs[2] = {hb::variant(kArgs[0], 1, hb::kU8), hb::variant(kArgs[4], 1, hb::kU8)};

// The one launch of a call: the register-window kernel at patch / search 3/7 and 7/7 (unless the variant hook asks for
// the generic one), else the generic kernel.
template<typename T, bool IL, bool FR>
void launch(const NLVideoParams &v, dim3 grid, size_t smem, cudaStream_t s) {
    const NLParamsOf<IL, FR> &q = v;
    const bool window = g_variant != 1;
    if (window && q.p == 3 && q.s == 7) {
        constexpr size_t sm = nl_window_smem<3, 7>();
        static_assert(sm <= 48 * 1024, "no opt-in needed");
        HB_LAUNCH("nl_means_window", (nl_means_window_kernel<T, 3, 7, IL, FR>), grid, 256, sm, s, q);
    } else if (window && q.p == 7 && q.s == 7) {
        constexpr size_t sm = nl_window_smem<7, 7>();
        static_assert(sm <= 48 * 1024, "no opt-in needed");
        HB_LAUNCH("nl_means_window", (nl_means_window_kernel<T, 7, 7, IL, FR>), grid, 256, sm, s, q);
    } else {
        auto kernel = nl_means_kernel<T, IL, FR>;
        hb::allow_smem(kernel, smem);
        HB_LAUNCH("nl_means", kernel, grid, 256, smem, s, q);
    }
}

// Every nl_means entry point, on args = {input, output} of element type T (float, or uint8_t for the 8-bit ones): 3-D
// (x, y, c) buffers for one frame, 4-D (x, y, c, n) for a batch; args[*].interleaved selects the pixel-interleaved layout.
template<typename T>
int run_nl_means(hb::Arg *args, int32_t patch_size, int32_t search_area, float sigma, const char *what) {
    int r;
    if ((r = hb::check_args(args, 2))) return r;
    halide_buffer_t *input = args[0].b, *output = args[1].b;
    const hb::Clip c = hb::clip_of(args[0], args[1], 3);
    const bool il = args[0].interleaved;
    // every input access is clamped in x, y and c: a query is answered with the output's x/y region, 3 channels and (a
    // batch) the output's frames
    const hb::Region region =
        c.with_frames({{output->dim[0].min, output->dim[1].min, 0}, {output->dim[0].extent, output->dim[1].extent, 3}, false});
    const hb::Region need[2] = {region, region};
    if (hb::answer_bounds_query(args, need, 2)) return 0;
    if ((r = hb::check_shapes(args, 2))) return r;
    // explicit constraint: non_local_means.dim(2).set_bounds(0, 3) (generator :68)
    if (output->dim[2].min != 0 || output->dim[2].extent != 3) {
        return hb::fail(halide_error_code_constraint_violated,
                        "Constraint violated: non_local_means.min.2 (%d) == 0 and non_local_means.extent.2 (%d) == 3",
                        output->dim[2].min, output->dim[2].extent);
    }
    const int W = output->dim[0].extent, H = output->dim[1].extent, N = c.N;
    if (W <= 0 || H <= 0 || N <= 0) return 0;
    if (input->dim[0].extent <= 0 || input->dim[1].extent <= 0 || input->dim[2].extent <= 0) {
        return hb::fail(halide_error_code_access_out_of_bounds, "Input buffer input is empty");
    }
    // output frame n reads input frame n, which is not clamped: the input's frames must cover the output's
    const hb::Region frames = c.with_frames({{}, {}, true});  // (extents of 0: x, y and c are not checked)
    if ((r = hb::check_required(args, &frames, 1))) return r;
    if (patch_size < 1 || search_area < 1 || patch_size > 31 || search_area > 63) {
        return hb::fail(patch_size < 1 || search_area < 1 ? halide_error_code_param_too_small : halide_error_code_param_too_large,
                        "nl_means: patch_size %d / search_area %d outside the supported range [1,31] / [1,63]", patch_size,
                        search_area);
    }
    if ((r = hb::acquire(args, 2))) return r;

    NLVideoParams q;
    q.in = (const float *)((const T *)args[0].dev + c.in_off);  // the input frame output frame 0 reads
    q.in_sy = input->dim[1].stride; q.in_sc = input->dim[2].stride;
    q.in_x0 = input->dim[0].min; q.in_y0 = input->dim[1].min; q.in_c0 = input->dim[2].min;
    q.in_w = input->dim[0].extent; q.in_h = input->dim[1].extent; q.in_c = input->dim[2].extent;
    q.out = (float *)args[1].dev;
    q.out_sy = output->dim[1].stride; q.out_sc = output->dim[2].stride;
    q.out_x0 = output->dim[0].min; q.out_y0 = output->dim[1].min; q.W = W; q.H = H;
    q.p = patch_size; q.s = search_area;
    q.p_lo = -(patch_size / 2); q.s_lo = -(search_area / 2);
    // inv_sigma_sq = -1.0f / (sigma * sigma * patch_size * patch_size) (generator :24)
    q.inv_sigma_sq = -1.0f / (((sigma * sigma) * (float)patch_size) * (float)patch_size);
    q.iw = TX + patch_size + search_area - 2; q.ih = TY + patch_size + search_area - 2;
    q.dw = TX + patch_size - 1; q.dh = TY + patch_size - 1;
    q.in_px = input->dim[0].stride; q.out_px = output->dim[0].stride;
    q.in_sn = c.in_sn;
    q.out_sn = c.out_sn;
    q.N = N;
    const size_t fixed = (size_t)3 * q.iw * q.ih * sizeof(float);
    const size_t per_dx = (size_t)(q.dh + TY) * q.dw * sizeof(float);
    const size_t budget = 100 * 1024;
    int nd = search_area;
    while (nd > 1 && fixed + nd * per_dx > budget) nd--;
    q.nd = nd;
    const size_t smem = fixed + nd * per_dx;
    if (smem > 220 * 1024) {
        return hb::fail(halide_error_code_param_too_large, "nl_means: patch/search sizes need %zu bytes of shared memory", smem);
    }
    cudaStream_t s = hb::stream();
    {
        hb::CallTimer timer(s);
        dim3 grid((W + TX - 1) / TX, (H + TY - 1) / TY, std::min(N, hb::kMaxGridZ));
        if (il && c.clip) launch<T, true, true>(q, grid, smem, s);
        else if (il) launch<T, true, false>(q, grid, smem, s);
        else if (c.clip) launch<T, false, true>(q, grid, smem, s);
        else launch<T, false, false>(q, grid, smem, s);
    }
    return hb::finish(args, 2, what);
}
}  // namespace

extern "C" void halide_b200_nl_means_variant(int v) {
    g_variant = v;
}

extern "C" int nl_means(halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kArgs[0]}, {output, kArgs[4]}};
    return run_nl_means<float>(args, patch_size, search_area, sigma, "nl_means launch");
}
HB_EXPORT_FILTER(nl_means, kArgs)
HB_EXPORT_AUTO_SCHEDULE(nl_means, kArgs)

// 8-bit entry point (library extension): out8 = to_u8(nl_means(to_f32(in8), patch_size, search_area, sigma)) bit for
// bit, with the reference's element conversions (to_f32(v) = v / 255.0f, to_u8(f) = lround(f * 255.0f)) done inside the
// kernels.  Buffer rules (channels clamped, the output's channels [0, 3)), parameter checks, error codes, the bounds query
// and the variant hook are nl_means'.
extern "C" int halide_b200_nl_means_u8(halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                                       halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8Args[0]}, {output, kU8Args[1]}};
    return run_nl_means<uint8_t>(args, patch_size, search_area, sigma, "nl_means_u8 launch");
}

// Batch and interleaved entry points (library extensions): nl_means / nl_means_u8 on every frame of a 4-D (x, y, c, n)
// buffer in one launch, and on pixel-interleaved buffers (dim[2].stride == 1, dim[0].stride = the pixel pitch, at least
// the channel extent), bit for bit what the planar one-frame entry points give frame by frame on planar copies.
extern "C" int halide_b200_nl_means_batch(halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                                          halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kBatchArgs[0]}, {output, kBatchArgs[1]}};
    return run_nl_means<float>(args, patch_size, search_area, sigma, "nl_means_batch launch");
}
extern "C" int halide_b200_nl_means_interleaved(halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                                                halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kArgs[0], nullptr, true}, {output, kArgs[4], nullptr, true}};
    return run_nl_means<float>(args, patch_size, search_area, sigma, "nl_means_interleaved launch");
}
extern "C" int halide_b200_nl_means_interleaved_batch(halide_buffer_t *input, int32_t patch_size, int32_t search_area,
                                                      float sigma, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kBatchArgs[0], nullptr, true}, {output, kBatchArgs[1], nullptr, true}};
    return run_nl_means<float>(args, patch_size, search_area, sigma, "nl_means_interleaved_batch launch");
}
extern "C" int halide_b200_nl_means_u8_batch(halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                                             halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8BatchArgs[0]}, {output, kU8BatchArgs[1]}};
    return run_nl_means<uint8_t>(args, patch_size, search_area, sigma, "nl_means_u8_batch launch");
}
extern "C" int halide_b200_nl_means_u8_interleaved(halide_buffer_t *input, int32_t patch_size, int32_t search_area,
                                                   float sigma, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8Args[0], nullptr, true}, {output, kU8Args[1], nullptr, true}};
    return run_nl_means<uint8_t>(args, patch_size, search_area, sigma, "nl_means_u8_interleaved launch");
}
extern "C" int halide_b200_nl_means_u8_interleaved_batch(halide_buffer_t *input, int32_t patch_size, int32_t search_area,
                                                         float sigma, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8BatchArgs[0], nullptr, true}, {output, kU8BatchArgs[1], nullptr, true}};
    return run_nl_means<uint8_t>(args, patch_size, search_area, sigma, "nl_means_u8_interleaved_batch launch");
}
