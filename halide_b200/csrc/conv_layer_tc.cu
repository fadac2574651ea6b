// conv_layer_tc.cu — conv_layer's dense contraction on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Same contract as conv_layer.cu (apps/conv_layer/conv_layer_generator.cpp:17-50); this is the only pipeline of the
// seven whose hot loop is GEMM-shaped: M = output pixels, N = 128 output channels, K = 3*3*128.
//
// Formulation.  The input is (N=5, 82, 102, CI=128) channel-innermost, i.e. a row-major matrix In[41820][128].  If the
// output is ALSO enumerated over the padded width (q = y*102 + x, x < 102; columns x >= 100 are discarded), the input
// row feeding output q at tap (ky,kx) is simply q + ky*102 + kx: every tap is the same 2-D tile shifted by a constant
// number of rows, so the implicit-GEMM A operand of a 128-pixel tile is one TMA box load per (tap, 32-channel chunk)
// — no im2col.  The filter is re-laid once per call as Bt[(ky*3+kx)*128 + co][ci] (K-major).
// Precision.  TF32 MMAs read 10 mantissa bits, not enough for the 1e-4 bar on rand()-scale data (SURVEY.md R8), so
// both operands are split hi = tf32(x), lo = x - hi and three products are accumulated (hi*hi + hi*lo + lo*hi) into
// fp32 accumulators: relative error ~2^-19 per product.
//
// Kernel: one CTA per (128-pixel tile, image), 288 threads, warp-specialised:
//   warp 8       TMA producer: per K step 4 box loads (A_hi, A_lo, B_hi, B_lo: rows x 32 floats, SWIZZLE_128B) into a
//                3-stage shared-memory ring, mbarrier complete_tx
//   warps 0-7    two consumer warpgroups, one per 64-pixel half of the tile: 4 x 3 wgmma.m64n128k8 (TF32, both operands
//                from shared memory) per stage into register accumulators, then + bias, relu and the stores
//
// Any shape (conv_layer_tc_run_any_shape, conv_layer_tc_any_kernel): the same kernel body with the shape in a kernel
// parameter (ConvShape).  Output rows are enumerated flat over the whole padded batch, q in [0, N*HP*WP), so a tile of 128
// rows runs across image boundaries and small images do not leave tiles half empty; rows with y >= H or x >= W are
// discarded, and the tap shift ky*WP + kx is unchanged (a discarded row's taps may reach into the next image; rows past
// the end read as zeros from TMA).  The split input and the re-laid filter are this file's own scratch, so their channel
// pitch is CIp = round_up(CI, 32) and Bt's rows per tap are padded to the N tile, both with zeros: every TMA box is
// whole for any CI and CO.  The N tile is 128 (wgmma.m64n128k8) or, for CO <= 64, 64 (wgmma.m64n64k8); CTAs of the
// same rows and successive CO tiles are neighbours in the 1-D grid.  With more than 36 K steps (CI > 128) the two
// alternating accumulators are added in round-to-nearest into a third register set every 36 K steps, so no chain of
// truncating tensor-core additions is longer than the fixed shape's 216 whatever CI is.  Three sets are 192 registers
// at N = 128: these kernels run 384 threads (the producer is a whole warpgroup, one thread of which works) and move
// the producer's registers to the consumers with setmaxnreg.
#include "conv_layer_tc.h"
#include "hb_common.h"
#include "hb_tma.cuh"

namespace {

constexpr int N = 5, CI = 128, CO = 128, W = 100, H = 80;
constexpr int WP = W + 2, HP = H + 2;
constexpr int ROWS_PER_IMAGE = HP * WP;          // 8364 input rows per image
constexpr int A_ROWS = N * ROWS_PER_IMAGE;       // 41820
constexpr int TILE_M = 128, TILE_N = CO, TILE_K = 32;  // 32 tf32 = 128 bytes = one swizzle row
constexpr int TILES_PER_IMAGE = (H * WP + TILE_M - 1) / TILE_M;  // 64 (outputs enumerated over the padded width)
constexpr int K_STEPS = 9 * (CI / TILE_K);       // 36
constexpr int STAGES = 3;
constexpr int CONSUMER_WARPS = 8;                // two warpgroups of 64 output pixels each
constexpr int THREADS = (CONSUMER_WARPS + 1) * 32;
constexpr int THREADS_ANY = (CONSUMER_WARPS + 4) * 32;  // any-shape kernels: the producer is a warpgroup (setmaxnreg)
constexpr int FOLD_STEPS = K_STEPS;              // K steps between two folds of the accumulators: the fixed shape's chain
constexpr int A_TILE_BYTES = TILE_M * TILE_K * 4;  // 16 KB
__host__ __device__ constexpr int b_tile_bytes(int tn) { return tn * TILE_K * 4; }                            // 16 KB at N = 128, 8 KB at 64
__host__ __device__ constexpr int stage_bytes(int tn) { return 2 * A_TILE_BYTES + 2 * b_tile_bytes(tn); }     // A_hi, A_lo, B_hi, B_lo
__host__ __device__ constexpr int smem_bytes(int tn) { return STAGES * stage_bytes(tn) + 1024 /*alignment slack*/ + 256 /*barriers*/; }

// The shape of an any-shape call, as the kernel needs it (ConvProblem, conv_layer_tc.h, is the host's view).
struct ConvShape {
    int wp, rows_per_image;      // W + 2, (H + 2) * (W + 2)
    int W, H, CO;
    int m_rows;                  // output rows enumerated: up to the last valid one of the last image
    int k_chunks, k_steps;       // CIp / 32, 9 * k_chunks
    int co_tiles, co_pad;        // CO tiles of TN channels; Bt rows per tap = co_tiles * TN
    int vec2;                    // relu's base and strides keep channel pairs 8-byte aligned
    long long out_sx, out_sy, out_sn;
    int CI;                      // the recompute's view of input and filter (conv_recompute)
    long long in_sx, in_sy, in_sn, f_skx, f_sky, f_sci;
};

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (PTX ISA "Matrix Descriptor Format"): start address >> 4
// in [0,14), leading byte offset (unused for swizzled K-major, 1) in [16,30), stride byte offset 1024 B between 8-row
// groups in [32,46), layout type 1 = 128-byte swizzle in [62,64).  The tile base must be 1024-byte aligned.
__device__ __forceinline__ uint64_t wgmma_desc(const void *tile) {
    return (uint64_t)((tma::smem_u32(tile) & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template<int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

#define HB_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// d[64] += A(64 x 8, tf32) * B(8 x 128, tf32)^T, both K-major in shared memory.  Accumulator fragment of thread t of the
// warpgroup: d[4j + {0,1}] = (row 16*(t/32) + (t%32)/4, columns 8j + 2*(t%4) + {0,1}), d[4j + {2,3}] = the same 8 rows down.
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1;"
                 : HB_D8(0), HB_D8(8), HB_D8(16), HB_D8(24), HB_D8(32), HB_D8(40), HB_D8(48), HB_D8(56)
                 : "l"(a_desc), "l"(b_desc)
                 : "memory");
}
// The same with 64 output channels: d[32], fragment layout as above with j < 8.
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1;"
                 : HB_D8(0), HB_D8(8), HB_D8(16), HB_D8(24)
                 : "l"(a_desc), "l"(b_desc)
                 : "memory");
}
#undef HB_D8
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t a, uint64_t b) { wgmma_m64n128k8_tf32(d, a, b); }
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t a, uint64_t b) { wgmma_m64n64k8_tf32(d, a, b); }
template<int REGS>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }
template<int REGS>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }

// ---- operand preparation ----------------------------------------------------------------------------------------------
// The split of a non-finite x gives lo = NaN (inf - inf, or NaN - hi), so every product it enters, including the ones
// against a zero, is NaN, and so is the sum of every output whose receptive field holds it: the epilogue recomputes
// those outputs (conv_recompute).
__global__ void conv_split_input_kernel(const float4 *__restrict__ in, float4 *__restrict__ hi, float4 *__restrict__ lo, size_t n4) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 v = in[i], h, l;
    h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u); l.x = v.x - h.x;
    h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u); l.y = v.y - h.y;
    h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u); l.z = v.z - h.z;
    h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u); l.w = v.w - h.w;
    hi[i] = h;
    lo[i] = l;
}
// filter(co, kx, ky, ci) co-innermost  ->  Bt[(ky*3+kx)*CO + co][ci], split
__global__ void conv_prep_filter_kernel(const float *__restrict__ f, float *__restrict__ hi, float *__restrict__ lo) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;  // index into Bt
    if (i >= 9 * CO * CI) return;
    int ci = i % CI, co = (i / CI) % CO, tap = i / (CI * CO);
    int ky = tap / 3, kx = tap - ky * 3;
    float v = f[co + kx * CO + ky * (CO * 3) + (size_t)ci * (CO * 9)];
    float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    hi[i] = h;
    lo[i] = v - h;
}
// Any shape: 8 rows of In per block, one (x, y, n) of the padded image each; the lanes walk its CIp channels, reading
// input through its strides and writing zeros into the channel padding.  vec4: CI, the base and the strides are multiples
// of four floats, so a lane moves float4s.
__device__ __forceinline__ void split_store(float v, float &h, float &l) {
    h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    l = v - h;
}
__global__ void conv_split_input_any_kernel(const float *__restrict__ in, long long sx, long long sy, long long sn, int CI, int CIp, int wp,
                                            int hp, int rows, int vec4, float *__restrict__ hi, float *__restrict__ lo) {
    const int row = blockIdx.x * 8 + threadIdx.y;
    if (row >= rows) return;
    const int t = row / wp, x = row - t * wp, n = t / hp, y = t - n * hp;
    const float *src = in + x * sx + y * sy + n * sn;
    const size_t dst = (size_t)row * CIp;
    if (vec4) {
        for (int c = 4 * threadIdx.x; c < CIp; c += 128) {
            const float4 v = c < CI ? *reinterpret_cast<const float4 *>(src + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            float4 h, l;
            split_store(v.x, h.x, l.x);
            split_store(v.y, h.y, l.y);
            split_store(v.z, h.z, l.z);
            split_store(v.w, h.w, l.w);
            *reinterpret_cast<float4 *>(hi + dst + c) = h;
            *reinterpret_cast<float4 *>(lo + dst + c) = l;
        }
        return;
    }
    for (int c = threadIdx.x; c < CIp; c += 32) {
        float h, l;
        split_store(c < CI ? src[c] : 0.f, h, l);
        hi[dst + c] = h;
        lo[dst + c] = l;
    }
}
// Any shape: filter through its strides  ->  Bt[tap * co_pad + co][ci] with row pitch CIp, zeros in both paddings.  One
// block transposes a 32 co x 32 ci tile of one tap through shared memory: reads run along co, writes along ci.
__global__ void conv_prep_filter_any_kernel(const float *__restrict__ f, long long skx, long long sky, long long sci, int CI, int CIp, int CO,
                                            int co_pad, float *__restrict__ hi, float *__restrict__ lo) {
    __shared__ float tile[32][33];
    const int ci_tiles = CIp / 32, co0 = (blockIdx.x / ci_tiles) * 32, ci0 = (blockIdx.x % ci_tiles) * 32, tap = blockIdx.y;
    const int ky = tap / 3, kx = tap - ky * 3;
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int ci = ci0 + r, co = co0 + threadIdx.x;
        tile[r][threadIdx.x] = (ci < CI && co < CO) ? f[co + kx * skx + ky * sky + ci * sci] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += 8) {
        const size_t o = ((size_t)tap * co_pad + co0 + r) * CIp + ci0 + threadIdx.x;
        split_store(tile[threadIdx.x][r], hi[o], lo[o]);
    }
}

// ---- the GEMM ---------------------------------------------------------------------------------------------------------
// One K step (32 input channels of one tap) of one consumer warpgroup into accumulator d; releases the stage of the
// previous K step once the MMAs that read it have completed.
template<int TN>
__device__ __forceinline__ void consume_step(float (&d)[TN / 2], const uint8_t *tiles, uint64_t *full_bar, uint64_t *empty_bar, int it, int wg,
                                             int lane) {
    const int s = it % STAGES;
    tma::mbar_wait(&full_bar[s], (it / STAGES) & 1);
    const uint8_t *st = tiles + s * stage_bytes(TN);
    const int a_off = wg * 64 * TILE_K * 4;  // this warpgroup's 64 rows of the A tiles (8 KB, a multiple of the 1024-byte swizzle atom)
    const uint64_t a_hi = wgmma_desc(st + a_off), a_lo = wgmma_desc(st + A_TILE_BYTES + a_off);
    const uint64_t b_hi = wgmma_desc(st + 2 * A_TILE_BYTES), b_lo = wgmma_desc(st + 2 * A_TILE_BYTES + b_tile_bytes(TN));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TILE_K / 8; k++) {  // K = 8 tf32 = 32 bytes per MMA: advance the start addresses by 2 (16-byte units)
        const uint64_t adv = (uint64_t)(2 * k);
        wgmma_tf32(d, a_hi + adv, b_hi + adv);
        wgmma_tf32(d, a_hi + adv, b_lo + adv);
        wgmma_tf32(d, a_lo + adv, b_hi + adv);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous K step's MMAs are done: its stage can be refilled
    if (it > 0 && lane == 0) tma::mbar_arrive(&empty_bar[(it - 1) % STAGES]);
}

// The generator's relu, max(0, conv), as Halide lowers it: select(conv > 0, conv, 0).  +inf stays +inf; NaN and -0.0
// give +0.0.
__device__ __forceinline__ float relu(float v) { return v > 0.f ? v : 0.f; }

// One output in the generator's order: bias, then ky, kx, ci ascending, each term a separate fp32 multiply and add (the
// library builds with --fmad=false), then relu.  `in` is the input at the output's (x, y, n), `f` the filter at its co.
// The epilogue calls it for the sums that are not finite, where the split's products say nothing about which of +inf,
// -inf and NaN the generator's sum is.
__device__ float conv_recompute(const float *in, long long in_sx, long long in_sy, const float *f, long long f_skx, long long f_sky,
                                long long f_sci, int ci_n, float acc) {
    for (int ky = 0; ky < 3; ky++)
        for (int kx = 0; kx < 3; kx++) {
            const float *a = in + kx * in_sx + ky * in_sy, *w = f + kx * f_skx + ky * f_sky;
            for (int ci = 0; ci < ci_n; ci++) acc = acc + w[ci * f_sci] * a[ci];
        }
    return relu(acc);
}

// Output pixel (n, y, x) of row q of the output enumeration; false for a discarded row.
template<bool ANY>
__device__ __forceinline__ bool output_pixel(int q, int img, const ConvShape &sh, int &n, int &y, int &x) {
    if (!ANY) {
        n = img, y = q / WP, x = q - y * WP;
        return y < H && x < W;
    }
    if (q >= sh.m_rows) return false;
    n = q / sh.rows_per_image;  // q runs over the whole padded batch
    const int r = q - n * sh.rows_per_image;
    y = r / sh.wp, x = r - y * sh.wp;
    return y < sh.H && x < sh.W;
}

// The kernel body.  ANY = false is the fixed shape (every quantity a constant, `sh` unused, grid (tiles, images));
// ANY = true reads the shape from `sh` (1-D grid, CO tile fastest).  TN is the N tile; FOLD adds the third register set.
template<int TN, bool ANY, bool FOLD>
__device__ __forceinline__ void conv_tc_body(const CUtensorMap *map_a_hi, const CUtensorMap *map_a_lo, const CUtensorMap *map_b_hi,
                                             const CUtensorMap *map_b_lo, const ConvShape &sh, const float *__restrict__ in,
                                             const float *__restrict__ filt, const float *__restrict__ bias, float *__restrict__ out) {
    constexpr int NACC = TN / 2;  // accumulator registers per set
    extern __shared__ uint8_t smem_raw[];
    uint8_t *tiles = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);  // SWIZZLE_128B needs 1024-byte alignment
    uint64_t *full_bar = (uint64_t *)(tiles + STAGES * stage_bytes(TN));
    uint64_t *empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = ANY ? blockIdx.x / sh.co_tiles : blockIdx.x, img = blockIdx.y;
    const int co0 = ANY ? (blockIdx.x - tile * sh.co_tiles) * TN : 0;  // first output channel of this CTA
    const int a_row0 = ANY ? tile * TILE_M : img * ROWS_PER_IMAGE + tile * TILE_M;
    const int wp = ANY ? sh.wp : WP, k_chunks = ANY ? sh.k_chunks : CI / TILE_K, k_steps = ANY ? sh.k_steps : K_STEPS;
    const int b_rows_per_tap = ANY ? sh.co_pad : CO;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) {
            tma::mbar_init(&full_bar[s], 1);
            tma::mbar_init(&empty_bar[s], CONSUMER_WARPS);  // one arrival per consumer warp
        }
        tma::fence_barrier_init();
    }
    __syncthreads();

    if (ANY ? warp >= CONSUMER_WARPS : warp == CONSUMER_WARPS) {
        if (ANY) setmaxnreg_dec<40>();
        if (warp == CONSUMER_WARPS && lane == 0) {
            // ===== TMA producer =====
            for (int it = 0; it < k_steps; it++) {
                const int s = it % STAGES, round = it / STAGES;
                if (round > 0) tma::mbar_wait(&empty_bar[s], (round - 1) & 1);
                const int tap = it / k_chunks, kc = it % k_chunks;
                const int ky = tap / 3, kx = tap - ky * 3;
                uint8_t *st = tiles + s * stage_bytes(TN);
                tma::mbar_expect_tx(&full_bar[s], stage_bytes(TN));
                tma::load_2d(st, map_a_hi, &full_bar[s], kc * TILE_K, a_row0 + ky * wp + kx);
                tma::load_2d(st + A_TILE_BYTES, map_a_lo, &full_bar[s], kc * TILE_K, a_row0 + ky * wp + kx);
                tma::load_2d(st + 2 * A_TILE_BYTES, map_b_hi, &full_bar[s], kc * TILE_K, tap * b_rows_per_tap + co0);
                tma::load_2d(st + 2 * A_TILE_BYTES + b_tile_bytes(TN), map_b_lo, &full_bar[s], kc * TILE_K, tap * b_rows_per_tap + co0);
            }
        }
        return;
    }
    if (ANY) setmaxnreg_inc<232>();

    // ===== consumers: warpgroup wg owns output rows 64*wg .. 64*wg+63 of the tile =====
    const int wg = warp >> 2;
    // Two accumulators, K steps alternating between them, summed in round-to-nearest at the end: the tensor core's own
    // fp32 accumulation does not round to nearest, and halving the chain of 432 MMA additions halves that bias.  FOLD:
    // the two are also added into `sum` and cleared every FOLD_STEPS K steps, which bounds the chain for any CI.  An
    // odd step count leaves the last step in acc0.
    float acc0[NACC], acc1[NACC], sum[FOLD ? NACC : 1];
#pragma unroll
    for (int j = 0; j < NACC; j++) acc0[j] = acc1[j] = 0.f;
    if (FOLD) {
#pragma unroll
        for (int j = 0; j < NACC; j++) sum[j] = 0.f;
    }
    int fold_at = FOLD_STEPS;
#pragma unroll 1
    for (int it = 0; it < k_steps; it += 2) {
        consume_step<TN>(acc0, tiles, full_bar, empty_bar, it, wg, lane);
        if (!ANY || it + 1 < k_steps) consume_step<TN>(acc1, tiles, full_bar, empty_bar, it + 1, wg, lane);
        if (FOLD && it + 2 == fold_at && it + 2 < k_steps) {
            fold_at += FOLD_STEPS;
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < NACC; j++) {
                asm volatile("" : "+f"(acc0[j]), "+f"(acc1[j])::"memory");  // read the accumulators after the wait, not before
                sum[j] += acc0[j] + acc1[j];
                acc0[j] = acc1[j] = 0.f;
            }
        }
    }
    wgmma_wait<0>();

    // ===== epilogue: + bias, relu, float2 stores of the valid pixels =====
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    uint64_t redo = 0;  // bit i: accumulator i's sum is not finite
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int q = tile * TILE_M + r0 + 8 * h;  // output index over the padded width
        int n, y, x;
        if (!output_pixel<ANY>(q, img, sh, n, y, x)) continue;
        if constexpr (!ANY) {
            float *orow = out + (((size_t)img * H + y) * W + x) * CO;
#pragma unroll
            for (int j = 0; j < TN / 8; j++) {
                const int c = 8 * j + 2 * (lane & 3);
                const float2 b = __ldg(reinterpret_cast<const float2 *>(bias + c));
                const float s0 = (acc0[4 * j + 2 * h] + acc1[4 * j + 2 * h]) + b.x;
                const float s1 = (acc0[4 * j + 2 * h + 1] + acc1[4 * j + 2 * h + 1]) + b.y;
                redo |= (uint64_t)!isfinite(s0) << (4 * j + 2 * h) | (uint64_t)!isfinite(s1) << (4 * j + 2 * h + 1);
                *reinterpret_cast<float2 *>(orow + c) = make_float2(relu(s0), relu(s1));
            }
        } else {
            float *orow = out + n * sh.out_sn + y * sh.out_sy + x * sh.out_sx;
#pragma unroll
            for (int j = 0; j < TN / 8; j++) {
                const int c = co0 + 8 * j + 2 * (lane & 3);
                if (c >= sh.CO) continue;
                const bool pair = c + 1 < sh.CO;
                float s0 = acc0[4 * j + 2 * h] + acc1[4 * j + 2 * h], s1 = acc0[4 * j + 2 * h + 1] + acc1[4 * j + 2 * h + 1];
                if (FOLD) s0 += sum[4 * j + 2 * h], s1 += sum[4 * j + 2 * h + 1];
                s0 += __ldg(bias + c);
                s1 = pair ? s1 + __ldg(bias + c + 1) : 0.f;
                redo |= (uint64_t)!isfinite(s0) << (4 * j + 2 * h) | (uint64_t)!isfinite(s1) << (4 * j + 2 * h + 1);
                const float2 v = make_float2(relu(s0), relu(s1));
                if (pair && sh.vec2) {
                    *reinterpret_cast<float2 *>(orow + c) = v;
                } else {
                    orow[c] = v.x;
                    if (pair) orow[c + 1] = v.y;
                }
            }
        }
    }
    // Outputs whose sum is not finite: an operand is +-inf or NaN (conv_split_input_kernel), or the sum overflowed.  Each
    // is computed again in the generator's order and overwrites what the loop above stored.  Rare, so a plain loop.
#pragma unroll 1
    while (redo) {
        const int i = __ffsll((long long)redo) - 1;
        redo &= redo - 1;
        const int h = (i >> 1) & 1, c = co0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        int n, y, x;
        output_pixel<ANY>(tile * TILE_M + r0 + 8 * h, img, sh, n, y, x);
        if constexpr (!ANY) {
            out[(((size_t)n * H + y) * W + x) * CO + c] =
                conv_recompute(in + (((size_t)n * HP + y) * WP + x) * CI, CI, WP * CI, filt + c, CO, 3 * CO, 9 * CO, CI, bias[c]);
        } else {
            out[n * sh.out_sn + y * sh.out_sy + x * sh.out_sx + c] = conv_recompute(
                in + x * sh.in_sx + y * sh.in_sy + n * sh.in_sn, sh.in_sx, sh.in_sy, filt + c, sh.f_skx, sh.f_sky, sh.f_sci, sh.CI, bias[c]);
        }
    }
}

__global__ void __launch_bounds__(THREADS, 1) conv_layer_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi,
                                                                   const __grid_constant__ CUtensorMap map_a_lo,
                                                                   const __grid_constant__ CUtensorMap map_b_hi,
                                                                   const __grid_constant__ CUtensorMap map_b_lo,
                                                                   const float *__restrict__ in, const float *__restrict__ filt,
                                                                   const float *__restrict__ bias, float *__restrict__ out) {
    conv_tc_body<TILE_N, false, false>(&map_a_hi, &map_a_lo, &map_b_hi, &map_b_lo, ConvShape{}, in, filt, bias, out);
}

template<int TN, bool FOLD>
__global__ void __launch_bounds__(THREADS_ANY, 1) conv_layer_tc_any_kernel(const __grid_constant__ CUtensorMap map_a_hi,
                                                                           const __grid_constant__ CUtensorMap map_a_lo,
                                                                           const __grid_constant__ CUtensorMap map_b_hi,
                                                                           const __grid_constant__ CUtensorMap map_b_lo,
                                                                           const __grid_constant__ ConvShape sh,
                                                                           const float *__restrict__ in, const float *__restrict__ filt,
                                                                           const float *__restrict__ bias, float *__restrict__ out) {
    conv_tc_body<TN, true, FOLD>(&map_a_hi, &map_a_lo, &map_b_hi, &map_b_lo, sh, in, filt, bias, out);
}

// rows x pitch floats, boxes of box_rows x 32
bool make_map(CUtensorMap *m, void *base, uint64_t rows, uint32_t box_rows, uint64_t pitch = CI) {
    const uint64_t dims[2] = {pitch, rows};
    const int64_t strides[1] = {(int64_t)(pitch * sizeof(float))};
    const uint32_t box[2] = {(uint32_t)TILE_K, box_rows};
    return tma::encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

template<int TN, bool FOLD>
void launch_any(unsigned grid, cudaStream_t s, const CUtensorMap &ma_hi, const CUtensorMap &ma_lo, const CUtensorMap &mb_hi,
                const CUtensorMap &mb_lo, const ConvShape &sh, const ConvProblem &p) {
    hb::allow_smem(conv_layer_tc_any_kernel<TN, FOLD>, smem_bytes(TN));
    HB_LAUNCH(TN == 128 ? (FOLD ? "conv_layer_tc_n128_fold" : "conv_layer_tc_n128") : (FOLD ? "conv_layer_tc_n64_fold" : "conv_layer_tc_n64"),
              (conv_layer_tc_any_kernel<TN, FOLD>), grid, THREADS_ANY, smem_bytes(TN), s, ma_hi, ma_lo, mb_hi, mb_lo, sh, p.in, p.filt,
              p.bias, p.out);
}

}  // namespace

// Returns 0 on success, a negative halide error code otherwise.  din/df/db/dout are device pointers in the generator's layouts.
int conv_layer_tc_run(const float *din, const float *df, const float *db, float *dout, cudaStream_t s) {
    if (!tma::encoder()) return hb::fail(halide_error_code_generic_error, "conv_layer: cuTensorMapEncodeTiled is not available");
    hb::Scratch scratch;
    const size_t a_elems = (size_t)A_ROWS * CI, b_elems = (size_t)9 * CO * CI;
    float *a_hi = scratch.get<float>(a_elems), *a_lo = scratch.get<float>(a_elems);
    float *b_hi = scratch.get<float>(b_elems), *b_lo = scratch.get<float>(b_elems);
    if (!a_hi || !a_lo || !b_hi || !b_lo) return hb::fail(halide_error_code_device_malloc_failed, "conv_layer: scratch allocation failed");
    CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
    if (!make_map(&ma_hi, a_hi, A_ROWS, TILE_M) || !make_map(&ma_lo, a_lo, A_ROWS, TILE_M) || !make_map(&mb_hi, b_hi, 9 * CO, TILE_N) ||
        !make_map(&mb_lo, b_lo, 9 * CO, TILE_N)) {
        return hb::fail(halide_error_code_generic_error, "conv_layer: cuTensorMapEncodeTiled failed");
    }
    hb::allow_smem(conv_layer_tc_kernel, smem_bytes(TILE_N));
    HB_LAUNCH("conv_split_input", conv_split_input_kernel, (unsigned)((a_elems / 4 + 255) / 256), 256, 0, s, (const float4 *)din, (float4 *)a_hi,
              (float4 *)a_lo, a_elems / 4);
    HB_LAUNCH("conv_prep_filter", conv_prep_filter_kernel, (unsigned)((b_elems + 255) / 256), 256, 0, s, df, b_hi, b_lo);
    HB_LAUNCH("conv_layer_tc", conv_layer_tc_kernel, dim3(TILES_PER_IMAGE, N), THREADS, smem_bytes(TILE_N), s, ma_hi, ma_lo, mb_hi, mb_lo, din,
              df, db, dout);
    return 0;
}

int conv_layer_tc_run_any_shape(const ConvProblem &p, cudaStream_t s) {
    if (!tma::encoder()) return hb::fail(halide_error_code_generic_error, "conv_layer: cuTensorMapEncodeTiled is not available");
    const int tn = p.CO <= 64 ? 64 : 128;
    const int hp = p.H + 2;
    // (a filter of no input channels still gets one chunk, of zeros: the result is relu(bias))
    const int CIp = (p.CI > 0 ? (p.CI + TILE_K - 1) / TILE_K : 1) * TILE_K;
    ConvShape sh;
    sh.wp = p.W + 2;
    sh.rows_per_image = hp * sh.wp;
    sh.W = p.W, sh.H = p.H, sh.CO = p.CO;
    sh.m_rows = (p.N - 1) * sh.rows_per_image + (p.H - 1) * sh.wp + p.W;
    sh.k_chunks = CIp / TILE_K;
    sh.k_steps = 9 * sh.k_chunks;
    sh.co_tiles = (p.CO + tn - 1) / tn;
    sh.co_pad = sh.co_tiles * tn;
    sh.out_sx = p.out_sx, sh.out_sy = p.out_sy, sh.out_sn = p.out_sn;
    sh.vec2 = ((uintptr_t)p.out % 8 == 0) && p.out_sx % 2 == 0 && p.out_sy % 2 == 0 && p.out_sn % 2 == 0;
    sh.CI = p.CI;
    sh.in_sx = p.in_sx, sh.in_sy = p.in_sy, sh.in_sn = p.in_sn;
    sh.f_skx = p.f_skx, sh.f_sky = p.f_sky, sh.f_sci = p.f_sci;
    const int rows = p.N * sh.rows_per_image;  // fits: input's extents multiply to less than 2^31
    const long long m_tiles = ((long long)sh.m_rows + TILE_M - 1) / TILE_M;
    if (m_tiles * sh.co_tiles > 0x7fffffffLL) {
        return hb::fail(halide_error_code_generic_error, "conv_layer: %lld x %d tiles exceed the launch grid", m_tiles, sh.co_tiles);
    }

    hb::Scratch scratch;
    const size_t a_elems = (size_t)rows * CIp, b_elems = (size_t)9 * sh.co_pad * CIp;
    float *a_hi = scratch.get<float>(a_elems), *a_lo = scratch.get<float>(a_elems);
    float *b_hi = scratch.get<float>(b_elems), *b_lo = scratch.get<float>(b_elems);
    if (!a_hi || !a_lo || !b_hi || !b_lo) return hb::fail(halide_error_code_device_malloc_failed, "conv_layer: scratch allocation failed");
    CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
    if (!make_map(&ma_hi, a_hi, rows, TILE_M, CIp) || !make_map(&ma_lo, a_lo, rows, TILE_M, CIp) ||
        !make_map(&mb_hi, b_hi, 9ull * sh.co_pad, tn, CIp) || !make_map(&mb_lo, b_lo, 9ull * sh.co_pad, tn, CIp)) {
        return hb::fail(halide_error_code_generic_error, "conv_layer: cuTensorMapEncodeTiled failed");
    }
    const bool vec4 = p.CI % 4 == 0 && (uintptr_t)p.in % 16 == 0 && p.in_sx % 4 == 0 && p.in_sy % 4 == 0 && p.in_sn % 4 == 0;
    HB_LAUNCH("conv_split_input_any", conv_split_input_any_kernel, (unsigned)((rows + 7) / 8), dim3(32, 8), 0, s, p.in, (long long)p.in_sx,
              (long long)p.in_sy, (long long)p.in_sn, p.CI, CIp, sh.wp, hp, rows, (int)vec4, a_hi, a_lo);
    HB_LAUNCH("conv_prep_filter_any", conv_prep_filter_any_kernel, dim3((unsigned)((sh.co_pad / 32) * (CIp / 32)), 9), dim3(32, 8), 0, s, p.filt,
              (long long)p.f_skx, (long long)p.f_sky, (long long)p.f_sci, p.CI, CIp, p.CO, sh.co_pad, b_hi, b_lo);
    const unsigned grid = (unsigned)(m_tiles * sh.co_tiles);
    const bool fold = sh.k_steps > FOLD_STEPS;
    if (tn == 128) {
        if (fold) launch_any<128, true>(grid, s, ma_hi, ma_lo, mb_hi, mb_lo, sh, p);
        else launch_any<128, false>(grid, s, ma_hi, ma_lo, mb_hi, mb_lo, sh, p);
    } else {
        if (fold) launch_any<64, true>(grid, s, ma_hi, ma_lo, mb_hi, mb_lo, sh, p);
        else launch_any<64, false>(grid, s, ma_hi, ma_lo, mb_hi, mb_lo, sh, p);
    }
    return 0;
}
