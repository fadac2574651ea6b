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
#include <cuda.h>
#include "hb_common.h"

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
constexpr int A_TILE_BYTES = TILE_M * TILE_K * 4;  // 16 KB
constexpr int B_TILE_BYTES = TILE_N * TILE_K * 4;  // 16 KB
constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;  // A_hi, A_lo, B_hi, B_lo
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*alignment slack*/ + 256 /*barriers*/;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (PTX ISA "Matrix Descriptor Format"): start address >> 4
// in [0,14), leading byte offset (unused for swizzled K-major, 1) in [16,30), stride byte offset 1024 B between 8-row
// groups in [32,46), layout type 1 = 128-byte swizzle in [62,64).  The tile base must be 1024-byte aligned.
__device__ __forceinline__ uint64_t wgmma_desc(const void *tile) {
    return (uint64_t)((smem_u32(tile) & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
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
#undef HB_D8

// ---- operand preparation ----------------------------------------------------------------------------------------------
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

// ---- the GEMM ---------------------------------------------------------------------------------------------------------
// One K step (32 input channels of one tap) of one consumer warpgroup into accumulator d; releases the stage of the
// previous K step once the MMAs that read it have completed.
__device__ __forceinline__ void consume_step(float (&d)[64], const uint8_t *tiles, uint64_t *full_bar, uint64_t *empty_bar, int it, int wg,
                                             int lane) {
    const int s = it % STAGES;
    mbar_wait(&full_bar[s], (it / STAGES) & 1);
    const uint8_t *st = tiles + s * STAGE_BYTES;
    const int a_off = wg * 64 * TILE_K * 4;  // this warpgroup's 64 rows of the A tiles (8 KB, a multiple of the 1024-byte swizzle atom)
    const uint64_t a_hi = wgmma_desc(st + a_off), a_lo = wgmma_desc(st + A_TILE_BYTES + a_off);
    const uint64_t b_hi = wgmma_desc(st + 2 * A_TILE_BYTES), b_lo = wgmma_desc(st + 2 * A_TILE_BYTES + B_TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TILE_K / 8; k++) {  // K = 8 tf32 = 32 bytes per MMA: advance the start addresses by 2 (16-byte units)
        const uint64_t adv = (uint64_t)(2 * k);
        wgmma_m64n128k8_tf32(d, a_hi + adv, b_hi + adv);
        wgmma_m64n128k8_tf32(d, a_hi + adv, b_lo + adv);
        wgmma_m64n128k8_tf32(d, a_lo + adv, b_hi + adv);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous K step's MMAs are done: its stage can be refilled
    if (it > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
}

__global__ void __launch_bounds__(THREADS, 1) conv_layer_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi,
                                                                   const __grid_constant__ CUtensorMap map_a_lo,
                                                                   const __grid_constant__ CUtensorMap map_b_hi,
                                                                   const __grid_constant__ CUtensorMap map_b_lo,
                                                                   const float *__restrict__ bias, float *__restrict__ out) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *tiles = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);  // SWIZZLE_128B needs 1024-byte alignment
    uint64_t *full_bar = (uint64_t *)(tiles + STAGES * STAGE_BYTES);
    uint64_t *empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x, img = blockIdx.y;
    const int a_row0 = img * ROWS_PER_IMAGE + tile * TILE_M;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CONSUMER_WARPS);  // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONSUMER_WARPS) {
        if (lane == 0) {
            // ===== TMA producer =====
            for (int it = 0; it < K_STEPS; it++) {
                const int s = it % STAGES, round = it / STAGES;
                if (round > 0) mbar_wait(&empty_bar[s], (round - 1) & 1);
                const int tap = it / (CI / TILE_K), kc = it % (CI / TILE_K);
                const int ky = tap / 3, kx = tap - ky * 3;
                uint8_t *st = tiles + s * STAGE_BYTES;
                mbar_expect_tx(&full_bar[s], STAGE_BYTES);
                tma_load_2d(st, &map_a_hi, &full_bar[s], kc * TILE_K, a_row0 + ky * WP + kx);
                tma_load_2d(st + A_TILE_BYTES, &map_a_lo, &full_bar[s], kc * TILE_K, a_row0 + ky * WP + kx);
                tma_load_2d(st + 2 * A_TILE_BYTES, &map_b_hi, &full_bar[s], kc * TILE_K, tap * CO);
                tma_load_2d(st + 2 * A_TILE_BYTES + B_TILE_BYTES, &map_b_lo, &full_bar[s], kc * TILE_K, tap * CO);
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns output rows 64*wg .. 64*wg+63 of the tile =====
    const int wg = warp >> 2;
    // Two accumulators, K steps alternating between them, summed in round-to-nearest at the end: the tensor core's own
    // fp32 accumulation does not round to nearest, and halving the chain of 432 MMA additions halves that bias.
    float acc0[64], acc1[64];
#pragma unroll
    for (int j = 0; j < 64; j++) acc0[j] = acc1[j] = 0.f;
#pragma unroll 1
    for (int it = 0; it < K_STEPS; it += 2) {
        consume_step(acc0, tiles, full_bar, empty_bar, it, wg, lane);
        consume_step(acc1, tiles, full_bar, empty_bar, it + 1, wg, lane);
    }
    wgmma_wait<0>();

    // ===== epilogue: + bias, relu, float2 stores of the valid pixels =====
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int q = tile * TILE_M + r0 + 8 * h;  // output index over the padded width
        const int y = q / WP, x = q - y * WP;
        if (y >= H || x >= W) continue;
        float *orow = out + (((size_t)img * H + y) * W + x) * CO;
#pragma unroll
        for (int j = 0; j < TILE_N / 8; j++) {
            const int c = 8 * j + 2 * (lane & 3);
            const float2 b = __ldg(reinterpret_cast<const float2 *>(bias + c));
            float2 v;
            v.x = fmaxf((acc0[4 * j + 2 * h] + acc1[4 * j + 2 * h]) + b.x, 0.f);
            v.y = fmaxf((acc0[4 * j + 2 * h + 1] + acc1[4 * j + 2 * h + 1]) + b.y, 0.f);
            *reinterpret_cast<float2 *>(orow + c) = v;
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_map(EncodeTiledFn enc, CUtensorMap *m, void *base, uint64_t rows, int box_rows) {
    cuuint64_t dims[2] = {(cuuint64_t)CI, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)CI * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)TILE_K, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

}  // namespace

// Returns 0 on success, a negative halide error code otherwise.  din/df/db/dout are device pointers in the generator's layouts.
int conv_layer_tc_run(const float *din, const float *df, const float *db, float *dout, cudaStream_t s) {
    static EncodeTiledFn enc = nullptr;
    if (!enc) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) {
            cudaGetLastError();
            return hb::fail(halide_error_code_generic_error, "conv_layer: cuTensorMapEncodeTiled is not available");
        }
        enc = (EncodeTiledFn)fn;
    }
    hb::Scratch scratch;
    const size_t a_elems = (size_t)A_ROWS * CI, b_elems = (size_t)9 * CO * CI;
    float *a_hi = scratch.get<float>(a_elems), *a_lo = scratch.get<float>(a_elems);
    float *b_hi = scratch.get<float>(b_elems), *b_lo = scratch.get<float>(b_elems);
    if (!a_hi || !a_lo || !b_hi || !b_lo) return hb::fail(halide_error_code_device_malloc_failed, "conv_layer: scratch allocation failed");
    CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
    if (make_map(enc, &ma_hi, a_hi, A_ROWS, TILE_M) || make_map(enc, &ma_lo, a_lo, A_ROWS, TILE_M) ||
        make_map(enc, &mb_hi, b_hi, 9 * CO, TILE_N) || make_map(enc, &mb_lo, b_lo, 9 * CO, TILE_N)) {
        return hb::fail(halide_error_code_generic_error, "conv_layer: cuTensorMapEncodeTiled failed");
    }
    static hb::PerDeviceOnce attr;
    attr.run([] { cudaFuncSetAttribute(conv_layer_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES); });
    HB_LAUNCH("conv_split_input", conv_split_input_kernel, (unsigned)((a_elems / 4 + 255) / 256), 256, 0, s, (const float4 *)din, (float4 *)a_hi,
              (float4 *)a_lo, a_elems / 4);
    HB_LAUNCH("conv_prep_filter", conv_prep_filter_kernel, (unsigned)((b_elems + 255) / 256), 256, 0, s, df, b_hi, b_lo);
    HB_LAUNCH("conv_layer_tc", conv_layer_tc_kernel, dim3(TILES_PER_IMAGE, N), THREADS, SMEM_BYTES, s, ma_hi, ma_lo, mb_hi, mb_lo, db,
              dout);
    return 0;
}
