// hb_tma.cuh — TMA (cp.async.bulk.tensor) + mbarrier helpers shared by the tile kernels, and the host-side tensor-map
// encoder (cuTensorMapEncodeTiled reached through cudaGetDriverEntryPoint: the library links only the CUDA runtime).
//
// How the image kernels use it: an INTERIOR tile of a frame — or any tile whose out-of-range part may read as zero —
// is fetched with one bulk tensor copy issued by one thread and awaited on an mbarrier, so the loads cost no
// registers, no address arithmetic and no per-thread latency; tiles that need repeat_edge replication take the
// kernels' clamped load path instead (TMA fills out-of-bounds elements with zeros, it cannot clamp).
// TMA constraints checked by the hosts before they choose this path: base address and every byte stride a multiple of
// 16, inner box extent * element size a multiple of 16 bytes, box extents <= 256.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tma {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
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
__device__ __forceinline__ void load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void load_3d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}

// ---- host side ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encoder() {
    static EncodeTiledFn enc = [] {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) {
            cudaGetLastError();
            return (EncodeTiledFn) nullptr;
        }
        return (EncodeTiledFn)fn;
    }();
    return enc;
}

// Whether a dense-innermost image with these byte strides can be described by a tensor map at all.
inline bool strides_ok(const void *base, const int64_t *stride_bytes, int nstrides) {
    if (((uintptr_t)base & 15) != 0) return false;
    for (int i = 0; i < nstrides; i++) {
        if (stride_bytes[i] <= 0 || (stride_bytes[i] & 15) != 0 || stride_bytes[i] >= (1ll << 40)) return false;
    }
    return true;
}

// rank-`rank` tiled map (no interleave, zero fill out of bounds): dims / box in elements, innermost first;
// stride_bytes[i] = byte stride of dimension i+1.  Returns false when the driver refuses it or the encoder is missing.
inline bool encode(CUtensorMap *m, CUtensorMapDataType type, int rank, void *base, const uint64_t *dims, const int64_t *stride_bytes,
                   const uint32_t *box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_NONE) {
    EncodeTiledFn enc = encoder();
    if (!enc) return false;
    cuuint64_t d[5], st[4];
    cuuint32_t b[5], es[5];
    for (int i = 0; i < rank; i++) {
        d[i] = dims[i];
        b[i] = box[i];
        es[i] = 1;
        if (i + 1 < rank) st[i] = (cuuint64_t)stride_bytes[i];
    }
    return enc(m, type, (cuuint32_t)rank, base, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tma
