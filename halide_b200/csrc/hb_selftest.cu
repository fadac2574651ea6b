// hb_selftest.cu — device evaluation hook for the scalar primitives of hl_math.cuh.
//
// halide_b200_selftest_math evaluates one hl:: primitive element by element over device arrays, each case calling the
// __forceinline__ function itself, compiled with the library's flags (--fmad=false, IEEE division).  The CPU oracle
// exports the same cases (oracle/oracle_prims.cpp: oracle_math_vec, same numbering), so a test can compare the two
// copies of every primitive on any input set; tests/test_hl_math_gpu.py does, on every float32 input where there is one
// operand.
#include <algorithm>

#include "hb_common.h"
#include "hl_math.cuh"

namespace {

// Coefficient sets for the evaluate_polynomial cases: halide_exp's (even count), halide_log's (a zero at an odd index)
// and a set of odd count with a zero at an even index, so every branch of the evaluation is taken.
__device__ const float kPolyExp[8] = {0.00031965933071842413f, 0.00119156835564003744f, 0.00848988645943932717f,
                                      0.04160188091348320655f, 0.16667983794100929562f, 0.49999899033463041098f,
                                      1.0f, 1.0f};
__device__ const float kPolyLog[10] = {0.05111976432738144643f, -0.11793923497136414580f, 0.14971993724699017569f,
                                       -0.16862004708254804686f, 0.19980668101718729313f, -0.24991211576292837737f,
                                       0.33333435275479328386f, -0.50000106292873236491f, 1.0f, 0.0f};
__device__ const float kPolyOdd[7] = {0.25f, -0.5f, 0.0f, 1.5f, -2.0f, 0.125f, 3.0f};

// Case numbers (halide_b200_runtime.h lists them with their operand types).
enum Fn {
    kExp = 0, kLog, kFastExp, kClamp01, kPow, kClampf, kLerpf, kPoly8, kPoly10, kPoly7,
    kToF32U8, kFromF32U8, kFrameValU8, kFrameNarrowU8, kPairU16U8, kNumFn
};

template<int FN>
__global__ void math_kernel(const void *a_, const void *b_, void *out_, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        if constexpr (FN == kToF32U8) {
            ((float *)out_)[i] = hl::frame_to_f32(((const uint8_t *)a_)[i]);
        } else if constexpr (FN == kFrameValU8) {
            ((float *)out_)[i] = hl::frame_val(((const uint8_t *)a_)[i]);
        } else if constexpr (FN == kFrameNarrowU8) {
            ((uint8_t *)out_)[i] = (uint8_t)hl::frame_narrow<uint8_t>(((const uint16_t *)a_)[i]);
        } else if constexpr (FN == kPairU16U8) {
            ((uint32_t *)out_)[i] = hl::pair_u16<uint8_t>(((const uint16_t *)a_)[i]);
        } else {
            const float a = ((const float *)a_)[i];
            const float *b = (const float *)b_;
            float r;
            if constexpr (FN == kFromF32U8) {
                ((uint8_t *)out_)[i] = hl::frame_from_f32<uint8_t>(a);
                continue;
            } else if constexpr (FN == kExp) r = hl::halide_exp(a);
            else if constexpr (FN == kLog) r = hl::halide_log(a);
            else if constexpr (FN == kFastExp) r = hl::fast_exp(a);
            else if constexpr (FN == kClamp01) r = hl::clamp01(a);
            else if constexpr (FN == kPow) r = hl::halide_pow(a, b[i]);
            else if constexpr (FN == kClampf) r = hl::clampf(a, b[2 * i], b[2 * i + 1]);
            else if constexpr (FN == kLerpf) r = hl::lerpf(a, b[2 * i], b[2 * i + 1]);
            else if constexpr (FN == kPoly8) r = hl::evaluate_polynomial(a, kPolyExp);
            else if constexpr (FN == kPoly10) r = hl::evaluate_polynomial(a, kPolyLog);
            else r = hl::evaluate_polynomial(a, kPolyOdd);
            ((float *)out_)[i] = r;
        }
    }
}

template<int... FN>
void launch(int fn, const void *a, const void *b, void *out, long long n, cudaStream_t s, std::integer_sequence<int, FN...>) {
    const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)hb::sm_count() * 16);
    ((fn == FN ? (math_kernel<FN><<<blocks, 256, 0, s>>>(a, b, out, n), 0) : 0), ...);
}

}  // namespace

extern "C" int halide_b200_selftest_math(int fn, const void *a, const void *b, void *out, long long n) {
    if (fn < 0 || fn >= kNumFn || n < 0 || (n > 0 && (!a || !out))) {
        return hb::fail(halide_error_code_generic_error, "halide_b200_selftest_math: bad arguments (fn %d, n %lld)", fn, n);
    }
    if ((fn == kPow || fn == kClampf || fn == kLerpf) && n > 0 && !b) {
        return hb::fail(halide_error_code_generic_error, "halide_b200_selftest_math: case %d needs a second operand", fn);
    }
    if (n == 0) return 0;
    cudaStream_t s = hb::stream();
    launch(fn, a, b, out, n, s, std::make_integer_sequence<int, kNumFn>{});
    int r = hb::check_cuda(cudaGetLastError(), "halide_b200_selftest_math launch", halide_error_code_device_run_failed);
    if (r) return r;
    return hb::check_cuda(cudaStreamSynchronize(s), "halide_b200_selftest_math", halide_error_code_device_run_failed);
}
