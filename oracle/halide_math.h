// oracle/halide_math.h — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// CPU restatement of the Halide expression semantics the seven app pipelines rely on
// (SURVEY.md Appendix A).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may compile, link or call anything under oracle/.
//
// Every helper evaluates IEEE binary32 in exactly the written order; the oracle is built with
// -ffp-contract=off and without -ffast-math so no FMA contraction or re-association happens.
// References (paths under /root/reference):
//   evaluate_polynomial   src/IROperator.cpp:33-62
//   halide_log            src/IROperator.cpp:845-919
//   halide_exp            src/IROperator.cpp:921-966
//   fast_exp              src/IROperator.cpp:1616-1643
//   pow_f32 lowering      src/CodeGen_LLVM.cpp:3925-3942
//   Euclidean div/mod     src/IROperator.h:253-311
//   lerp (float)          src/Lerp.cpp:74,126-128  ( z*(1-w) + o*w )
//   clamp                 src/IROperator.cpp:2222-2236 ( max(min(a,hi),lo) )
//   x / const -> x * (1/const) folded in double then rounded  src/Simplify_Div.cpp:204
#pragma once

#include <math.h>
#include <stdint.h>
#include <string.h>

namespace hl {

static inline float as_float(int32_t i) {
    float f;
    memcpy(&f, &i, 4);
    return f;
}
static inline int32_t as_int(float f) {
    int32_t i;
    memcpy(&i, &f, 4);
    return i;
}

// Integer division rounding toward -inf and the matching non-negative remainder, with x/0 == 0.
static inline int div_floor(int a, int b) {
    if (b == 0) return 0;
    int q = a / b, r = a % b;
    if (r != 0 && ((r < 0) != (b < 0))) q -= 1;
    return q;
}
static inline int mod_floor(int a, int b) {
    if (b == 0) return 0;
    int r = a % b;
    if (r < 0) r += (b < 0 ? -b : b);
    return r;
}

static inline int clampi(int a, int lo, int hi) {
    int m = a < hi ? a : hi;
    return m > lo ? m : lo;
}
static inline float clampf(float a, float lo, float hi) {
    float m = a < hi ? a : hi;  // min(a, hi)
    return m > lo ? m : lo;     // max(., lo)
}
static inline float lerpf(float zero_val, float one_val, float w) {
    return zero_val * (1.0f - w) + one_val * w;
}

// Constant folded the way the simplifier does it: reciprocal in double, then rounded to f32.
static inline float recip_const(float c) {
    return (float)(1.0 / (double)c);
}
// x / c for a constant c.  Default ("target=host", apps/support/Makefile.inc:22): the simplifier rewrites it to
// x * fold(1/c) (src/Simplify_Div.cpp:204).  With -DORACLE_STRICT_FLOAT the oracle restates a `strict_float` build
// (src/Target.cpp:603, src/StrictifyFloat.cpp:10-60), where that rewrite does not fire and the division is a true IEEE
// divide — the flag to flip the day a contraction-free Halide build exists to diff against (SURVEY.md §8c).
static inline float div_const(float x, float c) {
#ifdef ORACLE_STRICT_FLOAT
    return x / c;
#else
    return x * recip_const(c);
#endif
}

// High-order coefficient first; n = number of coefficients (degree + 1).
static inline float evaluate_polynomial(float x, const float *coeff, int n) {
    float x2 = x * x;
    float even_terms = coeff[0];
    float odd_terms = coeff[1];
    for (int i = 2; i < n; i++) {
        if ((i & 1) == 0) {
            if (coeff[i] == 0.0f) even_terms = even_terms * x2;
            else even_terms = even_terms * x2 + coeff[i];
        } else {
            if (coeff[i] == 0.0f) odd_terms = odd_terms * x2;
            else odd_terms = odd_terms * x2 + coeff[i];
        }
    }
    if ((n & 1) == 0) return even_terms * x + odd_terms;
    return odd_terms * x + even_terms;
}

// k = floor(x / ln 2) as an int: NaN -> 0, anything else clamped to [-256, 256] (past the ends the result is +inf or 0
// either way).  Halide leaves the plain conversion undefined for NaN and values outside int32 (x86 gives INT_MIN, the
// GPU's cvt.rzi saturates, NaN -> 0) and k + 127 could overflow; hl_math.cuh: exp_k converts the same way.
static inline int32_t exp_k(float k_real) {
    if (k_real != k_real) return 0;
    return (int32_t)clampf(k_real, -256.0f, 256.0f);
}

static inline float halide_exp(float x_full) {
    const float ln2_part1 = 0.6931457519f;
    const float ln2_part2 = 1.4286067653e-6f;
    const float one_over_ln2 = 1.0f / logf(2.0f);
    float scaled = x_full * one_over_ln2;
    float k_real = floorf(scaled);
    int32_t k = exp_k(k_real);
    float x = x_full - k_real * ln2_part1;
    x = x - k_real * ln2_part2;
    static const float coeff[] = {0.00031965933071842413f, 0.00119156835564003744f, 0.00848988645943932717f,
                                  0.04160188091348320655f, 0.16667983794100929562f, 0.49999899033463041098f,
                                  1.0f, 1.0f};
    float result = evaluate_polynomial(x, coeff, 8);
    int32_t biased = k + 127;
    float two_to_the_n = as_float((int32_t)((uint32_t)biased << 23));
    result = result * two_to_the_n;
    if (!(biased < 255)) result = INFINITY;
    if (!(biased > 0)) result = 0.0f;
    return result;
}

static inline float halide_log(float x_full) {
    bool use_nan = x_full < 0.0f;
    bool use_neg_inf = x_full == 0.0f;
    bool exceptional = use_nan || use_neg_inf;
    float patched = exceptional ? 1.0f : x_full;
    // range reduction: patched = 2^exponent * reduced, reduced in [0.75, 1.5)
    int32_t int_version = as_int(patched);
    int32_t no_exponent = int_version & (int32_t)0x807fffff;
    int32_t new_exponent = no_exponent >> 22;
    int32_t new_biased_exponent = 127 - new_exponent;
    int32_t old_biased_exponent = int_version >> 23;
    int32_t exponent = old_biased_exponent - new_biased_exponent;
    int32_t blended = no_exponent | (int32_t)((uint32_t)new_biased_exponent << 23);
    float reduced = as_float(blended);
    static const float coeff[] = {0.05111976432738144643f, -0.11793923497136414580f, 0.14971993724699017569f,
                                  -0.16862004708254804686f, 0.19980668101718729313f, -0.24991211576292837737f,
                                  0.33333435275479328386f, -0.50000106292873236491f, 1.0f, 0.0f};
    float x1 = reduced - 1.0f;
    float result = evaluate_polynomial(x1, coeff, 10);
    result = result + (float)exponent * logf(2.0f);
    if (exceptional) result = use_nan ? NAN : -INFINITY;
    return result;
}

// pow(x, y) for f32 as the LLVM back-ends lower it.
static inline float halide_pow(float x, float y) {
    float abs_x_pow_y = halide_exp(halide_log(fabsf(x)) * y);
    float iy = floorf(y);
    if (x > 0) return abs_x_pow_y;
    if (y == 0.0f) return 1.0f;
    if (x == 0.0f) return 0.0f;
    if (y != iy) return NAN;
    if (fmodf(iy, 2.0f) == 0.0f) return abs_x_pow_y;
    return -abs_x_pow_y;
}

static inline float fast_exp(float x_full) {
    const float ln2 = logf(2.0f);
    float scaled = div_const(x_full, ln2);
    float k_real = floorf(scaled);
    int32_t k = exp_k(k_real);
    float x = x_full - k_real * ln2;
    static const float coeff[] = {0.01314350012789660196f, 0.03668965196652099192f, 0.16873890085469545053f,
                                  0.49970514590562437052f, 1.0f, 1.0f};
    float result = evaluate_polynomial(x, coeff, 6);
    int32_t biased = clampi(k, -127, 128) + 127;  // clamp(k + 127, 0, 255)
    float two_to_the_n = as_float((int32_t)((uint32_t)biased << 23));
    return result * two_to_the_n;
}

}  // namespace hl
