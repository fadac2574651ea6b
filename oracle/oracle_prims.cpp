// oracle/oracle_prims.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle.h).
// Probes that expose the math helpers of halide_math.h to the tests.
#include <omp.h>

#include "halide_math.h"
#include "oracle.h"

extern "C" {
float oracle_halide_exp(float x) { return hl::halide_exp(x); }
float oracle_halide_log(float x) { return hl::halide_log(x); }
float oracle_halide_pow(float x, float y) { return hl::halide_pow(x, y); }
float oracle_fast_exp(float x) { return hl::fast_exp(x); }
int oracle_div_floor(int a, int b) { return hl::div_floor(a, b); }
int oracle_mod_floor(int a, int b) { return hl::mod_floor(a, b); }
int oracle_num_threads(void) { return omp_get_max_threads(); }
void oracle_set_num_threads(int n) { omp_set_num_threads(n > 0 ? n : 1); }

// out[i] = f(a[i] [, b ...]) over n floats, numbered as the device hook halide_b200_selftest_math numbers them:
// 0 halide_exp, 1 halide_log, 2 fast_exp, 3 clamp01 (clampf(a, 0, 1)), 4 halide_pow(a[i], b[i]),
// 5 clampf(a[i], b[2i], b[2i+1]), 6 lerpf(a[i], b[2i], b[2i+1]), 7 / 8 / 9 evaluate_polynomial with halide_exp's 8, halide_log's
// 10 and an odd-count set of 7 coefficients.  Returns 0, or -1 for an unknown fn.
int oracle_math_vec(int fn, const float *a, const float *b, float *out, long long n) {
    static const float poly_exp[8] = {0.00031965933071842413f, 0.00119156835564003744f, 0.00848988645943932717f,
                                      0.04160188091348320655f, 0.16667983794100929562f, 0.49999899033463041098f,
                                      1.0f, 1.0f};
    static const float poly_log[10] = {0.05111976432738144643f, -0.11793923497136414580f, 0.14971993724699017569f,
                                       -0.16862004708254804686f, 0.19980668101718729313f, -0.24991211576292837737f,
                                       0.33333435275479328386f, -0.50000106292873236491f, 1.0f, 0.0f};
    static const float poly_odd[7] = {0.25f, -0.5f, 0.0f, 1.5f, -2.0f, 0.125f, 3.0f};
    if (fn < 0 || fn > 9) return -1;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; i++) {
        const float x = a[i];
        float r;
        switch (fn) {
        case 0: r = hl::halide_exp(x); break;
        case 1: r = hl::halide_log(x); break;
        case 2: r = hl::fast_exp(x); break;
        case 3: r = hl::clampf(x, 0.0f, 1.0f); break;
        case 4: r = hl::halide_pow(x, b[i]); break;
        case 5: r = hl::clampf(x, b[2 * i], b[2 * i + 1]); break;
        case 6: r = hl::lerpf(x, b[2 * i], b[2 * i + 1]); break;
        case 7: r = hl::evaluate_polynomial(x, poly_exp, 8); break;
        case 8: r = hl::evaluate_polynomial(x, poly_log, 10); break;
        default: r = hl::evaluate_polynomial(x, poly_odd, 7); break;
        }
        out[i] = r;
    }
    return 0;
}
}
