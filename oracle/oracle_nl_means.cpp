// oracle/oracle_nl_means.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle.h).
//
// CPU restatement of apps/nl_means/nl_means_generator.cpp:24-63, op order per SURVEY.md
// Appendix B.  Parity status: UNPINNED by the reference.  Float pipeline: the CUDA path matches it
// bit for bit; tests/test_nl_means_exact.py pins it against a float64 restatement.
#include <vector>

#include "halide_math.h"
#include "oracle.h"

extern "C" int oracle_nl_means(const oracle_image_t *in, int patch_size, int search_area, float sigma,
                               const oracle_image_t *out) {
    const float *ib = (const float *)in->base;
    float *ob = (float *)out->base;
    const int ox = out->min[0], oy = out->min[1], W = out->extent[0], H = out->extent[1];
    if (W <= 0 || H <= 0) return 0;
    auto clamped = [&](int x, int y, int c) -> float {
        x = hl::clampi(x, in->min[0], in->min[0] + in->extent[0] - 1);
        y = hl::clampi(y, in->min[1], in->min[1] + in->extent[1] - 1);
        c = hl::clampi(c, in->min[2], in->min[2] + in->extent[2] - 1);
        return ib[(int64_t)(x - in->min[0]) * in->stride[0] + (int64_t)(y - in->min[1]) * in->stride[1] +
                  (int64_t)(c - in->min[2]) * in->stride[2]];
    };
    // inv_sigma_sq = -1.0f / (sigma * sigma * patch_size * patch_size) (generator :24)
    const float inv_sigma_sq = -1.0f / (((sigma * sigma) * (float)patch_size) * (float)patch_size);
    const int p0 = -(patch_size / 2), s0 = -(search_area / 2);
    auto d = [&](int x, int y, int dx, int dy) -> float {  // generator :32-37: pow(.,2) == e*e, channels 0..2
        float s = 0.0f;
        for (int c = 0; c < 3; c++) {
            float e = clamped(x, y, c) - clamped(x + dx, y + dy, c);
            s = s + e * e;
        }
        return s;
    };
#pragma omp parallel for schedule(dynamic, 4)
    for (int y = oy; y < oy + H; y++) {
        for (int x = ox; x < ox + W; x++) {
            float sum[4] = {0.f, 0.f, 0.f, 0.f};
            for (int sy = s0; sy < s0 + search_area; sy++) {       // s_dom.y outer
                for (int sx = s0; sx < s0 + search_area; sx++) {   // s_dom.x inner
                    float bd = 0.0f;                               // blur_d = sum_x(blur_d_y)
                    for (int px = p0; px < p0 + patch_size; px++) {
                        float bdy = 0.0f;                          // blur_d_y = sum_y(d)
                        for (int py = p0; py < p0 + patch_size; py++) bdy = bdy + d(x + px, y + py, sx, sy);
                        bd = bd + bdy;
                    }
                    float w = hl::fast_exp(bd * inv_sigma_sq);
                    sum[0] = sum[0] + w * clamped(x + sx, y + sy, 0);
                    sum[1] = sum[1] + w * clamped(x + sx, y + sy, 1);
                    sum[2] = sum[2] + w * clamped(x + sx, y + sy, 2);
                    sum[3] = sum[3] + w * 1.0f;
                }
            }
            for (int c = 0; c < 3; c++) {
                float v = hl::clampf(sum[c] / sum[3], 0.0f, 1.0f);
                ob[(int64_t)(x - ox) * out->stride[0] + (int64_t)(y - oy) * out->stride[1] + (int64_t)c * out->stride[2]] = v;
            }
        }
    }
    return 0;
}
