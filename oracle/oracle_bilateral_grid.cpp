// oracle/oracle_bilateral_grid.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle.h).
//
// CPU restatement of apps/bilateral_grid/bilateral_grid_generator.cpp:17-67 (any s_sigma), op
// order per SURVEY.md Appendix B.  Parity status: UNPINNED by the reference (no golden output;
// libHalide unbuildable here); pinned instead to tests/bilateral_grid_exact.py's float64
// restatement.  The clamp is Halide's select-based min / max (hl::clampf): NaN pixels become 1.
// The CUDA path is compared bit for bit: the any-S kernels on any input, s_sigma = 8 wherever its
// bin sums are exact (frames of multiples of 2^-16); only s_sigma = 8 on arbitrary float data is
// compared within 1e-4 relative, because its histogram adds each bin as two 4-column partial sums.
#include <algorithm>
#include <vector>

#include "halide_math.h"
#include "oracle.h"

extern "C" int oracle_bilateral_grid(const oracle_image_t *in, float r_sigma, const oracle_image_t *out, int s_sigma) {
    const float *ib = (const float *)in->base;
    float *ob = (float *)out->base;
    const int ox = out->min[0], oy = out->min[1], W = out->extent[0], H = out->extent[1];
    if (W <= 0 || H <= 0) return 0;
    const int S = s_sigma;
    auto in_at = [&](int x, int y) -> float {
        return ib[(int64_t)(x - in->min[0]) * in->stride[0] + (int64_t)(y - in->min[1]) * in->stride[1]];
    };
    auto clamped = [&](int x, int y) -> float {  // repeat_edge (generator :17)
        x = hl::clampi(x, in->min[0], in->min[0] + in->extent[0] - 1);
        y = hl::clampi(y, in->min[1], in->min[1] + in->extent[1] - 1);
        return in_at(x, y);
    };
    const float inv_r = 1.0f / r_sigma;
    // grid cells the slice touches: xi .. xi+1, grown by 2 for blury and 2 for blurx
    const int gx0 = hl::div_floor(ox, S) - 2, gx1 = hl::div_floor(ox + W - 1, S) + 1 + 2;
    const int gy0 = hl::div_floor(oy, S) - 2, gy1 = hl::div_floor(oy + H - 1, S) + 1 + 2;
    const int zmax = (int)(1.0f * inv_r + 0.5f);  // largest bin written (val = 1)
    // histogram z in [-2, zmax+2+1] so that blurz over [0, zmax+1] reads in range
    const int hz0 = -2, hz1 = zmax + 3, bz0 = 0, bz1 = zmax + 1;
    const int GW = gx1 - gx0 + 1, GH = gy1 - gy0 + 1, HZ = hz1 - hz0 + 1, BZ = bz1 - bz0 + 1;
    std::vector<float> hist((size_t)GW * GH * HZ * 2, 0.f);
    auto H_at = [&](int x, int y, int z, int c) -> float & {
        return hist[(((size_t)(y - gy0) * GW + (x - gx0)) * HZ + (z - hz0)) * 2 + c];
    };
#pragma omp parallel for schedule(static)
    for (int gy = gy0; gy <= gy1; gy++) {
        for (int gx = gx0; gx <= gx1; gx++) {
            for (int ry = 0; ry < S; ry++) {      // RDom r(0,S,0,S): r.x innermost (generator :20)
                for (int rx = 0; rx < S; rx++) {
                    float val = clamped(gx * S + rx - S / 2, gy * S + ry - S / 2);
                    val = hl::clampf(val, 0.0f, 1.0f);
                    int zi = (int)(val * inv_r + 0.5f);
                    H_at(gx, gy, zi, 0) += val;
                    H_at(gx, gy, zi, 1) += 1.0f;
                }
            }
        }
    }
    auto blur5 = [](float a, float b, float c, float d, float e) -> float {
        return (((a + b * 4.0f) + c * 6.0f) + d * 4.0f) + e;  // generator :33-47
    };
    std::vector<float> bz((size_t)GW * GH * BZ * 2), bx((size_t)GW * GH * BZ * 2), by((size_t)GW * GH * BZ * 2);
    auto idx = [&](int x, int y, int z, int c) -> size_t {
        return (((size_t)(y - gy0) * GW + (x - gx0)) * BZ + (z - bz0)) * 2 + c;
    };
#pragma omp parallel for schedule(static)
    for (int gy = gy0; gy <= gy1; gy++)
        for (int gx = gx0; gx <= gx1; gx++)
            for (int z = bz0; z <= bz1; z++)
                for (int c = 0; c < 2; c++)
                    bz[idx(gx, gy, z, c)] = blur5(H_at(gx, gy, z - 2, c), H_at(gx, gy, z - 1, c), H_at(gx, gy, z, c),
                                                  H_at(gx, gy, z + 1, c), H_at(gx, gy, z + 2, c));
#pragma omp parallel for schedule(static)
    for (int gy = gy0; gy <= gy1; gy++)
        for (int gx = gx0 + 2; gx <= gx1 - 2; gx++)
            for (int z = bz0; z <= bz1; z++)
                for (int c = 0; c < 2; c++)
                    bx[idx(gx, gy, z, c)] = blur5(bz[idx(gx - 2, gy, z, c)], bz[idx(gx - 1, gy, z, c)], bz[idx(gx, gy, z, c)],
                                                  bz[idx(gx + 1, gy, z, c)], bz[idx(gx + 2, gy, z, c)]);
#pragma omp parallel for schedule(static)
    for (int gy = gy0 + 2; gy <= gy1 - 2; gy++)
        for (int gx = gx0 + 2; gx <= gx1 - 2; gx++)
            for (int z = bz0; z <= bz1; z++)
                for (int c = 0; c < 2; c++)
                    by[idx(gx, gy, z, c)] = blur5(bx[idx(gx, gy - 2, z, c)], bx[idx(gx, gy - 1, z, c)], bx[idx(gx, gy, z, c)],
                                                  bx[idx(gx, gy + 1, z, c)], bx[idx(gx, gy + 2, z, c)]);
    const float inv_s = hl::recip_const((float)S);
#pragma omp parallel for schedule(static)
    for (int y = oy; y < oy + H; y++) {
        for (int x = ox; x < ox + W; x++) {
            float val = hl::clampf(in_at(x, y), 0.0f, 1.0f);  // unclamped coordinates (generator :50)
            float zv = val * inv_r;
            int zi = (int)zv;
            float zf = zv - (float)zi;
            float xf = (float)hl::mod_floor(x, S) * inv_s;
            float yf = (float)hl::mod_floor(y, S) * inv_s;
            int xi = hl::div_floor(x, S), yi = hl::div_floor(y, S);
            float interp[2];
            for (int c = 0; c < 2; c++) {
                auto B = [&](int xx, int yy, int zz) { return by[idx(xx, yy, zz, c)]; };
                interp[c] = hl::lerpf(
                    hl::lerpf(hl::lerpf(B(xi, yi, zi), B(xi + 1, yi, zi), xf),
                              hl::lerpf(B(xi, yi + 1, zi), B(xi + 1, yi + 1, zi), xf), yf),
                    hl::lerpf(hl::lerpf(B(xi, yi, zi + 1), B(xi + 1, yi, zi + 1), xf),
                              hl::lerpf(B(xi, yi + 1, zi + 1), B(xi + 1, yi + 1, zi + 1), xf), yf),
                    zf);
            }
            ob[(int64_t)(x - ox) * out->stride[0] + (int64_t)(y - oy) * out->stride[1]] = interp[0] / interp[1];
        }
    }
    return 0;
}
