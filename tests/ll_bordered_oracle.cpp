// tests/ll_bordered_oracle.cpp — TEST INFRASTRUCTURE: local_laplacian evaluated with every pyramid level stored only
// inside its constant border, for pyramid depths the literal oracle (oracle/oracle_local_laplacian.cpp) cannot hold in
// memory.  Compiled on first use by tests/ll_bordered.py, with oracle/Makefile's parity flags, into a library of its own.
//
// The literal oracle is included in place: this evaluation shares its region arithmetic (regions), level storage (Plane),
// remap table (oracle_ll_remap) and upsample for the output-side levels, and differs only in where the Gaussian-side
// levels are stored and how they are read.
#include "oracle_local_laplacian.cpp"

// ---- the same pipeline with every level stored only inside its constant border -------------------------------------
// oracle_local_laplacian evaluates each level on the whole region bounds inference gives it, which grows by about
// 2^(J+1) px per axis at level 0: past J = 11 or so that no longer fits in memory even for a 1x1 output.  But only the
// input is edge-clamped, so every level is constant beyond a border: level 0 (gray, gPyramid[0]) for x <= L_0 = the
// input's first column and x >= R_0 = its last, and if level j is constant for x <= L_j and x >= R_j, level j+1 (which
// reads 2x-1 .. 2x+2) is constant for x <= L_{j+1} = floor((L_j - 2) / 2) and x >= R_{j+1} = floor((R_j + 2) / 2);
// likewise for rows.  So a level stored on its region cut to [L_j, R_j] and read with coordinates clamped into that cut
// holds every value of the literal evaluation.  tests/test_ll_pyramid_levels.py checks the two bit for bit at J <= 11.
namespace {

Rng cut(Rng g, int lo, int hi) { return {std::max(g.lo, lo), std::min(g.hi, hi)}; }

inline float at_clamped(const Plane &p, int x, int y, int k) {
    return p.at(hl::clampi(x, p.X.lo, p.X.hi), hl::clampi(y, p.Y.lo, p.Y.hi), k);
}

// downsample(f) over the region of `dst`, reading src clamped into its stored region
void downsample_clamped(const Plane &src, Plane &dst) {
    const int xlo = 2 * dst.X.lo - 1, xhi = 2 * dst.X.hi + 2;
#pragma omp parallel
    {
        std::vector<float> tmp(xhi - xlo + 1);
#pragma omp for collapse(2) schedule(static)
        for (int k = 0; k < dst.K; k++) {
            for (int y = dst.Y.lo; y <= dst.Y.hi; y++) {
                for (int x = xlo; x <= xhi; x++) {
                    tmp[x - xlo] = ((at_clamped(src, x, 2 * y - 1, k) +
                                     3.0f * (at_clamped(src, x, 2 * y, k) + at_clamped(src, x, 2 * y + 1, k))) +
                                    at_clamped(src, x, 2 * y + 2, k)) * 0.125f;
                }
                for (int x = dst.X.lo; x <= dst.X.hi; x++) {
                    const float *t = &tmp[2 * x - 1 - xlo];
                    dst.at(x, y, k) = ((t[0] + 3.0f * (t[1] + t[2])) + t[3]) * 0.125f;
                }
            }
        }
    }
}

inline float upsample_clamped(const Plane &f, int x, int y, int k) {
    const float wx = (float)(hl::mod_floor(x, 2) * 2 + 1) * 0.25f;
    const float wy = (float)(hl::mod_floor(y, 2) * 2 + 1) * 0.25f;
    const int xa = hl::div_floor(x + 1, 2), xb = hl::div_floor(x - 1, 2);
    const int ya = hl::div_floor(y + 1, 2), yb = hl::div_floor(y - 1, 2);
    const float upx_a = hl::lerpf(at_clamped(f, xa, ya, k), at_clamped(f, xb, ya, k), wx);
    const float upx_b = hl::lerpf(at_clamped(f, xa, yb, k), at_clamped(f, xb, yb, k), wx);
    return hl::lerpf(upx_a, upx_b, wy);
}

}  // namespace

extern "C" int oracle_local_laplacian_bordered(const oracle_image_t *in, int levels, float alpha, float beta,
                                               const oracle_image_t *out, int J) {
    if (levels < 2 || J < 1 || J > 20) return -1;
    const uint16_t *ibase = (const uint16_t *)in->base;
    uint16_t *obase = (uint16_t *)out->base;
    const int ox = out->min[0], oy = out->min[1], oc = out->min[2];
    const int W = out->extent[0], H = out->extent[1], C = out->extent[2];
    if (W <= 0 || H <= 0 || C <= 0) return 0;

    auto in_clamped = [&](int x, int y, int c) -> uint16_t {
        x = hl::clampi(x, in->min[0], in->min[0] + in->extent[0] - 1);
        y = hl::clampi(y, in->min[1], in->min[1] + in->extent[1] - 1);
        c = hl::clampi(c, in->min[2], in->min[2] + in->extent[2] - 1);
        return ibase[(int64_t)(x - in->min[0]) * in->stride[0] + (int64_t)(y - in->min[1]) * in->stride[1] +
                     (int64_t)(c - in->min[2]) * in->stride[2]];
    };

    std::vector<Rng> OX, GX, OY, GY;
    regions(ox, ox + W - 1, J, OX, GX);
    regions(oy, oy + H - 1, J, OY, GY);
    // stored regions: G_j cut to the level's constant border [L_j, R_j] (per axis)
    std::vector<Rng> SX(J), SY(J);
    int lx = in->min[0], rx = in->min[0] + in->extent[0] - 1, ly = in->min[1], ry = in->min[1] + in->extent[1] - 1;
    for (int j = 0; j < J; j++) {
        if (j > 0) {
            lx = hl::div_floor(lx - 2, 2); rx = hl::div_floor(rx + 2, 2);
            ly = hl::div_floor(ly - 2, 2); ry = hl::div_floor(ry + 2, 2);
        }
        SX[j] = cut(GX[j], lx, rx);
        SY[j] = cut(GY[j], ly, ry);
        if (SX[j].n() <= 0 || SY[j].n() <= 0) return -1;  // (only if the input does not cover the output)
    }

    const int K = levels;
    const int lut_half = 256 * (levels - 1);
    std::vector<float> lut(2 * lut_half + 1);
    for (int i = -lut_half; i <= lut_half; i++) lut[i + lut_half] = oracle_ll_remap(i, alpha);
    const float flm1 = (float)(levels - 1);
    const float inv_lm1 = 1.0f / flm1;

    Plane gray;
    gray.init(SX[0], SY[0], 1);
#pragma omp parallel for schedule(static)
    for (int y = SY[0].lo; y <= SY[0].hi; y++) {
        for (int x = SX[0].lo; x <= SX[0].hi; x++) {
            const float f0 = hl::div_const((float)in_clamped(x, y, 0), 65535.0f);
            const float f1 = hl::div_const((float)in_clamped(x, y, 1), 65535.0f);
            const float f2 = hl::div_const((float)in_clamped(x, y, 2), 65535.0f);
            gray.at(x, y, 0) = (0.299f * f0 + 0.587f * f1) + 0.114f * f2;
        }
    }
    auto gp0 = [&](int x, int y, int k) -> float {
        const float g = at_clamped(gray, x, y, 0);
        const float level = (float)k * inv_lm1;
        int idx = (int)((g * flm1) * 256.0f);
        idx = hl::clampi(idx, 0, (levels - 1) * 256);
        return ((beta * (g - level)) + level) + lut[idx - 256 * k + lut_half];
    };

    std::vector<Plane> gP(J), inG(J);
    if (J > 1) {
        gP[1].init(SX[1], SY[1], K);
        const int xlo = 2 * SX[1].lo - 1, xhi = 2 * SX[1].hi + 2;
#pragma omp parallel
        {
            std::vector<float> tmp(xhi - xlo + 1);
#pragma omp for collapse(2) schedule(static)
            for (int k = 0; k < K; k++) {
                for (int y = SY[1].lo; y <= SY[1].hi; y++) {
                    for (int x = xlo; x <= xhi; x++) {
                        tmp[x - xlo] = ((gp0(x, 2 * y - 1, k) + 3.0f * (gp0(x, 2 * y, k) + gp0(x, 2 * y + 1, k))) +
                                        gp0(x, 2 * y + 2, k)) * 0.125f;
                    }
                    for (int x = SX[1].lo; x <= SX[1].hi; x++) {
                        const float *t = &tmp[2 * x - 1 - xlo];
                        gP[1].at(x, y, k) = ((t[0] + 3.0f * (t[1] + t[2])) + t[3]) * 0.125f;
                    }
                }
            }
        }
        inG[1].init(SX[1], SY[1], 1);
        downsample_clamped(gray, inG[1]);
    }
    for (int j = 2; j < J; j++) {
        gP[j].init(SX[j], SY[j], K);
        downsample_clamped(gP[j - 1], gP[j]);
        inG[j].init(SX[j], SY[j], 1);
        downsample_clamped(inG[j - 1], inG[j]);
    }

    std::vector<Plane> outG(J);
    for (int j = J - 1; j >= 0; j--) {
        outG[j].init(OX[j], OY[j], 1);
#pragma omp parallel for schedule(static)
        for (int y = OY[j].lo; y <= OY[j].hi; y++) {
            for (int x = OX[j].lo; x <= OX[j].hi; x++) {
                const float ing = (j == 0) ? at_clamped(gray, x, y, 0) : at_clamped(inG[j], x, y, 0);
                const float level = ing * flm1;
                const int li = hl::clampi((int)level, 0, levels - 2);
                const float lf = level - (float)li;
                float l0, l1;
                const float g0 = (j == 0) ? gp0(x, y, li) : at_clamped(gP[j], x, y, li);
                const float g1 = (j == 0) ? gp0(x, y, li + 1) : at_clamped(gP[j], x, y, li + 1);
                if (j == J - 1) {
                    l0 = g0;
                    l1 = g1;
                } else {
                    l0 = g0 - upsample_clamped(gP[j + 1], x, y, li);
                    l1 = g1 - upsample_clamped(gP[j + 1], x, y, li + 1);
                }
                const float outl = (1.0f - lf) * l0 + lf * l1;
                outG[j].at(x, y, 0) = (j == J - 1) ? outl : upsample_at(outG[j + 1], x, y, 0) + outl;
            }
        }
    }

    const float eps = 0.01f;
#pragma omp parallel for collapse(2) schedule(static)
    for (int c = oc; c < oc + C; c++) {
        for (int y = oy; y < oy + H; y++) {
            for (int x = ox; x < ox + W; x++) {
                const uint16_t iv = ibase[(int64_t)(x - in->min[0]) * in->stride[0] + (int64_t)(y - in->min[1]) * in->stride[1] +
                                          (int64_t)(c - in->min[2]) * in->stride[2]];
                const float color = ((float)iv * (outG[0].at(x, y, 0) + eps)) / (at_clamped(gray, x, y, 0) + eps);
                const float cl = hl::clampf(color, 0.0f, 65535.0f);
                obase[(int64_t)(x - ox) * out->stride[0] + (int64_t)(y - oy) * out->stride[1] +
                      (int64_t)(c - oc) * out->stride[2]] = (uint16_t)cl;
            }
        }
    }
    return 0;
}
