// camera_pipe.cu — camera_pipe(input, matrix_3200, matrix_7000, color_temp, gamma, contrast,
// sharpen_strength, blackLevel, whiteLevel, processed) for sm_90a.
//
// Reference algorithm: apps/camera_pipe/camera_pipe_generator.cpp — shift(16,12) :412, hot-pixel suppression
// :240-249, GRBG deinterleave :251-261, gradient-directed demosaic :57-146, 3x4 Q8.8 colour matrix :263-295,
// 1024-entry tone curve :297-367, 1-2-1 unsharp mask :369-404.  Integer pipeline (uint16 raw -> uint8 RGB) with
// Halide's no-promotion typing; bit-exact against oracle/oracle_camera_pipe.cpp.
//
// HBM-bound by construction: 5 algorithmic bytes per output pixel (2 raw + 3 out).  Like the reference's own GPU
// schedule (generator :471-497) every intermediate of a tile lives in shared memory, so the frame is read
// once and written once:
//   cp_tables_kernel   12-entry Q8.8 matrix, 1024-entry curve (halide_pow), sharpen strength — once per call
//   camera_pipe_kernel one 64x32 output tile per block and frame (blockIdx.z walks the frames of a burst):
//        raw (+apron) -> smem -> denoised -> g_r/g_b at half resolution -> demosaic + matrix + curve (u8, tile+1)
//        -> unsharp mask -> 4 pixels per thread, stored as one 32-bit word per channel (planar output) or, for a
//        pixel-interleaved output, as the 4 pixels' samples side by side (three 32-bit words for dense RGB)
#include <algorithm>

#include "hb_common.h"
#include "hl_math.cuh"

namespace {

typedef uint16_t u16;
typedef int16_t i16;
typedef uint8_t u8;

constexpr int TW = 64, TH = 32;              // output tile
constexpr int CW = TW + 2, CH = TH + 2;      // curved tile (unsharp apron 1)
constexpr int HW = TW / 2 + 3, HH = TH / 2 + 3;  // half-res sites needed by the curved tile (any parity of the origin)
constexpr int GW = HW + 2, GH = HH + 2;      // g_r / g_b tile (demosaic apron 1)
constexpr int DW = 2 * GW, DH = 2 * GH;      // denoised tile (full-res)
constexpr int RW = DW + 4, RH = DH + 4;      // raw tile (hot-pixel apron 2)

struct CPTables {
    i16 matrix[12];  // [y*4 + x]
    u8 s32;
    u8 curve[1024];
};

struct CPParams {
    const u16 *in;  // element at the input mins (x, y) of the output's first frame
    int64_t in_sy, in_sn;
    int in_x0, in_y0, in_w, in_h;
    u8 *out;  // element at the output mins
    int64_t out_sy, out_sc, out_sn;
    int out_px;  // interleaved output: the pixel pitch (out_sc is 1)
    int out_x0, out_y0, W, H, C, out_c0, N;
    const CPTables *tab;
};

__device__ __forceinline__ u16 avg16(u16 a, u16 b) { return (u16)(((uint32_t)a + (uint32_t)b + 1u) >> 1); }  // generator :16-19
__device__ __forceinline__ u16 absd16(u16 a, u16 b) { return a > b ? (u16)(a - b) : (u16)(b - a); }
__device__ __forceinline__ u8 avg8(u8 a, u8 b) { return (u8)(((uint32_t)a + (uint32_t)b + 1u) >> 1); }
__device__ __forceinline__ u8 blur121_8(u8 a, u8 b, u8 c) { return avg8(avg8(a, c), b); }
__device__ __forceinline__ int fdiv2(int a) { return a >> 1; }

// ---- tables: colour matrix, tone curve, sharpen strength (generator :263-271, :297-332, :372) --------------------
__global__ void cp_tables_kernel(CPTables *t, const float *m3200, int64_t m32_sx, int64_t m32_sy, const float *m7000, int64_t m70_sx,
                                 int64_t m70_sy, float color_temp, float gamma, float contrast, float sharpen_strength,
                                 int blackLevel, int whiteLevel, float inv_c_diff) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x < 12) {
        // alpha = (1/kelvin - 1/3200) / (1/7000 - 1/3200); the constant divisor is folded to a reciprocal multiply
        const float c3200 = 1.0f / 3200;
        float alpha = __fmul_rn(__fsub_rn(__fdiv_rn(1.0f, color_temp), c3200), inv_c_diff);
        int mx = x & 3, my = x >> 2;
        float a = m3200[mx * m32_sx + my * m32_sy], b = m7000[mx * m70_sx + my * m70_sy];
        float val = __fadd_rn(__fmul_rn(a, alpha), __fmul_rn(b, __fsub_rn(1.0f, alpha)));
        t->matrix[x] = (i16)(int)__fmul_rn(val, 256.0f);
    }
    if (x == 12) {
        float s = fmaxf(__fmul_rn(sharpen_strength, 32.0f), 0.0f);  // u8_sat: clamp low, saturate high, truncate
        t->s32 = s >= 255.0f ? (u8)255 : (u8)(int)s;
    }
    if (x < 1024) {
        const int minRaw = 0 + blackLevel, maxRaw = whiteLevel;
        const float invRange = __fdiv_rn(1.0f, (float)(maxRaw - minRaw));
        const float b = __fsub_rn(2.0f, hl::halide_pow(2.0f, __fmul_rn(contrast, 0.01f)));  // contrast / 100.0f folds to * 0.01f
        const float a = __fsub_rn(2.0f, __fmul_rn(2.0f, b));
        float xf = hl::clampf(__fmul_rn((float)(x - minRaw), invRange), 0.0f, 1.0f);
        float g = hl::halide_pow(xf, __fdiv_rn(1.0f, gamma));
        float omg = __fsub_rn(1.0f, g);
        float z_hi = __fsub_rn(1.0f, __fadd_rn(__fmul_rn(__fmul_rn(a, omg), omg), __fmul_rn(b, omg)));
        float z_lo = __fadd_rn(__fmul_rn(__fmul_rn(a, g), g), __fmul_rn(b, g));
        float z = g > 0.5f ? z_hi : z_lo;
        u8 val = (u8)(int)hl::clampf(__fadd_rn(__fmul_rn(z, 255.0f), 0.5f), 0.0f, 255.0f);
        t->curve[x] = x <= minRaw ? (u8)0 : (x > maxRaw ? (u8)255 : val);
    }
}

// Unsharp mask (generator :384-401) of output tile row ly, pixels 4q .. 4q + 3, of one curved plane: the 4 bytes of a
// little-endian word.
__device__ __forceinline__ uint32_t unsharp4(const u8 (*cv)[CW + 2], int ly, int q, int s32) {
    uint32_t packed = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        int lx = 4 * q + k;  // tile-local output x; curved tile index = lx + 1, ly + 1
        const int cx = lx + 1, cy = ly + 1;
        u8 uy_m = blur121_8(cv[cy - 1][cx - 1], cv[cy][cx - 1], cv[cy + 1][cx - 1]);
        u8 uy_0 = blur121_8(cv[cy - 1][cx], cv[cy][cx], cv[cy + 1][cx]);
        u8 uy_p = blur121_8(cv[cy - 1][cx + 1], cv[cy][cx + 1], cv[cy + 1][cx + 1]);
        u8 unsharp = blur121_8(uy_m, uy_0, uy_p);
        int in_v = (int)cv[cy][cx];
        i16 mask = (i16)(in_v - (int)unsharp);
        i16 prod = (i16)((int)mask * s32);          // i16 * u8 stays i16 and wraps (src/IROperator.cpp:769-816)
        int sum = (int)(i16)(in_v + ((int)prod >> 5));  // floor division by 32
        packed |= (uint32_t)min(max(sum, 0), 255) << (8 * k);
    }
    return packed;
}

// ---- the fused tile kernel -------------------------------------------------------------------------------------
// IL: the output is pixel-interleaved (the channels of a pixel adjacent, pixels p.out_px bytes apart).
template<bool IL>
__global__ void __launch_bounds__(256) camera_pipe_kernel(CPParams p) {
    __shared__ u16 s_raw[RH][RW];
    __shared__ u16 s_den[DH][DW];
    __shared__ u16 s_gr[GH][GW];  // g_r at half-res sites
    __shared__ u16 s_gb[GH][GW];  // g_b
    __shared__ u8 s_cv[3][CH][CW + 2];
    __shared__ u8 s_curve[1024];
    __shared__ int s_m[12];
    const int X0 = p.out_x0 + blockIdx.x * TW, Y0 = p.out_y0 + blockIdx.y * TH;  // absolute output coords of the tile
    // half-res origin of the sites the curved tile [X0-1, X0+TW] needs, grown by 1 for g_r / g_b
    const int gx0 = fdiv2(X0 - 1) - 1, gy0 = fdiv2(Y0 - 1) - 1;
    const int dx0 = 2 * gx0, dy0 = 2 * gy0;  // denoised tile origin (full-res, shifted coordinates)
    const int rx0 = dx0 - 2, ry0 = dy0 - 2;  // raw tile origin

    for (int i = threadIdx.x; i < 1024; i += 256) s_curve[i] = p.tab->curve[i];
    if (threadIdx.x < 12) s_m[threadIdx.x] = (int)p.tab->matrix[threadIdx.x];
    const int s32 = (int)p.tab->s32;
    // Frames n = blockIdx.z, + gridDim.z, ...: one launch serves any burst.  (No barrier is needed between frames: the
    // raw tile, the first array a frame writes, was last read before three of the previous frame's barriers.)
    for (int n = blockIdx.z; n < p.N; n += gridDim.z) {
        const int tid = hl::frame_tid();
        const u16 *in = p.in + (int64_t)n * p.in_sn;
        // raw tile: shifted(x,y) = input(x+16, y+12) (generator :412).  Coordinates the output never depends on may fall
        // outside the buffer at the frame's far edges of the last tiles; they are clamped (values unused).
        for (int i = tid; i < RW * RH; i += 256) {
            int ly = i / RW, lx = i - ly * RW;
            int ax = min(max(rx0 + lx + 16 - p.in_x0, 0), p.in_w - 1);  // buffer-relative, kept inside the buffer
            int ay = min(max(ry0 + ly + 12 - p.in_y0, 0), p.in_h - 1);
            s_raw[ly][lx] = __ldg(in + (int64_t)ay * p.in_sy + ax);
        }
        __syncthreads();
        // denoised = clamp(in, 0, max of the 4 neighbours at distance 2) (generator :240-249)
        for (int i = tid; i < DW * DH; i += 256) {
            int ly = i / DW, lx = i - ly * DW;
            int ry = ly + 2, rx = lx + 2;
            u16 a = max(max(s_raw[ry][rx - 2], s_raw[ry][rx + 2]), max(s_raw[ry - 2][rx], s_raw[ry + 2][rx]));
            s_den[ly][lx] = min(s_raw[ry][rx], a);
        }
        __syncthreads();
        // deinterleaved channel accessors at half-res site (sx, sy) relative to (gx0, gy0) (generator :57-60, :255-259)
#define G_GR(sx, sy) s_den[2 * (sy)][2 * (sx)]
#define R_R(sx, sy) s_den[2 * (sy)][2 * (sx) + 1]
#define B_B(sx, sy) s_den[2 * (sy) + 1][2 * (sx)]
#define G_GB(sx, sy) s_den[2 * (sy) + 1][2 * (sx) + 1]
        // green at red and blue sites (generator :70-82); border sites of the tile whose taps fall outside are never consumed
        for (int i = tid; i < GW * GH; i += 256) {
            int sy = i / GW, sx = i - sy * GW;
            int ym = max(sy - 1, 0), yp = min(sy + 1, GH - 1), xm = max(sx - 1, 0), xp = min(sx + 1, GW - 1);
            u16 gv_r = avg16(G_GB(sx, ym), G_GB(sx, sy)), gvd_r = absd16(G_GB(sx, ym), G_GB(sx, sy));
            u16 gh_r = avg16(G_GR(xp, sy), G_GR(sx, sy)), ghd_r = absd16(G_GR(xp, sy), G_GR(sx, sy));
            s_gr[sy][sx] = ghd_r < gvd_r ? gh_r : gv_r;
            u16 gv_b = avg16(G_GR(sx, yp), G_GR(sx, sy)), gvd_b = absd16(G_GR(sx, yp), G_GR(sx, sy));
            u16 gh_b = avg16(G_GB(xm, sy), G_GB(sx, sy)), ghd_b = absd16(G_GB(xm, sy), G_GB(sx, sy));
            s_gb[sy][sx] = ghd_b < gvd_b ? gh_b : gv_b;
        }
        __syncthreads();
        // demosaic + colour matrix + curve on the curved tile [X0-1, X0+TW] x [Y0-1, Y0+TH]
        for (int i = tid; i < CW * CH; i += 256) {
            int ly = i / CW, lx = i - ly * CW;
            int X = X0 - 1 + lx, Y = Y0 - 1 + ly;
            int x = fdiv2(X) - gx0, y = fdiv2(Y) - gy0;  // half-res site within the tiles
            bool xe = (X & 1) == 0, ye = (Y & 1) == 0;
            u16 r, g, b;
            if (ye && xe) {  // gr site (generator :89-96)
                g = G_GR(x, y);
                u16 corr = (u16)(g - avg16(s_gr[y][x], s_gr[y][x - 1]));
                r = (u16)(corr + avg16(R_R(x - 1, y), R_R(x, y)));
                corr = (u16)(g - avg16(s_gb[y][x], s_gb[y - 1][x]));
                b = (u16)(corr + avg16(B_B(x, y), B_B(x, y - 1)));
            } else if (ye) {  // r site (generator :121-130)
                r = R_R(x, y);
                g = s_gr[y][x];
                u16 corr = (u16)(g - avg16(s_gb[y][x], s_gb[y - 1][x + 1]));
                u16 bp = (u16)(corr + avg16(B_B(x, y), B_B(x + 1, y - 1)));
                u16 bpd = absd16(B_B(x, y), B_B(x + 1, y - 1));
                corr = (u16)(g - avg16(s_gb[y][x + 1], s_gb[y - 1][x]));
                u16 bn = (u16)(corr + avg16(B_B(x + 1, y), B_B(x, y - 1)));
                u16 bnd = absd16(B_B(x + 1, y), B_B(x, y - 1));
                b = bpd < bnd ? bp : bn;
            } else if (xe) {  // b site (generator :111-119)
                b = B_B(x, y);
                g = s_gb[y][x];
                u16 corr = (u16)(g - avg16(s_gr[y][x], s_gr[y + 1][x - 1]));
                u16 rp = (u16)(corr + avg16(R_R(x, y), R_R(x - 1, y + 1)));
                u16 rpd = absd16(R_R(x, y), R_R(x - 1, y + 1));
                corr = (u16)(g - avg16(s_gr[y][x - 1], s_gr[y + 1][x]));
                u16 rn = (u16)(corr + avg16(R_R(x - 1, y), R_R(x, y + 1)));
                u16 rnd = absd16(R_R(x - 1, y), R_R(x, y + 1));
                r = rpd < rnd ? rp : rn;
            } else {  // gb site (generator :98-102)
                g = G_GB(x, y);
                u16 corr = (u16)(g - avg16(s_gr[y][x], s_gr[y + 1][x]));
                r = (u16)(corr + avg16(R_R(x, y), R_R(x, y + 1)));
                corr = (u16)(g - avg16(s_gb[y][x], s_gb[y][x + 1]));
                b = (u16)(corr + avg16(B_B(x, y), B_B(x + 1, y)));
            }
            // i16 reinterpretation (generator :146), colour matrix in i32 with floor division by 256 (generator :277-292)
            const int ir = (int)(i16)r, ig = (int)(i16)g, ib = (int)(i16)b;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                int acc = ((s_m[c * 4 + 3] + s_m[c * 4 + 0] * ir) + s_m[c * 4 + 1] * ig) + s_m[c * 4 + 2] * ib;
                int cc = (int)(i16)(acc >> 8);
                s_cv[c][ly][lx] = s_curve[min(max(cc, 0), 1023)];
            }
        }
        __syncthreads();
#undef G_GR
#undef R_R
#undef B_B
#undef G_GB
        // unsharp mask (generator :384-401): 4 horizontally adjacent pixels per thread
        u8 *out = p.out + (int64_t)n * p.out_sn;
        if (!IL) {  // planar: one 32-bit store per channel
            for (int i = tid; i < (TW / 4) * TH * 3; i += 256) {
                int c = i / ((TW / 4) * TH), rem = i - c * (TW / 4) * TH;
                int ly = rem / (TW / 4), q = rem - ly * (TW / 4);
                if (c >= p.C) continue;
                int oy = blockIdx.y * TH + ly;
                if (oy >= p.H) continue;
                uint32_t packed = unsharp4(s_cv[p.out_c0 + c], ly, q, s32);  // absolute channel 0..2 -> curved plane
                int ox = blockIdx.x * TW + 4 * q;
                u8 *dst = out + (int64_t)c * p.out_sc + (int64_t)oy * p.out_sy + ox;
                if (ox + 3 < p.W && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
                    *reinterpret_cast<uint32_t *>(dst) = packed;
                } else {
                    for (int k = 0; k < 4; k++)
                        if (ox + k < p.W) dst[k] = (u8)(packed >> (8 * k));
                }
            }
        } else {  // interleaved: all of the output's channels of the 4 pixels
            for (int i = tid; i < (TW / 4) * TH; i += 256) {
                int ly = i / (TW / 4), q = i - ly * (TW / 4);
                int oy = blockIdx.y * TH + ly;
                if (oy >= p.H) continue;
                int ox = blockIdx.x * TW + 4 * q;
                u8 *dst = out + (int64_t)oy * p.out_sy + (int64_t)ox * p.out_px;
                uint32_t packed[3];
#pragma unroll
                for (int c = 0; c < 3; c++) packed[c] = c < p.C ? unsharp4(s_cv[p.out_c0 + c], ly, q, s32) : 0u;
                if (p.out_px == 3 && p.C == 3 && ox + 3 < p.W && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
                    // RGB RGB RGB RGB as three words: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
                    const uint32_t r = packed[0], g = packed[1], b = packed[2];
                    uint32_t *d = reinterpret_cast<uint32_t *>(dst);
                    d[0] = __byte_perm(__byte_perm(r, g, 0x1040), b, 0x3410);
                    d[1] = __byte_perm(__byte_perm(g, b, 0x2051), r, 0x3610);
                    d[2] = __byte_perm(__byte_perm(b, r, 0x3072), g, 0x3710);
                } else {  // exactly the covered samples: pitch 4 (alpha untouched), channel crops, frame edges, odd bases
                    for (int k = 0; k < 4; k++) {
                        if (ox + k >= p.W) break;
                        for (int c = 0; c < p.C; c++) dst[k * p.out_px + c] = (u8)(packed[c] >> (8 * k));
                    }
                }
            }
        }
    }  // frames
}

int64_t est_in[2][2] = {{0, 2592}, {0, 1968}}, est_m[2][2] = {{0, 4}, {0, 3}}, est_out[3][2] = {{0, 2592}, {0, 1968}, {0, 3}};
const int64_t *const est_in_p[4] = {&est_in[0][0], &est_in[0][1], &est_in[1][0], &est_in[1][1]};
const int64_t *const est_m_p[4] = {&est_m[0][0], &est_m[0][1], &est_m[1][0], &est_m[1][1]};
const int64_t *const est_out_p[6] = {&est_out[0][0], &est_out[0][1], &est_out[1][0], &est_out[1][1], &est_out[2][0], &est_out[2][1]};
const halide_scalar_value_t sv[6] = {hb::scalar_f32(3700), hb::scalar_f32(2.0f), hb::scalar_f32(50), hb::scalar_f32(1.0f),
                                     hb::scalar_i32(25), hb::scalar_i32(1023)};
const halide_filter_argument_t kArgs[10] = {
    {"input", halide_argument_kind_input_buffer, 2, {halide_type_uint, 16, 0}, nullptr, nullptr, nullptr, nullptr, est_in_p},
    {"matrix_3200", halide_argument_kind_input_buffer, 2, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_m_p},
    {"matrix_7000", halide_argument_kind_input_buffer, 2, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_m_p},
    {"color_temp", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv[0], nullptr},
    {"gamma", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv[1], nullptr},
    {"contrast", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv[2], nullptr},
    {"sharpen_strength", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv[3], nullptr},
    {"blackLevel", halide_argument_kind_input_scalar, 0, {halide_type_int, 32, 0}, nullptr, nullptr, nullptr, &sv[4], nullptr},
    {"whiteLevel", halide_argument_kind_input_scalar, 0, {halide_type_int, 32, 0}, nullptr, nullptr, nullptr, &sv[5], nullptr},
    {"processed", halide_argument_kind_output_buffer, 3, {halide_type_uint, 8, 0}, nullptr, nullptr, nullptr, nullptr, est_out_p},
};
// The burst entry points: the same buffers with a frame dimension n, input (x, y, n) and output (x, y, c, n).
const halide_filter_argument_t kBatchArgs[2] = {hb::variant(kArgs[0], 1), hb::variant(kArgs[9], 1)};

inline int fdiv(int a, int b) {
    int q = a / b;
    return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

// The raw region camera_pipe reads for output columns [ox, ox + W) and rows [oy, oy + H), by interval arithmetic over the
// stencil chain (no boundary condition anywhere): unsharp +-1 -> half-res sites -> demosaic +-1 site -> denoise +-2 ->
// shift (16,12).  Dimension 2 is left for a burst's frame range.
hb::Region raw_region(int ox, int oy, int W, int H) {
    const int hx0 = fdiv(ox - 1, 2), hx1 = fdiv(ox + W, 2), hy0 = fdiv(oy - 1, 2), hy1 = fdiv(oy + H, 2);
    const int need_x0 = 2 * (hx0 - 1) - 2 + 16, need_x1 = 2 * (hx1 + 1) + 1 + 2 + 16;
    const int need_y0 = 2 * (hy0 - 1) - 2 + 12, need_y1 = 2 * (hy1 + 1) + 1 + 2 + 12;
    return {{need_x0, need_y0}, {need_x1 - need_x0 + 1, need_y1 - need_y0 + 1}, true};
}

// Every camera_pipe entry point, on args = {input, matrix_3200, matrix_7000, processed}: input (x, y) and output (x, y, c)
// for one frame, or input (x, y, n) and output (x, y, c, n) for a burst; args[3].interleaved selects the output layout.
// One cp_tables launch and one tile launch whatever the number of frames.
int run_camera_pipe(hb::Arg *args, float color_temp, float gamma, float contrast, float sharpen_strength, int32_t blackLevel,
                    int32_t whiteLevel, const char *what) {
    int r;
    if ((r = hb::check_args(args, 4))) return r;
    halide_buffer_t *input = args[0].b, *m3200 = args[1].b, *m7000 = args[2].b, *out = args[3].b;
    const hb::Clip c = hb::clip_of(args[0], args[3], 3);  // (output frame n reads input frame n)
    const int ox = out->dim[0].min, oy = out->dim[1].min, W = out->dim[0].extent, H = out->dim[1].extent, N = c.N;
    const hb::Region matrix = {{0, 0}, {4, 3}, true};
    const hb::Region need[4] = {c.with_frames(raw_region(ox, oy, W, H)), matrix, matrix, hb::region_of(out, false)};
    if (hb::answer_bounds_query(args, need, 4)) return 0;
    if ((r = hb::check_shapes(args, 4))) return r;
    if (W <= 0 || H <= 0 || out->dim[2].extent <= 0 || N <= 0) return 0;
    if ((r = hb::check_required(args, need, 4))) return r;
    if (out->dim[2].min < 0 || out->dim[2].min + out->dim[2].extent > 3) {
        return hb::fail(halide_error_code_access_out_of_bounds, "Output buffer processed channel range [%d,%d) is outside [0,3)",
                        out->dim[2].min, out->dim[2].min + out->dim[2].extent);
    }
    if ((r = hb::acquire(args, 4))) return r;
    hb::Scratch scratch;
    CPTables *tab = scratch.get<CPTables>(1);
    if (!tab) return hb::fail(halide_error_code_device_malloc_failed, "camera_pipe: scratch allocation failed");

    CPParams p;
    p.in = (const u16 *)args[0].dev + c.in_off;  // the input frame output frame 0 reads
    p.in_sy = input->dim[1].stride;
    p.in_sn = c.in_sn;
    p.in_x0 = input->dim[0].min; p.in_y0 = input->dim[1].min;
    p.in_w = input->dim[0].extent; p.in_h = input->dim[1].extent;
    p.out = (u8 *)args[3].dev;
    p.out_sy = out->dim[1].stride; p.out_sc = out->dim[2].stride;
    p.out_sn = c.out_sn;
    p.out_px = out->dim[0].stride;
    p.out_x0 = ox; p.out_y0 = oy; p.W = W; p.H = H; p.C = out->dim[2].extent; p.out_c0 = out->dim[2].min; p.N = N;
    p.tab = tab;
    // (1/7000 - 1/3200) in float, reciprocal folded in double then rounded (src/Simplify_Div.cpp:204)
    const float c_diff = 1.0f / 7000 - 1.0f / 3200;
    const float inv_c_diff = (float)(1.0 / (double)c_diff);
    // offsets of matrix element (0,0)
    const float *m32p = (const float *)args[1].dev - m3200->dim[0].min * (int64_t)m3200->dim[0].stride - m3200->dim[1].min * (int64_t)m3200->dim[1].stride;
    const float *m70p = (const float *)args[2].dev - m7000->dim[0].min * (int64_t)m7000->dim[0].stride - m7000->dim[1].min * (int64_t)m7000->dim[1].stride;
    cudaStream_t s = hb::stream();
    {
        hb::CallTimer timer(s);
        HB_LAUNCH("cp_tables", cp_tables_kernel, 4, 256, 0, s, tab, m32p, (int64_t)m3200->dim[0].stride, (int64_t)m3200->dim[1].stride,
                  m70p, (int64_t)m7000->dim[0].stride, (int64_t)m7000->dim[1].stride, color_temp, gamma, contrast, sharpen_strength,
                  blackLevel, whiteLevel, inv_c_diff);
        dim3 grid((W + TW - 1) / TW, (H + TH - 1) / TH, std::min(N, hb::kMaxGridZ));
        if (args[3].interleaved) HB_LAUNCH("camera_pipe_il", camera_pipe_kernel<true>, grid, 256, 0, s, p);
        else HB_LAUNCH("camera_pipe", camera_pipe_kernel<false>, grid, 256, 0, s, p);
    }
    return hb::finish(args, 4, what);
}

}  // namespace

extern "C" int camera_pipe(halide_buffer_t *input, halide_buffer_t *m3200, halide_buffer_t *m7000, float color_temp, float gamma,
                           float contrast, float sharpen_strength, int32_t blackLevel, int32_t whiteLevel, halide_buffer_t *out) {
    hb::Arg args[4] = {{input, kArgs[0]}, {m3200, kArgs[1]}, {m7000, kArgs[2]}, {out, kArgs[9]}};
    return run_camera_pipe(args, color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel, "camera_pipe launch");
}
HB_EXPORT_FILTER(camera_pipe, kArgs)
HB_EXPORT_AUTO_SCHEDULE(camera_pipe, kArgs)

// Burst and interleaved entry points (library extensions): camera_pipe on every frame of a raw burst, and on
// pixel-interleaved outputs.  The matrices and scalars are camera_pipe's and shared by all frames.
extern "C" int halide_b200_camera_pipe_batch(halide_buffer_t *input, halide_buffer_t *m3200, halide_buffer_t *m7000, float color_temp,
                                             float gamma, float contrast, float sharpen_strength, int32_t blackLevel,
                                             int32_t whiteLevel, halide_buffer_t *out) {
    hb::Arg args[4] = {{input, kBatchArgs[0]}, {m3200, kArgs[1]}, {m7000, kArgs[2]}, {out, kBatchArgs[1]}};
    return run_camera_pipe(args, color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel, "camera_pipe_batch launch");
}
extern "C" int halide_b200_camera_pipe_interleaved(halide_buffer_t *input, halide_buffer_t *m3200, halide_buffer_t *m7000,
                                                   float color_temp, float gamma, float contrast, float sharpen_strength,
                                                   int32_t blackLevel, int32_t whiteLevel, halide_buffer_t *out) {
    hb::Arg args[4] = {{input, kArgs[0]}, {m3200, kArgs[1]}, {m7000, kArgs[2]}, {out, kArgs[9], nullptr, true}};
    return run_camera_pipe(args, color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel,
                           "camera_pipe_interleaved launch");
}
extern "C" int halide_b200_camera_pipe_interleaved_batch(halide_buffer_t *input, halide_buffer_t *m3200, halide_buffer_t *m7000,
                                                         float color_temp, float gamma, float contrast, float sharpen_strength,
                                                         int32_t blackLevel, int32_t whiteLevel, halide_buffer_t *out) {
    hb::Arg args[4] = {{input, kBatchArgs[0]}, {m3200, kArgs[1]}, {m7000, kArgs[2]}, {out, kBatchArgs[1], nullptr, true}};
    return run_camera_pipe(args, color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel,
                           "camera_pipe_interleaved_batch launch");
}
