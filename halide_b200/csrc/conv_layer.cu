// conv_layer.cu — conv_layer(input, filter, bias, relu) for sm_90a.
//
// Reference algorithm: apps/conv_layer/conv_layer_generator.cpp:17-27 with the fixed shapes the generator pins
// by constraints (:35-50): input (CI=128, W+2=102, H+2=82, N=5) channel-innermost, filter (CO=128, 3, 3, CI)
// output-channel-innermost, bias (128), relu (CO=128, W=100, H=80, N=5).
//   relu(co,x,y,n) = max(0, bias(co) + sum_{ky,kx,ci} filter(co,kx,ky,ci) * input(ci, x+kx, y+ky, n))
// Float pipeline: parity bar 1e-4 relative against oracle/oracle_conv_layer.cpp (a tiled contraction necessarily
// changes the summation order; the harness data are all positive so there is no cancellation).
//
// Two contractions: the tensor-core implicit GEMM of conv_layer_tc.cu (the default) and this FP32 SIMT kernel
// (register-tiled implicit GEMM, FFMA): M = 40 000 output pixels, N = 128, K = 1152, 11.8 GFLOP.  TF32 tensor
// cores need a 3-term split to hold 1e-4 on rand()-scale inputs because the conversion truncates.
// Block = 10x8 output pixels x 128 output channels, 256 threads, each thread 5 pixels x 8 channels in registers;
// per (ci-chunk of 32, ky, kx) one 16 KB filter slab is staged in shared memory; the input patch (12x10 pixels
// x 32 channels) is staged once per ci-chunk.  Operand loads are warp-broadcast or 16-byte conflict-free.
#include <stdlib.h>
#include <string.h>

#include "hb_common.h"

// wgmma / TMA implementation (conv_layer_tc.cu)
int conv_layer_tc_run(const float *din, const float *df, const float *db, float *dout, cudaStream_t s);

namespace {

// Which contraction runs: the wgmma implicit GEMM (3xTF32 split) or the FP32 SIMT kernel.  HALIDE_B200_CONV=simt|tc
// picks at start-up; halide_b200_conv_use_tensor_cores() switches at run time (tests cover both).
bool g_use_tc = [] {
    const char *e = getenv("HALIDE_B200_CONV");
    return !(e && strcmp(e, "simt") == 0);  // default: tensor cores
}();

constexpr int N = 5, CI = 128, CO = 128, W = 100, H = 80;  // generator :35-50 (process.cpp:14)
constexpr int TX = 10, TY = 8;                             // output tile
constexpr int PX = TX + 2, PY = TY + 2;                    // input patch
constexpr int KC = 32;                                     // ci per chunk
constexpr int KP = KC + 4;                                 // padded channel pitch of the input patch (bank spread)

__global__ void __launch_bounds__(256) conv_layer_kernel(const float *__restrict__ in, const float *__restrict__ filt,
                                                         const float *__restrict__ bias, float *__restrict__ out) {
    __shared__ __align__(16) float s_in[PY][PX][KP];   // 17 280 B
    __shared__ __align__(16) float s_f[KC][CO];        // 16 384 B
    const int tid = threadIdx.x;
    const int tc = tid & 15, tp = tid >> 4;            // 16 channel groups x 16 pixel groups
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY, n = blockIdx.z;
    const int prow = tp >> 1, pcol = (tp & 1) * 5;     // this thread's 5 pixels: row prow, cols pcol..pcol+4
    // 8 output channels per thread as two quads, co = 4*tc + {0..3} and 64 + 4*tc + {0..3}: the 16 threads of a
    // channel group then read 256 contiguous bytes of the filter slab per quad (conflict-free LDS.128)
    const int co0 = tc * 4, co1 = 64 + tc * 4;
    float acc[5][8];
#pragma unroll
    for (int j = 0; j < 5; j++)
#pragma unroll
        for (int k = 0; k < 8; k++) acc[j][k] = bias[(k < 4 ? co0 : co1 - 4) + k];

    const int64_t in_sx = CI, in_sy = (int64_t)CI * (W + 2), in_sn = in_sy * (H + 2);
    const float *in_n = in + n * in_sn;
    for (int c0 = 0; c0 < CI; c0 += KC) {
        __syncthreads();  // previous chunk's consumers are done with s_in / s_f
        // input patch: PY*PX pixels x KC channels, 8 float4 per pixel
        for (int i = tid; i < PY * PX * (KC / 4); i += 256) {
            int pix = i / (KC / 4), q = i - pix * (KC / 4);
            int py = pix / PX, px = pix - py * PX;
            int gy = min(y0 + py, H + 1), gx = min(x0 + px, W + 1);  // tiles never overhang (100 % 10 == 0, 80 % 8 == 0)
            float4 v = __ldg(reinterpret_cast<const float4 *>(in_n + gy * in_sy + gx * in_sx + c0) + q);
            *reinterpret_cast<float4 *>(&s_in[py][px][4 * q]) = v;
        }
        for (int kk = 0; kk < 9; kk++) {
            const int ky = kk / 3, kx = kk - ky * 3;
            __syncthreads();  // s_f free (and, first time round, s_in visible)
            // filter slab: KC rows of CO floats at filter(0, kx, ky, c0 + r)
            for (int i = tid; i < KC * (CO / 4); i += 256) {
                int r = i / (CO / 4), q = i - r * (CO / 4);
                float4 v = __ldg(reinterpret_cast<const float4 *>(filt + (int64_t)(c0 + r) * (CO * 9) + ky * (CO * 3) + kx * CO) + q);
                *reinterpret_cast<float4 *>(&s_f[r][4 * q]) = v;
            }
            __syncthreads();
            const float *a_base = &s_in[prow + ky][pcol + kx][0];
#pragma unroll 4
            for (int ci = 0; ci < KC; ci++) {
                float a[5];
#pragma unroll
                for (int j = 0; j < 5; j++) a[j] = a_base[j * KP + ci];
                float4 b0 = *reinterpret_cast<const float4 *>(&s_f[ci][co0]);
                float4 b1 = *reinterpret_cast<const float4 *>(&s_f[ci][co1]);
                const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int j = 0; j < 5; j++)
#pragma unroll
                    for (int k = 0; k < 8; k++) acc[j][k] = __fmaf_rn(b[k], a[j], acc[j][k]);
            }
        }
    }
    // relu + store: two quads of output channels per pixel
    const int64_t o_sx = CO, o_sy = (int64_t)CO * W, o_sn = o_sy * H;
#pragma unroll
    for (int j = 0; j < 5; j++) {
        float *o = out + n * o_sn + (int64_t)(y0 + prow) * o_sy + (int64_t)(x0 + pcol + j) * o_sx;
        float4 v0 = make_float4(fmaxf(acc[j][0], 0.f), fmaxf(acc[j][1], 0.f), fmaxf(acc[j][2], 0.f), fmaxf(acc[j][3], 0.f));
        float4 v1 = make_float4(fmaxf(acc[j][4], 0.f), fmaxf(acc[j][5], 0.f), fmaxf(acc[j][6], 0.f), fmaxf(acc[j][7], 0.f));
        *reinterpret_cast<float4 *>(o + co0) = v0;
        *reinterpret_cast<float4 *>(o + co1) = v1;
    }
}

// estimates = the fixed shapes (generator :52-68)
int64_t e_zero = 0, e_ci = CI, e_co = CO, e_wp = W + 2, e_hp = H + 2, e_w = W, e_h = H, e_n = N, e_3 = 3;
const int64_t *const est_in[8] = {&e_zero, &e_ci, &e_zero, &e_wp, &e_zero, &e_hp, &e_zero, &e_n};
const int64_t *const est_f[8] = {&e_zero, &e_co, &e_zero, &e_3, &e_zero, &e_3, &e_zero, &e_ci};
const int64_t *const est_b[2] = {&e_zero, &e_co};
const int64_t *const est_out[8] = {&e_zero, &e_co, &e_zero, &e_w, &e_zero, &e_h, &e_zero, &e_n};
const halide_filter_argument_t kArgs[4] = {
    {"input", halide_argument_kind_input_buffer, 4, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_in},
    {"filter", halide_argument_kind_input_buffer, 4, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_f},
    {"bias", halide_argument_kind_input_buffer, 1, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_b},
    {"relu", halide_argument_kind_output_buffer, 4, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, nullptr, est_out},
};
// the generator's set_bounds / set_stride constraints (:35-50): every buffer is exactly this region, densely packed
const hb::Region kShapes[4] = {{{0}, {CI, W + 2, H + 2, N}, false}, {{0}, {CO, 3, 3, CI}, false}, {{0}, {CO}, false},
                               {{0}, {CO, W, H, N}, false}};

int check_fixed(const hb::Arg &a, const hb::Region &shape) {
    const halide_buffer_t *b = a.b;
    const int *ext = shape.extent;
    int64_t stride = 1;
    for (int d = 0; d < b->dimensions; d++) {
        if (b->dim[d].min != 0 || b->dim[d].extent != ext[d] || b->dim[d].stride != stride) {
            return hb::fail(halide_error_code_constraint_violated,
                            "Constraint violated: %s.dim(%d) is (min %d, extent %d, stride %d) but must be (0, %d, %lld)", a.meta.name, d,
                            b->dim[d].min, b->dim[d].extent, b->dim[d].stride, ext[d], (long long)stride);
        }
        stride *= ext[d];
    }
    return 0;
}

}  // namespace

extern "C" int conv_layer(halide_buffer_t *input, halide_buffer_t *filter, halide_buffer_t *bias, halide_buffer_t *relu) {
    int r;
    hb::Arg args[4] = {{input, kArgs[0]}, {filter, kArgs[1]}, {bias, kArgs[2]}, {relu, kArgs[3]}};
    if ((r = hb::check_args(args, 4))) return r;
    if (hb::answer_bounds_query(args, kShapes, 4)) return 0;
    if ((r = hb::check_shapes(args, 4))) return r;
    if ((r = check_fixed(args[3], kShapes[3])) || (r = check_fixed(args[0], kShapes[0])) || (r = check_fixed(args[1], kShapes[1])) ||
        (r = check_fixed(args[2], kShapes[2])))
        return r;
    if ((r = hb::acquire(args, 4))) return r;
    const float *din = (const float *)args[0].dev, *df = (const float *)args[1].dev, *db = (const float *)args[2].dev;
    float *dout = (float *)args[3].dev;
    cudaStream_t s = hb::stream();
    {
        hb::CallTimer timer(s);
        if (g_use_tc) {
            if ((r = conv_layer_tc_run(din, df, db, dout, s))) return r;
        } else {
            dim3 grid(W / TX, H / TY, N);
            HB_LAUNCH("conv_layer_f32", conv_layer_kernel, grid, 256, 0, s, din, df, db, dout);
        }
    }
    return hb::finish(args, 4, "conv_layer launch");
}
HB_EXPORT_FILTER(conv_layer, kArgs)
HB_EXPORT_AUTO_SCHEDULE(conv_layer, kArgs)

extern "C" void halide_b200_conv_use_tensor_cores(int enable) {
    g_use_tc = enable != 0;
}
