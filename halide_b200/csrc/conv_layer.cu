// conv_layer.cu — conv_layer(input, filter, bias, relu) for sm_90a.
//
// Reference algorithm: apps/conv_layer/conv_layer_generator.cpp:17-27 with the fixed shapes the generator pins
// by constraints (:35-50): input (CI=128, W+2=102, H+2=82, N=5) channel-innermost, filter (CO=128, 3, 3, CI)
// output-channel-innermost, bias (128), relu (CO=128, W=100, H=80, N=5).
//   relu(co,x,y,n) = max(0, bias(co) + sum_{ky,kx,ci} filter(co,kx,ky,ci) * input(ci, x+kx, y+ky, n))
// Float pipeline: parity bar 1e-4 relative against oracle/oracle_conv_layer.cpp (a tiled contraction necessarily
// changes the summation order; the harness data are all positive so there is no cancellation).
//
// The contraction is the tensor-core implicit GEMM of conv_layer_tc.cu (wgmma + TMA, 3xTF32 split): M = 40 000
// output pixels, N = 128, K = 1152, 11.8 GFLOP.  This file holds the Halide call boundary and the fixed-shape checks,
// and halide_b200_conv_layer_any_shape: the same algorithm with the five constants read from the buffers.
#include "conv_layer_tc.h"  // the wgmma / TMA implementation
#include "hb_common.h"

namespace {

constexpr int N = 5, CI = 128, CO = 128, W = 100, H = 80;  // generator :35-50 (process.cpp:14)

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
        if ((r = conv_layer_tc_run(din, df, db, dout, s))) return r;
    }
    return hb::finish(args, 4, "conv_layer launch");
}
HB_EXPORT_FILTER(conv_layer, kArgs)
HB_EXPORT_AUTO_SCHEDULE(conv_layer, kArgs)

// conv_layer with the generator's set_bounds / set_stride constraints removed: CO, W, H, N and the mins (c0, x0, y0, n0)
// are relu's, CI is filter's last extent (input's first when filter is the buffer of a bounds query).  Nothing is
// edge-clamped, so input must cover [0,CI) x [x0, x0+W+2) x [y0, y0+H+2) x [n0, n0+N), filter [c0, c0+CO) x 3 x 3 x [0,CI)
// and bias [c0, c0+CO); buffers may be larger and every stride but the innermost (1) is free.
extern "C" int halide_b200_conv_layer_any_shape(halide_buffer_t *input, halide_buffer_t *filter, halide_buffer_t *bias,
                                                halide_buffer_t *relu) {
    int r;
    hb::Arg args[4] = {{input, kArgs[0]}, {filter, kArgs[1]}, {bias, kArgs[2]}, {relu, kArgs[3]}};
    if ((r = hb::check_args(args, 4))) return r;
    const halide_dimension_t *o = relu->dim;
    const bool filter_queried = filter->host == nullptr && filter->device == 0;
    const int co = o[0].extent, w = o[1].extent, h = o[2].extent, n = o[3].extent;
    const int ci = filter_queried ? input->dim[0].extent : filter->dim[3].extent;
    const hb::Region need[4] = {{{0, o[1].min, o[2].min, o[3].min}, {ci, w + 2, h + 2, n}, true},
                                {{o[0].min, 0, 0, 0}, {co, 3, 3, ci}, true},
                                {{o[0].min}, {co}, true},
                                hb::region_of(relu, false)};
    if (hb::answer_bounds_query(args, need, 4)) return 0;
    if ((r = hb::check_shapes(args, 4))) return r;
    if (co <= 0 || w <= 0 || h <= 0 || n <= 0) return 0;
    if ((r = hb::check_required(args, need, 4))) return r;
    if ((r = hb::acquire(args, 4))) return r;
    const halide_dimension_t *in = input->dim, *f = filter->dim;
    ConvProblem p;
    p.N = n, p.CI = ci, p.CO = co, p.W = w, p.H = h;
    p.in_sx = in[1].stride, p.in_sy = in[2].stride, p.in_sn = in[3].stride;
    p.in = (const float *)args[0].dev + (0 - in[0].min) + (o[1].min - in[1].min) * p.in_sx + (o[2].min - in[2].min) * p.in_sy +
           (o[3].min - in[3].min) * p.in_sn;
    p.f_skx = f[1].stride, p.f_sky = f[2].stride, p.f_sci = f[3].stride;
    p.filt = (const float *)args[1].dev + (o[0].min - f[0].min) + (0 - f[1].min) * p.f_skx + (0 - f[2].min) * p.f_sky + (0 - f[3].min) * p.f_sci;
    p.bias = (const float *)args[2].dev + (o[0].min - bias->dim[0].min);
    p.out = (float *)args[3].dev;
    p.out_sx = o[1].stride, p.out_sy = o[2].stride, p.out_sn = o[3].stride;
    cudaStream_t s = hb::stream();
    {
        hb::CallTimer timer(s);
        if ((r = conv_layer_tc_run_any_shape(p, s))) return r;
    }
    return hb::finish(args, 4, "conv_layer_any_shape launch");
}
