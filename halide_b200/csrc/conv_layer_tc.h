// conv_layer_tc.h — the wgmma / TMA contraction of conv_layer_tc.cu as conv_layer.cu calls it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// The generator's fixed shape (N5 CI128 CO128 100x80), dense buffers in the generator's layouts.
// Returns 0 on success, a negative halide error code otherwise.
int conv_layer_tc_run(const float *din, const float *df, const float *db, float *dout, cudaStream_t s);

// Any shape.  Every pointer addresses the first element the call touches (the buffers' mins are already applied), all
// buffers are channel-innermost with stride 1 there, and the other strides are in elements:
//   in    (ci 0, x0, y0, n0) of input,  read over [0,CI) x [0,W+2) x [0,H+2) x [0,N)
//   filt  (c0, 0, 0, 0) of filter,      read over [0,CO) x 3 x 3 x [0,CI)
//   bias  c0 of bias;  out (c0, x0, y0, n0) of relu, written over [0,CO) x [0,W) x [0,H) x [0,N)
struct ConvProblem {
    int N, CI, CO, W, H;
    const float *in;
    int64_t in_sx, in_sy, in_sn;
    const float *filt;
    int64_t f_skx, f_sky, f_sci;
    const float *bias;
    float *out;
    int64_t out_sx, out_sy, out_sn;
};
int conv_layer_tc_run_any_shape(const ConvProblem &p, cudaStream_t s);
