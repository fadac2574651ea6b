// stencil_chain.cu — stencil_chain(input, output): 32 successive 5x5 uint16 stencils;
// halide_b200_stencil_chain_stencils(input, stencils, output): the same chain with 1..100 stages.
//
// Reference algorithm: apps/stencil_chain/stencil_chain_generator.cpp:16-34.  Stage s+1 at (x,y) is
//   e = u16(0); for i in -2..2 (x offset) for j in -2..2 (y offset): e += u16((i+3)*(j+3)) * stage_s(x+i, y+j)
// entirely in uint16, i.e. arithmetic in the ring Z/2^16.  Only the input is edge-clamped
// (repeat_edge, generator :18); later stages are pure functions evaluated on grown regions.
//
// Because Z/2^16 is a commutative ring the result does not depend on summation order, so the
// weights' outer-product structure (i+3)*(j+3) is exploited exactly: a vertical 5-tap pass with
// weights (j+3) followed by a horizontal 5-tap pass with weights (i+3), both reduced mod 2^16
// (10 multiply-adds per pixel per stage instead of 25).  Bit-exact by construction; the parity
// tests compare with the oracle's literal 25-tap source-order loop.
//
// Kernel shape: ALU/shared-memory bound (800 MAC/px in the reference formulation, 4 B/px of
// compulsory HBM traffic).  kFuse stages run per launch on a shared-memory tile with a 2*kFuse
// apron (a chain whose length is not a multiple of kFuse ends with one shorter launch); the frame
// itself (7.9 MB at the harness size) stays L2-resident between launches.
//
// halide_b200_stencil_chain_batch / _stencils_batch run the same launches on a clip: each launch takes a group of frames,
// frame blockIdx.z each (FR instances).
#include <algorithm>
#include <type_traits>

#include "hb_common.h"

namespace {

constexpr int kStages = 32;     // GeneratorParam `stencils` of the shipped app (generator :9): stencil_chain's depth
constexpr int kMaxStages = 100; // the range the generator declares for it is [1, 100]
constexpr int kFuse = 4;        // stages per launch (the last launch of a chain may run fewer)
constexpr int kTile = 64;       // output tile edge per block
constexpr int kTileIn = kTile + 4 * kFuse;  // 80: input tile edge (2 px apron per fused stage, both sides)

struct Plane {
    const uint16_t *src;  // element (x0,y0) of the region this launch reads
    uint16_t *dst;        // element (x0+2f, y0+2f) of the region it writes
    int64_t src_sy, dst_sy;
    int src_w, src_h;     // extent of the source region
    // when reading the pipeline input: clamp coordinates into the buffer (repeat_edge)
    int clamp_x0, clamp_y0, clamp_w, clamp_h, do_clamp;
    int dst_w, dst_h;
    int src_words, dst_words;  // rows of src / dst keep pixel pairs 4-byte aligned (even stride, aligned base): 32-bit accesses
};
// The parameters of the FR instances, which run one launch's stages on a group of frames, frame blockIdx.z each: Plane
// with src and dst at the group's first frame, and the strides from one frame to the next.  src_words / dst_words hold
// for every frame of the group (an odd frame stride clears them).  (A separate type, so that the one-frame kernels keep
// their parameter block byte for byte.)
struct PlaneBatch : Plane {
    int64_t src_sn, dst_sn;  // frame strides in elements (the pipeline input's may be negative or zero)
};
template<bool FR>
using PlaneOf = std::conditional_t<FR, PlaneBatch, Plane>;

// The source and destination of the block's frame: blockIdx.z's in an FR instance, the parameter block's own otherwise.
// The parameter block is never written.
template<bool FR>
__device__ __forceinline__ const uint16_t *frame_src(const PlaneOf<FR> &p) {
    if constexpr (FR) return p.src + (int64_t)blockIdx.z * p.src_sn;
    else return p.src;
}
template<bool FR>
__device__ __forceinline__ uint16_t *frame_dst(const PlaneOf<FR> &p) {
    if constexpr (FR) return p.dst + (int64_t)blockIdx.z * p.dst_sn;
    else return p.dst;
}

// ---- register-window kernel (kFuse stages per launch) -------------------------------------------------------------
// The tile lives in shared memory as 32-bit words (two pixels), every edge length is a compile-time constant, and each
// pass is a sliding window held in registers:
//   vertical:   a thread owns a column PAIR on a segment of rows — per row one 32-bit load, eight multiply-adds (four
//               per pixel: v0 + 2 v1 + 3 v2 + 4 v3 + 5 v4 starts from v0), one PRMT to repack, one 32-bit store;
//   horizontal: a thread owns a row on a segment of output pairs — per output pair one new word, eight multiply-adds.
// Sums are taken in 32 bits and truncated by the repack (Z/2^16 arithmetic: any order, any carries above bit 15).
// Row pitch = 41 words (odd): the 32 lanes of a warp — consecutive column pairs in the vertical pass, consecutive rows
// in the horizontal one — fall into 32 different banks.
constexpr int kPW = (kTileIn + 2) / 2;  // words per shared-memory row

template<int EDGE>
__device__ __forceinline__ void stencil_stage(const uint32_t *cur, uint32_t *mid, uint32_t *nxt, int tid) {
    constexpr int VH = EDGE - 4, NP = EDGE / 2;
    {   // vertical pass: mid[y][x] = sum_j (j+1) * cur[y+j][x], y in [0, VH), all EDGE columns
        constexpr int SEG = 256 / NP, LEN = (VH + SEG - 1) / SEG;
        const int sgi = tid / NP, pc = tid - sgi * NP;
        const int r0 = sgi * LEN, r1 = min(r0 + LEN, VH);
        if (sgi < SEG && r0 < r1) {
            const uint32_t *c = cur + r0 * kPW + pc;
            uint32_t w = c[0];
            uint32_t l0 = w & 0xffffu, h0 = w >> 16;
            w = c[kPW];
            uint32_t l1 = w & 0xffffu, h1 = w >> 16;
            w = c[2 * kPW];
            uint32_t l2 = w & 0xffffu, h2 = w >> 16;
            w = c[3 * kPW];
            uint32_t l3 = w & 0xffffu, h3 = w >> 16;
            uint32_t *o = mid + r0 * kPW + pc;
#pragma unroll 4
            for (int r = r0; r < r1; r++) {
                w = c[4 * kPW];
                const uint32_t l4 = w & 0xffffu, h4 = w >> 16;
                const uint32_t al = l0 + 2u * l1 + 3u * l2 + 4u * l3 + 5u * l4;
                const uint32_t ah = h0 + 2u * h1 + 3u * h2 + 4u * h3 + 5u * h4;
                *o = __byte_perm(al, ah, 0x5410);
                l0 = l1; l1 = l2; l2 = l3; l3 = l4;
                h0 = h1; h1 = h2; h2 = h3; h3 = h4;
                c += kPW;
                o += kPW;
            }
        }
    }
    __syncthreads();
    {   // horizontal pass: nxt[y][x] = sum_i (i+1) * mid[y][x+i], x in [0, VH), VH rows
        constexpr int SEG = 256 / VH, NOP = VH / 2, LEN = (NOP + SEG - 1) / SEG;
        const int sgi = tid / VH, r = tid - sgi * VH;
        const int k0 = sgi * LEN, k1 = min(k0 + LEN, NOP);
        if (sgi < SEG && k0 < k1) {
            const uint32_t *c = mid + r * kPW + k0;
            uint32_t w = c[0];
            uint32_t v0 = w & 0xffffu, v1 = w >> 16;
            w = c[1];
            uint32_t v2 = w & 0xffffu, v3 = w >> 16;
            uint32_t *o = nxt + r * kPW + k0;
#pragma unroll 4
            for (int k = k0; k < k1; k++) {
                w = c[2];
                const uint32_t v4 = w & 0xffffu, v5 = w >> 16;
                const uint32_t a0 = v0 + 2u * v1 + 3u * v2 + 4u * v3 + 5u * v4;
                const uint32_t a1 = v1 + 2u * v2 + 3u * v3 + 4u * v4 + 5u * v5;
                *o = __byte_perm(a0, a1, 0x5410);
                v0 = v2; v1 = v3; v2 = v4; v3 = v5;
                c++;
                o++;
            }
        }
    }
    __syncthreads();
}

template<int EDGE, int LEFT>
struct StencilStages {
    static __device__ __forceinline__ const uint32_t *run(uint32_t *cur, uint32_t *mid, uint32_t *nxt, int tid) {
        stencil_stage<EDGE>(cur, mid, nxt, tid);
        return StencilStages<EDGE - 4, LEFT - 1>::run(nxt, mid, cur, tid);
    }
};
template<int EDGE>
struct StencilStages<EDGE, 0> {
    static __device__ __forceinline__ const uint32_t *run(uint32_t *cur, uint32_t *, uint32_t *, int) { return cur; }
};

template<int FUSE, bool FR = false>
__global__ void __launch_bounds__(256) stencil_chain_window_kernel(PlaneOf<FR> p) {
    static_assert(FUSE >= 1 && FUSE <= kFuse, "the shared-memory tiles hold an input tile of kFuse stages at most");
    constexpr int IN = kTile + 4 * FUSE, INW = IN / 2;
    __shared__ uint32_t A[kTileIn * kPW];
    __shared__ uint32_t B[kTileIn * kPW];
    __shared__ uint32_t C[kTileIn * kPW];
    const int tid = threadIdx.x;
    const int ox = blockIdx.x * kTile, oy = blockIdx.y * kTile;  // tile origin in dst coordinates (even)
    // source tile: dst (ox, oy) needs src (ox .. ox + IN - 1, oy .. oy + IN - 1); elements outside the source region are
    // only ever combined into outputs outside the destination region, so they may hold anything (zeros here)
    for (int t = tid; t < IN * INW; t += 256) {
        const int ly = t / INW, lw = t - ly * INW;
        const int sx = ox + 2 * lw, sy = oy + ly;
        uint32_t w = 0;
        if (p.do_clamp) {
            const int cy = min(max(sy + p.clamp_y0, 0), p.clamp_h - 1);
            const int cx0 = min(max(sx + p.clamp_x0, 0), p.clamp_w - 1), cx1 = min(max(sx + 1 + p.clamp_x0, 0), p.clamp_w - 1);
            const uint16_t *row = frame_src<FR>(p) + (int64_t)cy * p.src_sy;
            w = (uint32_t)row[cx0] | ((uint32_t)row[cx1] << 16);
        } else if (sy < p.src_h) {
            const uint16_t *e = frame_src<FR>(p) + (int64_t)sy * p.src_sy + sx;
            if (p.src_words && sx + 1 < p.src_w) {
                w = *reinterpret_cast<const uint32_t *>(e);
            } else {
                if (sx < p.src_w) w = e[0];
                if (sx + 1 < p.src_w) w |= (uint32_t)e[1] << 16;
            }
        }
        A[ly * kPW + lw] = w;
    }
    __syncthreads();
    const uint32_t *res = StencilStages<IN, FUSE>::run(A, C, B, tid);
    // res holds the kTile x kTile result (kTile / 2 words per row)
    for (int t = tid; t < kTile * (kTile / 2); t += 256) {
        const int ly = t / (kTile / 2), lw = t - ly * (kTile / 2);
        const int dx = ox + 2 * lw, dy = oy + ly;
        if (dy >= p.dst_h || dx >= p.dst_w) continue;
        const uint32_t w = res[ly * kPW + lw];
        uint16_t *e = frame_dst<FR>(p) + (int64_t)dy * p.dst_sy + dx;
        if (p.dst_words && dx + 1 < p.dst_w) {
            *reinterpret_cast<uint32_t *>(e) = w;
        } else {
            e[0] = (uint16_t)w;
            if (dx + 1 < p.dst_w) e[1] = (uint16_t)(w >> 16);
        }
    }
}

int64_t est_i[2][2] = {{0, 1536}, {0, 2560}};
const int64_t *const est_ptrs[4] = {&est_i[0][0], &est_i[0][1], &est_i[1][0], &est_i[1][1]};
const halide_filter_argument_t kArgs[2] = {
    {"input", halide_argument_kind_input_buffer, 2, {halide_type_uint, 16, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
    {"output", halide_argument_kind_output_buffer, 2, {halide_type_uint, 16, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
};
// The batch entry points: the same buffers with a third dimension, the frame index n.
const halide_filter_argument_t kBatchArgs[2] = {hb::variant(kArgs[0], 1), hb::variant(kArgs[1], 1)};

// Scratch a clip's call may hold: its frames run in groups whose intermediate planes together fit in kScratchBudget
// bytes (at least one frame a group, however large its planes), and the groups reuse one allocation per plane.  The
// device pool keeps freed blocks until they are released, so scratch sized to a whole clip would stay allocated after
// the call.  At S = 32, 256 MiB holds the two planes of 1 frame of 7680 x 4320 (138 MB), 7 of 3840 x 2160 (36 MB
// each), 27 of 1920 x 1080 and 150 of 640 x 480; chains of 4 stages or fewer need no scratch, so their groups hold up
// to kMaxGridZ frames.  A group of one frame runs through the one-frame kernels.  No minimum group size is set: groups
// of 2 or 3 frames were not measured against single calls (H100 80GB HBM3 at 700 W: 4 x 7680 x 4320 at S = 4, one
// group of 4, took 0.991 of four one-frame calls; at S = 32 and 100, one frame a group, 1.000).
constexpr size_t kScratchBudget = size_t(256) << 20;

// One launch of `fuse` stages (1..kFuse) on `frames` frames (FR) or on one frame.  Every depth is the same kernel and
// carries the same name.
template<bool FR>
void launch_window(int fuse, const PlaneOf<FR> &p, int frames, cudaStream_t s) {
    const dim3 grid((p.dst_w + kTile - 1) / kTile, (p.dst_h + kTile - 1) / kTile, frames);
    switch (fuse) {
    case 1: HB_LAUNCH("stencil_chain_window", (stencil_chain_window_kernel<1, FR>), grid, 256, 0, s, p); break;
    case 2: HB_LAUNCH("stencil_chain_window", (stencil_chain_window_kernel<2, FR>), grid, 256, 0, s, p); break;
    case 3: HB_LAUNCH("stencil_chain_window", (stencil_chain_window_kernel<3, FR>), grid, 256, 0, s, p); break;
    default: HB_LAUNCH("stencil_chain_window", (stencil_chain_window_kernel<kFuse, FR>), grid, 256, 0, s, p); break;
    }
}

// Every stencil_chain entry point: the chain of S = `stencils` stages.  Launch plan: floor(S / kFuse) launches of kFuse
// stages, then, when S mod kFuse is not 0, one launch of the remaining stages.  Launch k reads the region grown by
// Rin = 2 * (stages not yet run) and writes it grown by Rout = Rin - 2 * (its stages); the last launch writes the output
// itself.  Putting the short launch last keeps every intermediate apron, and with it the scratch (largest at launch 0:
// 2 * (S - kFuse)), as small as the order allows.  S = 32 is stencil_chain: 8 launches of 4 stages.
// 2-D (x, y) records take one frame; 3-D (x, y, n) ones a clip, output frame n reading input frame n (repeat_edge in x
// and y within the frame, never across frames), whose frames run the launch plan in groups of up to G (see
// kScratchBudget).
int run_stencil_chain(halide_buffer_t *input, int32_t stencils, halide_buffer_t *output,
                      const halide_filter_argument_t *rec, const char *what) {
    int r;
    hb::Arg args[2] = {{input, rec[0]}, {output, rec[1]}};
    if ((r = hb::check_args(args, 2))) return r;
    const hb::Clip c = hb::clip_of(args[0], args[1], 2);
    // every access to the input goes through repeat_edge in x and y: nothing beyond a non-empty frame is required there;
    // a clip's output frame n reads input frame n, not clamped: the input's frames must cover the output's (dimension 2).
    // A query is answered with the output region.
    const int N = c.N;
    const hb::Region need[2] = {hb::region_of(output, false), hb::region_of(output, false)};
    const hb::Region frames = c.with_frames({{}, {}, true});  // (extents of 0: x and y are not checked)
    if (hb::answer_bounds_query(args, need, 2)) return 0;
    if ((r = hb::check_shapes(args, 2)) || (r = hb::check_required(args, &frames, 1))) return r;
    const int W = output->dim[0].extent, H = output->dim[1].extent;
    if (W <= 0 || H <= 0 || N <= 0) return 0;
    if (input->dim[0].extent <= 0 || input->dim[1].extent <= 0) {
        return hb::fail(halide_error_code_access_out_of_bounds, "Input buffer input is empty");
    }
    if (stencils < 1 || stencils > kMaxStages) {
        return hb::fail(stencils < 1 ? halide_error_code_param_too_small : halide_error_code_param_too_large,
                        "Parameter stencils is %d but must be in [1, %d]", (int)stencils, kMaxStages);
    }
    if ((r = hb::acquire(args, 2))) return r;

    const int S = stencils;
    const int full = S / kFuse, rest = S % kFuse;
    const int groups = full + (rest ? 1 : 0);

    // ping-pong buffers for the intermediate stages on their grown regions, G frames side by side in each
    const int maxR = groups > 1 ? 2 * (S - kFuse) : 0;
    const int64_t bw = (W + 2 * maxR + 1) & ~(int64_t)1, bh = H + 2 * maxR;  // (even pitch: intermediate rows keep pixel pairs word-aligned)
    const int planes = groups > 2 ? 2 : groups > 1 ? 1 : 0;
    const size_t frame_bytes = (size_t)planes * bw * bh * sizeof(uint16_t);
    const size_t fit = frame_bytes ? std::max<size_t>(1, kScratchBudget / frame_bytes) : (size_t)hb::kMaxGridZ;
    const int G = (int)std::min<size_t>({(size_t)N, (size_t)hb::kMaxGridZ, fit});
    hb::Scratch scratch;
    uint16_t *buf[2] = {nullptr, nullptr};
    if (groups > 1) {
        buf[0] = scratch.get<uint16_t>((size_t)bw * bh * G);
        buf[1] = groups > 2 ? scratch.get<uint16_t>((size_t)bw * bh * G) : buf[0];
        if (!buf[0] || !buf[1]) return hb::fail(halide_error_code_device_malloc_failed, "stencil_chain: scratch allocation failed");
    }
    const uint16_t *in0 = (const uint16_t *)args[0].dev + c.in_off;  // the input frame output frame 0 reads
    uint16_t *out0 = (uint16_t *)args[1].dev;
    cudaStream_t s = hb::stream();
    {
        hb::CallTimer timer(s);
        for (int n0 = 0; n0 < N; n0 += G) {  // frames [n0, n0 + gn): scratch frames 0 .. gn - 1
            const int gn = std::min(G, N - n0);
            for (int g = 0; g < groups; g++) {
                const int F = g < full ? kFuse : rest;          // stages this launch runs
                const int Rin = 2 * (S - g * kFuse);            // apron of the region this launch reads
                const int Rout = Rin - 2 * F;                   // apron of the region it writes
                PlaneBatch p;
                p.dst_w = W + 2 * Rout;
                p.dst_h = H + 2 * Rout;
                p.src_w = W + 2 * Rin;
                p.src_h = H + 2 * Rin;
                if (g == 0) {
                    p.src = in0 + (int64_t)n0 * c.in_sn;
                    p.src_sy = input->dim[1].stride;
                    p.src_sn = c.in_sn;
                    p.do_clamp = 1;
                    // source-region local (0,0) is absolute (ox - Rin, oy - Rin); buffer-relative = minus input min
                    p.clamp_x0 = output->dim[0].min - Rin - input->dim[0].min;
                    p.clamp_y0 = output->dim[1].min - Rin - input->dim[1].min;
                    p.clamp_w = input->dim[0].extent;
                    p.clamp_h = input->dim[1].extent;
                } else {
                    p.src = buf[(g - 1) & 1];
                    p.src_sy = bw;
                    p.src_sn = bw * bh;
                    p.do_clamp = 0;
                    p.clamp_x0 = p.clamp_y0 = p.clamp_w = p.clamp_h = 0;
                }
                if (g == groups - 1) {
                    p.dst = out0 + (int64_t)n0 * c.out_sn;
                    p.dst_sy = output->dim[1].stride;
                    p.dst_sn = c.out_sn;
                } else {
                    p.dst = buf[g & 1];
                    p.dst_sy = bw;
                    p.dst_sn = bw * bh;
                }
                // 32-bit accesses only where every frame of the group keeps pixel pairs 4-byte aligned
                const int64_t src_sn = gn > 1 ? p.src_sn : 0, dst_sn = gn > 1 ? p.dst_sn : 0;
                p.src_words = ((reinterpret_cast<uintptr_t>(p.src) & 3) == 0 && ((p.src_sy | src_sn) & 1) == 0) ? 1 : 0;
                p.dst_words = ((reinterpret_cast<uintptr_t>(p.dst) & 3) == 0 && ((p.dst_sy | dst_sn) & 1) == 0) ? 1 : 0;
                if (G > 1) launch_window<true>(F, p, gn, s);
                else launch_window<false>(F, p, 1, s);
            }
        }
    }
    return hb::finish(args, 2, what);
}
}  // namespace

extern "C" int stencil_chain(halide_buffer_t *input, halide_buffer_t *output) {
    return run_stencil_chain(input, kStages, output, kArgs, "stencil_chain launch");
}

// stencil_chain with the stencils GeneratorParam as a run-time argument: what the generator built with stencils = S
// computes, for S in [1, 100].  Buffer rules, error codes and the bounds query are stencil_chain's.
extern "C" int halide_b200_stencil_chain_stencils(halide_buffer_t *input, int32_t stencils, halide_buffer_t *output) {
    return run_stencil_chain(input, stencils, output, kArgs, "stencil_chain launch");
}
HB_EXPORT_FILTER(stencil_chain, kArgs)
HB_EXPORT_AUTO_SCHEDULE(stencil_chain, kArgs)

// Batch entry points (library extensions): stencil_chain and halide_b200_stencil_chain_stencils on every frame of a 3-D
// (x, y, n) buffer, the launch plan run once per group of frames; output frame n is, bit for bit, the one-frame entry
// point's result on input frame n.
extern "C" int halide_b200_stencil_chain_batch(halide_buffer_t *input, halide_buffer_t *output) {
    return run_stencil_chain(input, kStages, output, kBatchArgs, "stencil_chain_batch launch");
}
extern "C" int halide_b200_stencil_chain_stencils_batch(halide_buffer_t *input, int32_t stencils, halide_buffer_t *output) {
    return run_stencil_chain(input, stencils, output, kBatchArgs, "stencil_chain_batch launch");
}
