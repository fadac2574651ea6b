// local_laplacian.cu — host side of local_laplacian(input, levels, alpha, beta, output) for sm_90a:
// the C-ABI entry points (reference: apps/local_laplacian/local_laplacian_generator.cpp:12-16,287 and
// the harness apps/local_laplacian/process.cpp:31), argument validation, pyramid geometry, scratch
// allocation, the launch sequence, and the row-sharded multi-GPU variant.  Kernels and the HBM layout of the
// callee-owned scratch: ll_kernels.cuh.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "hb_dist.h"
#include "ll_kernels.cuh"

namespace {

using namespace llk;

int g_shard_coarse_level = 0;  // halide_b200_ll_shard_coarse_level: 0 = choose by size, n >= 2 = gather level n
int g_force_naive = 0;  // test hook bitmask (halide_b200_ll_force_generic): 1 = generic down kernels, 2 = generic up, 4 = generic final, 8 = no fused coarse launch, 16 = general-layout final kernel, 64 = no TMA frame tile in the final kernel

int64_t est_i[3][2] = {{0, 1536}, {0, 2560}, {0, 3}};
const int64_t *const est_ptrs[6] = {&est_i[0][0], &est_i[0][1], &est_i[1][0], &est_i[1][1], &est_i[2][0], &est_i[2][1]};
const halide_scalar_value_t sv_levels = hb::scalar_i32(8), sv_alpha = hb::scalar_f32(1.0f), sv_beta = hb::scalar_f32(1.0f);
// Argument records as the generator declares them (generator :12-16, estimates :92-99).
const halide_filter_argument_t kArgs[5] = {
    {"input", halide_argument_kind_input_buffer, 3, {halide_type_uint, 16, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
    {"levels", halide_argument_kind_input_scalar, 0, {halide_type_int, 32, 0}, nullptr, nullptr, nullptr, &sv_levels, nullptr},
    {"alpha", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv_alpha, nullptr},
    {"beta", halide_argument_kind_input_scalar, 0, {halide_type_float, 32, 0}, nullptr, nullptr, nullptr, &sv_beta, nullptr},
    {"output", halide_argument_kind_output_buffer, 3, {halide_type_uint, 16, 0}, nullptr, nullptr, nullptr, nullptr, est_ptrs},
};
// halide_b200_local_laplacian_batch: the same buffers with a fourth dimension, the frame index n.
const halide_filter_argument_t kBatchArgs[2] = {hb::variant(kArgs[0], 1), hb::variant(kArgs[4], 1)};
// halide_b200_local_laplacian_u8 / _u8_batch: uint8 buffers of 3 / 4 dimensions.
const halide_filter_argument_t kU8Args[2] = {hb::variant(kArgs[0], 0, hb::kU8), hb::variant(kArgs[4], 0, hb::kU8)};
const halide_filter_argument_t kU8BatchArgs[2] = {hb::variant(kArgs[0], 1, hb::kU8), hb::variant(kArgs[4], 1, hb::kU8)};

// Everything one call needs on the device: frame description + per-level buffers, for N frames of one geometry.
// T = the frame's element type (uint16_t, or uint8_t for the 8-bit entry points).
template<typename T>
struct PlanT {
    LLFrameT<T> f;
    LevelSetDeep ls{};  // levels 1 .. J-1 (level 0 is never stored: its slot stays zero)
    int J = ll::kMaxJ;  // pyramid levels (8 but for the pyramid_levels entry points)
    int N;  // frames (1 but for a batch)
    FrameStrides fs;  // all zero when N == 1 (but the pixel pitches); level slots: levels 0 .. 7
    LevelStridesDeep deep{};  // the level strides of every level (all zero when N == 1): those of levels past 7 live only here
    float alpha;
    bool il = false;  // interleaved frames (the kernels' IL instantiations)
};
using Plan = PlanT<uint16_t>;

// The non-final up-sweep launches read only the frame's scalars (levels, remap table), never a sample, so one
// instantiation of them serves every element type: they get the frame description retyped to uint16_t.
template<typename T>
LLFrame scalars_frame(const LLFrameT<T> &f) {
    if constexpr (std::is_same<T, uint16_t>::value) {
        return f;
    } else {
        static_assert(sizeof(LLFrame) == sizeof(LLFrameT<T>), "frame descriptions differ only in their pointer types");
        LLFrame g;
        memcpy(&g, &f, sizeof g);
        return g;
    }
}

// Grids index frames by blockIdx.z; batches beyond its limit launch in groups of frames [n0, n0 + count).
template<typename P, typename F>
void for_frame_groups(const P &p, F launch) {
    for (int n0 = 0; n0 < p.N; n0 += hb::kMaxGridZ) launch(n0, std::min(hb::kMaxGridZ, p.N - n0));
}

// The checks local_laplacian and its sharded and batch variants share, on args = {input, output}.  *done: return r now
// (an error, a bounds query or an empty output).  J: the pyramid_levels GeneratorParam, checked after levels.
int check_and_query(hb::Arg *args, int levels, bool *done, int J = ll::kMaxJ) {
    int r;
    *done = true;
    if ((r = hb::check_args(args, 2))) return r;
    // The only access that bypasses repeat_edge is input(x,y,c) in `color` (generator :84), so the input must cover
    // exactly the output region.
    const halide_buffer_t *output = args[1].b;
    const hb::Region need[2] = {hb::region_of(output, true), hb::region_of(output, false)};
    if (hb::answer_bounds_query(args, need, 2)) return 0;
    if ((r = hb::check_shapes(args, 2)) || (r = hb::check_required(args, need, 2))) return r;
    if (levels < 2 || levels > 32) {
        // 1/(levels-1) (generator :41) is meaningless below 2; the reference does not check, we do.
        return hb::fail(levels < 2 ? halide_error_code_param_too_small : halide_error_code_param_too_large,
                        "Parameter levels is %d but must be in [2, 32]", levels);
    }
    if (J < 1 || J > ll::kMaxLevels) {
        return hb::fail(J < 1 ? halide_error_code_param_too_small : halide_error_code_param_too_large,
                        "Parameter pyramid_levels is %d but must be in [1, %d]", J, ll::kMaxLevels);
    }
    for (int d = 0; d < output->dimensions; d++) {
        if (output->dim[d].extent <= 0) return 0;
    }
    *done = false;
    return 0;
}

template<typename T>
void fill_frame(PlanT<T> &p, const hb::Arg *args, int levels, float alpha, float beta) {
    const halide_buffer_t *input = args[0].b, *output = args[1].b;
    const hb::Clip c = hb::clip_of(args[0], args[1], 3);
    LLFrameT<T> &f = p.f;
    f.in = (const T *)args[0].dev + c.in_off;  // output frame n reads input frame n
    f.in_sy = input->dim[1].stride; f.in_sc = input->dim[2].stride;
    f.in_x0 = input->dim[0].min; f.in_y0 = input->dim[1].min; f.in_c0 = input->dim[2].min;
    f.in_w = input->dim[0].extent; f.in_h = input->dim[1].extent; f.in_c = input->dim[2].extent;
    f.clamp_y0 = f.in_y0; f.clamp_h = f.in_h;
    f.halo_top = f.halo_bot = nullptr;
    f.halo_top_rows = f.halo_bot_rows = f.halo_pitch = 0;
    f.out = (T *)args[1].dev;
    f.out_sy = output->dim[1].stride; f.out_sc = output->dim[2].stride;
    f.out_x0 = output->dim[0].min; f.out_y0 = output->dim[1].min; f.out_c0 = output->dim[2].min;
    f.W = output->dim[0].extent; f.H = output->dim[1].extent; f.C = output->dim[2].extent;
    p.fs = FrameStrides{};
    // interleaved buffers: channel stride 1 (in_sc / out_sc above), pixel pitch dim[0].stride
    p.il = args[0].interleaved;
    p.fs.px_in = p.il ? input->dim[0].stride : 1;
    p.fs.px_out = p.il ? output->dim[0].stride : 1;
    p.N = c.N;
    if (p.N > 1) {  // (one frame keeps stride 0: the same layout checks, hence kernels, as the 3-D call)
        p.fs.in = c.in_sn;
        p.fs.out = c.out_sn;
    }
    f.levels = levels;
    f.beta = beta;
    f.flm1 = (float)(levels - 1);
    f.inv_lm1 = 1.0f / (float)(levels - 1);
    f.lut_half = 256 * (levels - 1);
    p.alpha = alpha;
}

// ---- remap table: recomputed only when (levels, alpha) change --------------------------------------------------
// alpha is a runtime scalar, but a caller (the harness's benchmark loop, a video stream) passes the same value call
// after call: the 2*256*(levels-1)+1 halide_exp evaluations and their launch are kept per device and reused.  The table
// is immutable once built (a change of parameters builds a new one; the old ones are kept: kernels of an earlier call
// may still be reading them on another stream), and it is built synchronously, so any stream may read it afterwards.
// A call holds its table (holders > 0, LutHold) from the lookup until its last launch that reads it is enqueued: another
// thread's miss may evict in between, and cudaDeviceSynchronize only waits for work already enqueued.  Eviction frees the
// unheld tables once 64 of them are cached; held ones stay until a later eviction.
struct LutEntry {
    int device, levels;
    float alpha;
    float *lut;
    int holders;
};
std::mutex g_lut_mu;
std::vector<LutEntry> g_luts;

// The table of (current device, levels, alpha), built on stream s if missing, with one hold taken on it.
int lut_acquire(int levels, float alpha, cudaStream_t s, float **out) {
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(g_lut_mu);
    for (LutEntry &e : g_luts) {
        if (e.device == dev && e.levels == levels && memcmp(&e.alpha, &alpha, sizeof(float)) == 0) {
            e.holders++;
            *out = e.lut;
            return 0;
        }
    }
    // a caller sweeping alpha: drop the unheld tables once nothing can still be reading them
    if (std::count_if(g_luts.begin(), g_luts.end(), [](const LutEntry &e) { return e.holders == 0; }) >= 64) {
        cudaDeviceSynchronize();
        auto unheld = std::stable_partition(g_luts.begin(), g_luts.end(), [](const LutEntry &e) { return e.holders > 0; });
        for (auto it = unheld; it != g_luts.end(); ++it) cudaFree(it->lut);
        g_luts.erase(unheld, g_luts.end());
    }
    float *lut = nullptr;
    const int lut_half = 256 * (levels - 1), n = 2 * lut_half + 1;
    if (cudaMalloc((void **)&lut, ((size_t)n + 3) / 4 * 16) != cudaSuccess) {
        cudaGetLastError();
        return hb::fail(halide_error_code_device_malloc_failed, "local_laplacian: remap table allocation failed");
    }
    HB_LAUNCH("ll_lut", ll_lut_kernel, (n + 255) / 256, 256, 0, s, lut, lut_half, alpha);
    if (cudaStreamSynchronize(s) != cudaSuccess) {
        cudaGetLastError();
        cudaFree(lut);
        return hb::fail(halide_error_code_device_run_failed, "local_laplacian: remap table kernel failed");
    }
    g_luts.push_back({dev, levels, alpha, lut, 1});
    *out = lut;
    return 0;
}

// Drops one hold taken by lut_acquire; false if the table is not held.
bool lut_release(const float *lut) {
    std::lock_guard<std::mutex> lock(g_lut_mu);
    for (LutEntry &e : g_luts) {
        if (e.lut == lut && e.holders > 0) {
            e.holders--;
            return true;
        }
    }
    return false;
}

// A call's hold on its remap table, dropped when the call returns (after its last launch, or on an error).
struct LutHold {
    float *lut = nullptr;
    LutHold() = default;
    LutHold(const LutHold &) = delete;
    LutHold &operator=(const LutHold &) = delete;
    ~LutHold() {
        if (lut) lut_release(lut);
    }
};

template<typename T>
int get_lut(PlanT<T> &p, cudaStream_t s, LutHold &hold) {
    int r;
    if ((r = lut_acquire(p.f.levels, p.alpha, s, &hold.lut))) return r;
    p.f.lut = hold.lut;
    return 0;
}

// the fast level-1 kernel also produces level 2 (so the pyramid must have one: J >= 3).  It and ll_down_rows sum a
// downsample's 16 taps before one * 1/64 where the generator scales by 1/8 after each pass, which overflows 8 times
// sooner.  A level value is at most |beta| + 1 + 0.61 |alpha| in magnitude (remap(x) <= e^-1/2 |alpha|), so with both
// scalars below 2^100 no such sum comes near the float range; larger or non-finite ones take the generic kernels, which
// scale as the generator does.
template<typename P>
bool fast_down(const P &p) {
    return p.f.levels == 8 && p.J >= 3 && !(g_force_naive & 1) && fabsf(p.alpha) < 0x1p100f && fabsf(p.f.beta) < 0x1p100f;
}
// the fast final kernel also produces outGPyramid[1] (for its own tile) from level 2, so no up-sweep launch runs for
// level 1 (J >= 3 as well)
template<typename P>
bool fast_final(const P &p) { return p.f.levels == 8 && p.J >= 3 && !(g_force_naive & 4) && p.f.C <= 3; }
// lowest level the up-sweep launches produce
template<typename P>
int first_up_level(const P &p) { return fast_final(p) ? 2 : 1; }

template<typename P>
int alloc_levels(P &p, const ll::Geom &geom, hb::Scratch &scratch) {
    const int nq = (p.f.levels + 1) / 2;
    for (int j = 1; j < p.J; j++) {
        const ll::Level &lv = geom.lv[j];
        LevelBuf &b = p.ls.lv[j];
        b.sx = lv.sx; b.sy = lv.sy; b.ox = lv.ox; b.oy = lv.oy;
        b.cy = lv.cy; b.coy = lv.oy; b.gy = lv.gy;
        b.xo = lv.xo; b.nq = nq;
        b.gpitch = lv.gpitch; b.opitch = lv.opitch;
        // one allocation per array for all N frames; a frame's slice starts on 256 bytes, like an allocation of its own
        auto slice = [](size_t floats) { return (int64_t)((floats + 63) & ~size_t(63)); };
        const size_t gpix = (size_t)b.sy.n() * b.gpitch;
        const bool with_outg = j >= first_up_level(p);  // (level 1's is computed inside the fast final kernel)
        const int64_t gp_sn = slice(gpix * nq * 2), ing_sn = slice(gpix), outg_sn = with_outg ? slice((size_t)b.oy.n() * b.opitch) : 0;
        b.gp = scratch.get<float>((size_t)gp_sn * p.N);
        b.ing = scratch.get<float>((size_t)ing_sn * p.N);
        b.outg = with_outg ? scratch.get<float>((size_t)outg_sn * p.N) : nullptr;
        if (p.N > 1) {
            p.deep.gp[j] = gp_sn, p.deep.ing[j] = ing_sn, p.deep.outg[j] = outg_sn;
            if (j < ll::kMaxJ) p.fs.gp[j] = gp_sn, p.fs.ing[j] = ing_sn, p.fs.outg[j] = outg_sn;
        }
        if (!b.gp || !b.ing || (with_outg && !b.outg)) {
            return hb::fail(halide_error_code_device_malloc_failed, "local_laplacian: scratch allocation failed");
        }
    }
    return 0;
}

// ---- launch helpers ------------------------------------------------------------------------------------
const dim3 kBlk(32, 8);
dim3 grid_for(int w, int h, int nf) { return dim3((w + 31) / 32, (h + 7) / 8, nf); }  // z = frames

// Returns f(std::bool_constant<b>{}...) for the run-time flags b...: each becomes a template argument of the kernel f picks.
template<typename F>
auto with_flags(F &&f) { return f(); }
template<typename F, typename... B>
auto with_flags(F &&f, bool b, B... bs) {
    if (b) return with_flags([&](auto... c) { return f(std::true_type{}, c...); }, bs...);
    return with_flags([&](auto... c) { return f(std::false_type{}, c...); }, bs...);
}

// Whether each address, and each offset or stride in bytes, is a multiple of n bytes.
template<typename... B>
bool multiples_of(int64_t n, B... bytes) { return (((int64_t)(uintptr_t)bytes % n == 0) && ...); }

// The layouts the final and tone kernels have forms for: any planar or interleaved frame (General, GeneralIL), aligned
// planar words (Aligned; AlignedTma: with the final kernel's frame tile by TMA) and the frames il_form names.
enum class Form { General, GeneralIL, Aligned, AlignedTma, Rgb, RgbaToRgb, Rgba };

// An interleaved frame's aligned form, if its layout has one: channels [0, 3) of RGB -> RGB, RGBA -> RGB and RGBA -> RGBA
// frames, where an RGBA input must describe its fourth channel (the aligned forms read whole pixels).
template<typename T>
Form il_form(const PlanT<T> &p) {
    const int pin = p.fs.px_in, pout = p.fs.px_out;
    const bool rgb = p.f.C == 3 && p.f.in_c0 == 0 && p.f.out_c0 == 0 && p.f.in_c == pin &&
                     ((pin == 3 && pout == 3) || (pin == 4 && (pout == 3 || pout == 4)));
    return !rgb ? Form::GeneralIL : pin == 3 ? Form::Rgb : pout == 3 ? Form::RgbaToRgb : Form::Rgba;
}

// Levels 1 and 2 from the frame (K == 8): stores level-1 rows cy1 and level-2 rows cy2, reading the frame through f
// (the row-sharded path narrows both spans, and hides the halo rows from the launch that runs before they arrive).
template<bool BETA1, bool FRAMES, bool IL, typename T>
void launch_level12_kernel(PlanT<T> &p, const LLFrameT<T> &f, Span cy1, Span cy2, cudaStream_t s) {
    LevelBuf d1 = p.ls.lv[1], d2 = p.ls.lv[2];
    d1.cy = cy1;
    d2.cy = cy2;
    // one pair table and a stage per strip walker (warp pair or warp): one block per SM
    constexpr int pairs = kL1Walkers<FRAMES, T>;
    const size_t smem = kPairLutN * sizeof(float2) + pairs * sizeof(DownStage);
    const int slots = hb::resident_blocks(ll_level1_kernel<BETA1, FRAMES, T, IL>, kDWarps * 32, smem);
    // strips of 28 level-1 columns from xbase == xo (mod 4), far enough left that their level-2 columns (xbase/2 + 14k ..)
    // reach level 2's first column; chunks of 8 level-1 rows from an odd ybase, over the rows stored and the taps of
    // the level-2 rows stored
    const int xbase = d1.xo - ((d1.xo - 2 * d2.sx.lo > 0 ? d1.xo - 2 * d2.sx.lo + 3 : 0) & ~3);
    const int ns = std::max((d1.sx.hi - xbase) / kDCols + 1, (d2.sx.hi - xbase / 2) / (kDCols / 2) + 1);
    int lo = INT32_MAX, hi = INT32_MIN;
    if (cy1.n() > 0) lo = cy1.lo, hi = cy1.hi;
    if (cy2.n() > 0) lo = std::min(lo, 2 * cy2.lo - 1), hi = std::max(hi, 2 * cy2.hi + 2);
    if (lo > hi) return;
    const int ybase = lo - ((lo & 1) ^ 1);
    const int nc = (hi - ybase) / kDR + 1;
    // nr chunk ranges per strip: the fewest step-equivalents per walker over the rounds of runs (a lead-in computes 2 of
    // a chunk's 8 rows: a quarter chunk), over the N * ns strips of the batch.  Warp pairs take, of the counts within 1 %
    // of the fewest, the most ranges (the shortest runs): counts the cost puts within 1 % of each other ran up to 5 %
    // apart, the shorter runs faster (16K on an H100, DESIGN §9).
    const long long np = (long long)slots * pairs, strips = (long long)p.N * ns;
    std::vector<long long> cost(nc + 1);
    int nr = 1;
    for (int r = 1; r <= nc; r++) {
        cost[r] = (strips * r + np - 1) / np * (4ll * ((nc + r - 1) / r) + 1);
        if (cost[r] < cost[nr]) nr = r;
    }
    if (kL1Pairs<FRAMES, T>) {
        const long long best = cost[nr];
        for (nr = nc; cost[nr] * 100 > best * 101;) nr--;
    }
    const long long runs = strips * nr;
    const int g = (int)std::min<long long>(slots, (runs + pairs - 1) / pairs);
    // aligned 4-byte words (a column pair of uint16, the pairs of two lanes of uint8): every byte offset between the
    // frame's first element and a staged word is a multiple of 4; 32-bit element offsets from the frame's first element
    const int64_t eb = sizeof(T);
    const int wide = multiples_of(4, f.in, f.in_sy * eb, f.in_sc * eb, p.fs.in * eb, f.in_x0 * eb, f.halo_top, f.halo_bot, f.halo_pitch * eb);
    // (an interleaved frame's columns are px_in elements apart: its last sample is up to in_w * px_in further)
    const int idx32 = f.in_sy > 0 && f.in_sc > 0 &&
                      (int64_t)f.in_h * f.in_sy + (int64_t)f.in_c * f.in_sc + (IL ? (int64_t)f.in_w * p.fs.px_in : 0) < (1ll << 31);
    HB_LAUNCH("ll_level1", (ll_level1_kernel<BETA1, FRAMES, T, IL>), g, kDWarps * 32, smem, s, f, d1, d2, xbase, ybase, ns, nc, nr, wide, idx32,
              p.N, p.fs);
}

template<typename T>
void launch_level12(PlanT<T> &p, const LLFrameT<T> &f, Span cy1, Span cy2, cudaStream_t s) {
    with_flags([&](auto beta1, auto frames, auto il) { launch_level12_kernel<beta1, frames, il>(p, f, cy1, cy2, s); },
               p.f.beta == 1.0f, p.N > 1, p.il);
}

// The strides a launch that produces level j reads, and the index that stands for level j in them (*js).  FrameStrides'
// level arrays have ll::kMaxJ slots, and such a launch reads those of levels j - 1 .. j + 1: up to J == 8 the plan's own
// strides at j itself.  In a deeper pyramid the levels from 7 on, whose neighbours could reach slot 8, get a copy whose
// slots 5 .. 7 hold the strides of levels j - 1 .. j + 1 and j is slot 6 (a single frame's are all zero, as the copy's).
template<typename P>
FrameStrides level_strides(const P &p, int j, int *js) {
    *js = p.J <= ll::kMaxJ ? j : std::min(j, ll::kMaxJ - 2);
    if (*js == j) return p.fs;
    FrameStrides w = p.fs;
    for (int k = 0; k < 3; k++) {
        const int lv = j - 1 + k;  // (level J, the top's neighbour above, does not exist: stride 0)
        w.gp[*js - 1 + k] = lv < p.J ? p.deep.gp[lv] : 0;
        w.ing[*js - 1 + k] = lv < p.J ? p.deep.ing[lv] : 0;
        w.outg[*js - 1 + k] = lv < p.J ? p.deep.outg[lv] : 0;
    }
    return w;
}

template<typename T>
void launch_down(PlanT<T> &p, int j, cudaStream_t s) {  // produce level j (j >= 1) rows cy
    LevelBuf *lb = p.ls.lv;
    if (fast_down(p)) {
        if (j == 1) {
            launch_level12(p, p.f, lb[1].cy, lb[2].cy, s);
        } else if (j > 2 && lb[j].cy.n() > 0) {
            // stored levels: load-bound row-group kernel
            const int ns = (lb[j].sx.n() + kRCols - 1) / kRCols, ng = (lb[j].cy.n() + kRG - 1) / kRG;
            const long long tasks = (long long)ns * ng * 5 * p.N;
            int js;
            const FrameStrides fs = level_strides(p, j, &js);
            const auto kern = with_flags([](auto frames) { return ll_down_rows_kernel<frames>; }, p.N > 1);
            const int slots = hb::resident_blocks(kern, 256, 0);
            HB_LAUNCH("ll_down_rows", kern, (int)std::min<long long>(slots, (tasks + 7) / 8), 256, 0, s, lb[j - 1], lb[j], ns, ng, p.N, js, fs);
        }
    } else if (lb[j].cy.n() <= 0) {
        return;
    } else if (j == 1) {
        for_frame_groups(p, [&](int n0, int nf) {
            HB_LAUNCH("ll_level1_generic", ll_level1_naive_kernel<T>, grid_for(lb[1].sx.n(), lb[1].cy.n(), nf), kBlk, 0, s, at_frame(p.f, p.fs, n0),
                      at_frame(lb[1], 1, p.fs, n0), p.fs);
        });
    } else {
        int js;
        const FrameStrides fs = level_strides(p, j, &js);
        for_frame_groups(p, [&](int n0, int nf) {
            HB_LAUNCH("ll_down", ll_down_naive_kernel, grid_for(lb[j].sx.n(), lb[j].cy.n(), nf), kBlk, 0, s, at_frame(lb[j - 1], js - 1, fs, n0),
                      at_frame(lb[j], js, fs, n0), p.f.levels, js, fs);
        });
    }
}

dim3 up_grid(int x_lo, int x_hi, int y_lo, int y_hi, int nf) {  // tiles on even absolute origins; z = frames
    return dim3((x_hi - (x_lo & ~1) + kUpTW) / kUpTW, (y_hi - (y_lo & ~1) + kUpTH) / kUpTH, nf);
}

template<typename P>
void launch_up(P &p, int j, cudaStream_t s) {  // produce outGPyramid[j] (1 <= j <= J-1) rows coy
    LevelBuf *lb = p.ls.lv;
    if (lb[j].coy.n() <= 0) return;
    const bool fast_up = p.f.levels == 8 && !(g_force_naive & 2);
    const bool top = j == p.J - 1;
    int js;
    const FrameStrides fs = level_strides(p, j, &js);
    for_frame_groups(p, [&](int n0, int nf) {
        if (fast_up && !top) {
            static const CUtensorMap no_map = {};
            const auto kern = with_flags([](auto frames) { return ll_up2_kernel<false, false, true, false, frames>; }, nf > 1);
            HB_LAUNCH("ll_up2", kern, up_grid(lb[j].ox.lo, lb[j].ox.hi, lb[j].coy.lo, lb[j].coy.hi, nf), 256, up2_smem_bytes(false, false), s,
                      scalars_frame(at_frame(p.f, fs, n0)), at_frame(lb[j], js, fs, n0), at_frame(lb[j + 1], js + 1, fs, n0), no_map, js, fs);
        } else {
            const int jc = top ? j : j + 1;
            HB_LAUNCH("ll_up", ll_up_naive_kernel, grid_for(lb[j].ox.n(), lb[j].coy.n(), nf), kBlk, 0, s, at_frame(lb[j], js, fs, n0),
                      at_frame(lb[jc], top ? js : js + 1, fs, n0), p.f.flm1, p.f.levels, top ? 1 : 0, js, fs);
        }
    });
}

// The fast final kernel's form for a call (the forms from AlignedTma on also need the frame tile's map, per group of
// frames).  Its ALIGNED path (32-bit addressing) moves one aligned word of two pixels per thread and channel, wb bytes, so
// every pointer and element offset to such a word is a multiple of wb bytes.  Interleaved frames take it with fixed pitches:
// the frame tile by TMA, and a pixel pair's output samples stored together as wb-byte words (so the output's base, row and
// frame strides in bytes are multiples of wb, and both its columns and the input's start even).
template<typename T>
Form final_form(const PlanT<T> &p) {
    const bool general = g_force_naive & 16, tile_tma = !(g_force_naive & 64);
    const LLFrameT<T> &f = p.f;
    const int64_t eb = sizeof(T), wb = 2 * eb;
    if (p.il) {
        const bool pairs = f.W % 2 == 0 && f.out_x0 % 2 == 0 && f.in_x0 % 2 == 0 && f.out_sy > 0 &&
                           multiples_of(wb, f.out, f.out_sy * eb, p.fs.out * eb);
        return pairs && !general && tile_tma ? il_form(p) : Form::GeneralIL;
    }
    const int64_t in_span = (int64_t)f.in_h * f.in_sy + 3 * f.in_sc, out_span = (int64_t)f.H * f.out_sy + 3 * f.out_sc;
    const bool aligned = f.C == 3 && f.in_c0 == 0 && f.out_c0 == 0 && f.in_c >= 3 && f.in_sy > 0 && f.in_sc > 0 && f.out_sy > 0 &&
                         f.out_sc > 0 && in_span < (1ll << 31) && out_span < (1ll << 31) &&
                         multiples_of(wb, f.W * eb, f.out_x0 * eb, f.in_x0 * eb, f.in, f.out, f.in_sy * eb, f.in_sc * eb,
                                      f.out_sy * eb, f.out_sc * eb, p.fs.in * eb, p.fs.out * eb);
    return !aligned || general ? Form::General : tile_tma ? Form::AlignedTma : Form::Aligned;
}

// The final kernel's frame tile by TMA for the nf frames from `in`: false if the buffer breaks TMA's rules (16-byte aligned
// base and strides) or a tile's first column would not start on a 16-byte boundary.  The map describes the input buffer
// itself, (x, y, c), or (x, y) with x over an interleaved RGB frame's samples or an RGBA frame's 4-sample pixels, and the
// group's frames as one more dimension if there are several: a tile reaching past it reads zeros, for pixels never stored.
template<typename T>
bool frame_tile_map(const PlanT<T> &p, const T *in, int nf, CUtensorMap *map) {
    const LLFrameT<T> &f = p.f;
    const int64_t eb = sizeof(T);
    const int xs = p.il && p.fs.px_in == 3 ? 3 : 1;
    uint64_t dims[4] = {(uint64_t)xs * f.in_w, (uint64_t)f.in_h};
    uint32_t box[4] = {(uint32_t)(xs * up_in_w<T>()), kUpTH};
    int64_t strides[3] = {f.in_sy * eb};
    int rank = 2;
    if (!p.il) dims[rank] = f.in_c, box[rank] = 3, strides[rank - 1] = f.in_sc * eb, rank++;
    if (nf > 1) dims[rank] = nf, box[rank] = 1, strides[rank - 1] = p.fs.in * eb, rank++;
    const CUtensorMapDataType dt = p.il && p.fs.px_in == 4 ? (eb == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT64)
                                                          : (eb == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16);
    return tma::strides_ok(in, strides, rank - 1) && multiples_of(16, ((f.out_x0 & ~1) - f.in_x0) * eb) &&
           tma::encode(map, dt, rank, (void *)in, dims, strides, box);
}

template<typename T>
void launch_final(PlanT<T> &p, cudaStream_t s) {
    LevelBuf *lb = p.ls.lv;
    const LLFrameT<T> &f = p.f;
    if (!fast_final(p)) {
        for_frame_groups(p, [&](int n0, int nf) {
            HB_LAUNCH("ll_final", ll_final_naive_kernel<T>, grid_for(f.W, f.H, nf), kBlk, 0, s, at_frame(f, p.fs, n0), at_frame(lb[1], 1, p.fs, n0),
                      1, p.fs);
        });
        return;
    }
    const Form form = final_form(p);
    for_frame_groups(p, [&](int n0, int nf) {
        const LLFrameT<T> fg = at_frame(f, p.fs, n0);
        CUtensorMap in_map = {};
        Form g = form;
        if (form >= Form::AlignedTma && !frame_tile_map(p, fg.in, nf, &in_map)) g = form == Form::AlignedTma ? Form::Aligned : Form::GeneralIL;
        // (the kernels of one element type take the same parameters)
        const auto kern = with_flags([&](auto beta1, auto frames) {
            switch (g) {
            case Form::General: return ll_up2_kernel<true, false, beta1, false, frames, T>;
            case Form::GeneralIL: return ll_up2_kernel<true, false, beta1, false, frames, T, 0, 0>;
            case Form::Aligned: return ll_up2_kernel<true, true, beta1, false, frames, T>;
            case Form::AlignedTma: return ll_up2_kernel<true, true, beta1, true, frames, T>;
            case Form::Rgb: return ll_up2_kernel<true, true, beta1, true, frames, T, 3, 3>;
            case Form::RgbaToRgb: return ll_up2_kernel<true, true, beta1, true, frames, T, 4, 3>;
            default: return ll_up2_kernel<true, true, beta1, true, frames, T, 4, 4>;  // Form::Rgba
            }
        }, f.beta == 1.0f, nf > 1);
        const int smem = up2_smem_bytes(true, g >= Form::AlignedTma, (int)sizeof(T), g >= Form::RgbaToRgb ? 4 : 3);
        hb::allow_smem(kern, smem);
        HB_LAUNCH("ll_final2", kern, up_grid(f.out_x0, f.out_x0 + f.W - 1, f.out_y0, f.out_y0 + f.H - 1, nf), 256, smem, s, fg,
                  at_frame(lb[1], 1, p.fs, n0), at_frame(lb[2], 2, p.fs, n0), in_map, 1, p.fs);
    });
}

// Coarse tail in one cooperative launch: levels j0+1 .. J-1 down and up (see ll_coarse_fused_kernel).
template<typename P>
bool launch_coarse_fused(P &p, int j0, cudaStream_t s) {
    if (!hb::cooperative_launch()) return false;
    // J <= 8: the LevelSet instantiations, on the first 8 slots; a deeper pyramid takes all of LevelSetDeep, and a deeper
    // batch the strides of every level too
    LevelSet ls8;
    memcpy(ls8.lv, p.ls.lv, sizeof ls8.lv);
    const bool deep = p.J > ll::kMaxJ, frames = p.N > 1;
    const void *kern = with_flags([](auto D, auto F) {
        return (const void *)ll_coarse_fused_kernel<F, std::conditional_t<D, LevelSetDeep, LevelSet>,
                                                    std::conditional_t<D && F, LevelStridesDeep, FrameStrides>>;
    }, deep, frames);
    const int max_blocks = std::min(hb::resident_blocks(kern, 256, 0), 2 * hb::sm_count());
    int J = p.J, K = p.f.levels, levels = p.f.levels, jd = fast_down(p) && j0 < 2 ? 2 : j0, nf = p.N;
    float flm1 = p.f.flm1;
    void *args[] = {deep ? (void *)&p.ls : (void *)&ls8, &J, &j0, &jd, &K, &flm1, &levels, &nf,
                    deep && frames ? (void *)&p.deep : (void *)&p.fs};
    hb::count_launch("ll_coarse_fused", s);
    cudaError_t e = cudaLaunchCooperativeKernel((void *)kern, dim3(max_blocks), dim3(256), args, 0, s);
    hb::after_launch(s);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return true;
}

// Last level of the sweep from from_level that has launches of its own: the levels above it, of at most 40 K pixels each
// (all N frames'), share the fused tail.
template<typename P>
int last_own_level(const P &p, int from_level) {
    int j0 = p.J - 1;
    if (!(g_force_naive & 8)) {
        // (level 1 always has its own launch: it is built from the frame, not from a stored level; on the fast path that
        // launch also builds level 2, and the fused tail's down-sweep starts after it).  The size is the batch's: all N
        // frames' pixels of the level.
        const int j_min = from_level < 1 ? 1 : from_level;
        while (j0 > j_min && (int64_t)p.ls.lv[j0].sx.n() * p.ls.lv[j0].sy.n() * p.N <= 40 * 1024) j0--;
    }
    return j0;
}

// Levels from_level+1 .. J-1 down, then J-1 .. from_level+1 up: the part of the sweep that runs on whole levels
// (everything on one GPU; the replicated coarse levels when row-sharded).  Small levels share one cooperative launch.
template<typename P>
void run_coarse_sweep(P &p, int from_level, cudaStream_t s) {
    // j0 = last level produced by its own launch; levels j0+1.. are fused (if any)
    const int j0 = last_own_level(p, from_level);
    bool fused = false;
    for (int j = from_level + 1; j <= j0; j++) launch_down(p, j, s);
    if (j0 < p.J - 1) fused = launch_coarse_fused(p, j0, s);
    if (!fused) {
        for (int j = j0 + 1; j < p.J; j++) launch_down(p, j, s);
        for (int j = p.J - 1; j > j0; j--) launch_up(p, j, s);
    }
    for (int j = j0; j > from_level && j >= first_up_level(p); j--) launch_up(p, j, s);
}

// J = 1: the whole filter is the pointwise tone kernel over the output region (ll_tone_kernel), one launch per group of
// frames.  Its aligned forms move a unit of kTonePx pixels as whole words, so every byte offset from a unit's first
// sample to another's (rows, planes, frames) and the first unit's address are multiples of the word size: planar frames,
// one word per plane row of kTonePx samples (16 bytes of uint16, 8 of uint8); interleaved RGB / RGBA frames of channels
// [0, 3), the unit's run of 8 * pitch samples (16-byte words, 8-byte ones for uint8 RGB), and for an RGBA output the word
// of a pixel's R and G (an RGBA input must describe its fourth channel: the run covers whole pixels).
template<typename T>
Form tone_form(const PlanT<T> &p) {
    const bool general = g_force_naive & 16;
    const LLFrameT<T> &f = p.f;
    const int pin = p.fs.px_in, pout = p.fs.px_out;
    const int64_t eb = sizeof(T);
    const T *in0 = f.in + (int64_t)(f.out_y0 - f.in_y0) * f.in_sy + (int64_t)(f.out_x0 - f.in_x0) * pin;
    if (p.il) {
        auto run_word = [&](int pitch) -> int64_t { return multiples_of(16, kTonePx * pitch * eb) ? 16 : 8; };
        const int64_t ai = run_word(pin), ao = pout == 3 ? run_word(3) : 2 * eb;
        const bool words = multiples_of(ai, in0, f.in_sy * eb, p.fs.in * eb) && multiples_of(ao, f.out, f.out_sy * eb, p.fs.out * eb);
        return words && !general ? il_form(p) : Form::GeneralIL;
    }
    const bool vec = multiples_of(kTonePx * eb, in0, f.in_sy * eb, f.in_sc * eb, p.fs.in * eb, f.out, f.out_sy * eb, f.out_sc * eb, p.fs.out * eb);
    return vec && !general ? Form::Aligned : Form::General;
}

template<typename T>
void launch_tone(PlanT<T> &p, cudaStream_t s) {
    const LLFrameT<T> &f = p.f;
    const int upr = (f.W + kTonePx - 1) / kTonePx;
    const long long units = (long long)upr * f.H;
    const size_t smem = (size_t)(2 * f.lut_half + 1) * sizeof(float);
    // the planar uint16 single-frame form: units counted in 64 bits, one launch
    auto launch1 = [&](auto kern) {
        const int slots = hb::resident_blocks(kern, 256, smem);  // (smem is above 48 KB for levels > 24)
        const int g = (int)std::min<long long>(slots, (units + 255) / 256);
        HB_LAUNCH("ll_tone", kern, g, 256, smem, s, f, upr, units, p.fs);
    };
    // the others: frame blockIdx.z of each group, the resident blocks shared out over the group's frames; their unit index
    // is 32-bit, so a frame of 2^31 units or more runs in bands of rows
    auto launch = [&](auto kern) {
        const int slots = hb::resident_blocks(kern, 256, smem);
        const int band = (int)std::min<long long>(f.H, INT32_MAX / upr);
        for_frame_groups(p, [&](int n0, int nf) {
            for (int y0 = 0; y0 < f.H; y0 += band) {
                LLFrameT<T> fb = at_frame(f, p.fs, n0);
                fb.out += (int64_t)y0 * f.out_sy;
                fb.out_y0 += y0;
                fb.H = std::min(band, f.H - y0);
                const long long bu = (long long)upr * fb.H;
                const dim3 g((unsigned)std::max<long long>(1, std::min<long long>((bu + 255) / 256, (slots + nf - 1) / nf)), 1, nf);
                HB_LAUNCH("ll_tone", kern, g, 256, smem, s, fb, upr, bu, p.fs);
            }
        });
    };
    const Form form = tone_form(p);
    if constexpr (std::is_same<T, uint16_t>::value) {
        if (!p.il && p.N == 1) return with_flags([&](auto vec) { launch1(ll_tone_kernel<vec>); }, form == Form::Aligned);
    }
    switch (form) {
    case Form::General: return launch(ll_tone_kernel<false, T, 1, 1, true>);
    case Form::Aligned: return launch(ll_tone_kernel<true, T, 1, 1, true>);
    case Form::GeneralIL: return launch(ll_tone_kernel<false, T, 0, 0, true>);
    case Form::Rgb: return launch(ll_tone_kernel<true, T, 3, 3, true>);
    case Form::RgbaToRgb: return launch(ll_tone_kernel<true, T, 4, 3, true>);
    case Form::Rgba: return launch(ll_tone_kernel<true, T, 4, 4, true>);
    case Form::AlignedTma: break;  // (final kernel only)
    }
}

// One GPU, args = {input, output} of 3 dimensions (one frame) or 4 (a batch of frames along dimension 3), elements T;
// J = pyramid levels (8 but for the pyramid_levels entry points).
template<typename T>
int run_local_laplacian(hb::Arg *args, int levels, float alpha, float beta, int J, const char *what) {
    int r;
    bool done;
    if ((r = check_and_query(args, levels, &done, J)) || done) return r;
    if ((r = hb::acquire(args, 2))) return r;

    PlanT<T> p;
    fill_frame(p, args, levels, alpha, beta);
    p.J = J;
    const int W = p.f.W, H = p.f.H;
    Span outx = {p.f.out_x0, p.f.out_x0 + W - 1}, outy = {p.f.out_y0, p.f.out_y0 + H - 1};
    Span inx = {p.f.in_x0, p.f.in_x0 + p.f.in_w - 1}, iny = {p.f.in_y0, p.f.in_y0 + p.f.in_h - 1};
    hb::Scratch scratch;
    if ((r = alloc_levels(p, ll::make_geom(outx, outy, inx, iny, J), scratch))) return r;

    cudaStream_t s = hb::stream();
    LutHold lut;
    if ((r = get_lut(p, s, lut))) return r;
    {
        hb::CallTimer timer(s);
        if (J == 1) {
            launch_tone(p, s);
        } else {
            run_coarse_sweep(p, 0, s);
            launch_final(p, s);
        }
    }
    return hb::finish(args, 2, what);
}

}  // namespace

extern "C" int local_laplacian(halide_buffer_t *input, int32_t levels, float alpha, float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kArgs[0]}, {output, kArgs[4]}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian launch");
}
HB_EXPORT_FILTER(local_laplacian, kArgs)

// Batch entry point (library extension): every frame of a 4-D (x, y, c, n) buffer through one launch sequence.
extern "C" int halide_b200_local_laplacian_batch(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                 halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kBatchArgs[0]}, {output, kBatchArgs[1]}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_batch launch");
}

// 8-bit entry points (library extensions): out8 = to_u8(local_laplacian(to_u16(in8))) with the reference's element
// conversions, computed in one pass — the conversions happen inside the kernels that read and write the frame.
extern "C" int halide_b200_local_laplacian_u8(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                              halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8Args[0]}, {output, kU8Args[1]}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_u8 launch");
}
extern "C" int halide_b200_local_laplacian_u8_batch(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                    halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8BatchArgs[0]}, {output, kU8BatchArgs[1]}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_u8_batch launch");
}

// Interleaved entry points (library extensions): the four above on pixel-interleaved buffers (RGBRGB..., RGBA...:
// dim[2].stride == 1, dim[0].stride = the pixel pitch, at least the channel extent), bit for bit what they give on planar
// copies of the same buffers.  The argument records are the planar ones; only the layout rule checked differs.
extern "C" int halide_b200_local_laplacian_interleaved(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                       halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kArgs[0], nullptr, true}, {output, kArgs[4], nullptr, true}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_interleaved launch");
}
extern "C" int halide_b200_local_laplacian_interleaved_batch(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                             halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kBatchArgs[0], nullptr, true}, {output, kBatchArgs[1], nullptr, true}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_interleaved_batch launch");
}
extern "C" int halide_b200_local_laplacian_u8_interleaved(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                          halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8Args[0], nullptr, true}, {output, kU8Args[1], nullptr, true}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_u8_interleaved launch");
}
extern "C" int halide_b200_local_laplacian_u8_interleaved_batch(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                                halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8BatchArgs[0], nullptr, true}, {output, kU8BatchArgs[1], nullptr, true}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, ll::kMaxJ, "local_laplacian_u8_interleaved_batch launch");
}
// The harness's second AOT variant (apps/local_laplacian/process.cpp:44-48): same implementation.
HB_EXPORT_AUTO_SCHEDULE(local_laplacian, kArgs)

// local_laplacian with the pyramid_levels GeneratorParam J (generator :6,10) as a run-time argument, 1 <= J <= 20: what
// the generator built with pyramid_levels = J computes, on the buffers local_laplacian takes.  J = 8 is local_laplacian
// itself (the same launches); J >= 3 runs the same kernels over J levels (the fast level-1 and final kernels need level
// 2), J = 2 the generic ones, and J = 1, where the filter is pointwise, only ll_tone.
extern "C" int halide_b200_local_laplacian_pyramid_levels(halide_buffer_t *input, int32_t pyramid_levels, int32_t levels, float alpha,
                                                          float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kArgs[0]}, {output, kArgs[4]}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, pyramid_levels, "local_laplacian_pyramid_levels launch");
}

// halide_b200_local_laplacian_pyramid_levels on the buffers of the batch, 8-bit and interleaved entry points above: each
// is its fixed-depth counterpart with J chosen per call (J = 8: the same launches), and on every frame bit for bit what
// halide_b200_local_laplacian_pyramid_levels gives on a planar uint16 copy (converted as the 8-bit entry points convert).
extern "C" int halide_b200_local_laplacian_pyramid_levels_batch(halide_buffer_t *input, int32_t pyramid_levels, int32_t levels, float alpha,
                                                                float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kBatchArgs[0]}, {output, kBatchArgs[1]}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, pyramid_levels, "local_laplacian_pyramid_levels_batch launch");
}
extern "C" int halide_b200_local_laplacian_pyramid_levels_u8(halide_buffer_t *input, int32_t pyramid_levels, int32_t levels, float alpha,
                                                             float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8Args[0]}, {output, kU8Args[1]}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, pyramid_levels, "local_laplacian_pyramid_levels_u8 launch");
}
extern "C" int halide_b200_local_laplacian_pyramid_levels_u8_batch(halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                                   float alpha, float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8BatchArgs[0]}, {output, kU8BatchArgs[1]}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, pyramid_levels, "local_laplacian_pyramid_levels_u8_batch launch");
}
extern "C" int halide_b200_local_laplacian_pyramid_levels_interleaved(halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                                      float alpha, float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kArgs[0], nullptr, true}, {output, kArgs[4], nullptr, true}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, pyramid_levels, "local_laplacian_pyramid_levels_interleaved launch");
}
extern "C" int halide_b200_local_laplacian_pyramid_levels_interleaved_batch(halide_buffer_t *input, int32_t pyramid_levels,
                                                                            int32_t levels, float alpha, float beta,
                                                                            halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kBatchArgs[0], nullptr, true}, {output, kBatchArgs[1], nullptr, true}};
    return run_local_laplacian<uint16_t>(args, levels, alpha, beta, pyramid_levels,
                                         "local_laplacian_pyramid_levels_interleaved_batch launch");
}
extern "C" int halide_b200_local_laplacian_pyramid_levels_u8_interleaved(halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                                         float alpha, float beta, halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8Args[0], nullptr, true}, {output, kU8Args[1], nullptr, true}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, pyramid_levels, "local_laplacian_pyramid_levels_u8_interleaved launch");
}
extern "C" int halide_b200_local_laplacian_pyramid_levels_u8_interleaved_batch(halide_buffer_t *input, int32_t pyramid_levels,
                                                                               int32_t levels, float alpha, float beta,
                                                                               halide_buffer_t *output) {
    hb::Arg args[2] = {{input, kU8BatchArgs[0], nullptr, true}, {output, kU8BatchArgs[1], nullptr, true}};
    return run_local_laplacian<uint8_t>(args, levels, alpha, beta, pyramid_levels,
                                        "local_laplacian_pyramid_levels_u8_interleaved_batch launch");
}

namespace {

// Row-sharded path: the level gathered all-to-all (levels from it upwards are replicated on every rank).
// Depends only on the whole frame's geometry and the rank count, so every rank computes the same value.
int choose_coarse_level(const ll::Geom &whole, int nranks, int J, int K) {
    if (g_shard_coarse_level > 0) return g_shard_coarse_level < 2 ? 2 : (g_shard_coarse_level > J - 1 ? J - 1 : g_shard_coarse_level);
    // The gathered level trades the two messages of a call against each other: gathering a finer level means a bigger
    // all-to-all (a rank receives (N-1)/N of the level: gPyramid + inGPyramid, (K + 1) floats per pixel) but a smaller
    // input halo (about 3 * 2^j frame rows of three uint16 channels per rank, which also is the recomputed work).  Pick the
    // level with the fewest bytes received per rank; ties go to the finer level (less recompute).
    const double frame_row_bytes = (double)whole.lv[0].sx.n() * 3 * sizeof(uint16_t);
    int best = J - 1;
    double best_bytes = 1e300;
    for (int j = 2; j < J; j++) {
        const double halo = 3.0 * (double)(1 << j) * frame_row_bytes;
        const double level = (double)whole.lv[j].sy.n() * whole.lv[j].gpitch * (K + 1) * sizeof(float);
        const double bytes = halo + level * (nranks - 1) / (nranks > 0 ? nranks : 1);
        if (bytes < best_bytes) {
            best_bytes = bytes;
            best = j;
        }
    }
    return best;
}

// ---- row-sharded variant (one process per GPU) -----------------------------------------------------------
// `input`/`output` describe this rank's band: all columns and channels of the frame, rows
// [dim[1].min, dim[1].min + extent) in the frame's coordinates.  frame_y_min/extent give the rows of the whole
// frame; ranks must be ordered top to bottom (rank r-1 holds the rows directly above rank r's).
// Communication per call (SURVEY.md §8e, see ll_geom.h): ONE exchange of input halo rows with the two neighbours
// (the only place the stencil footprint of the sharded levels crosses the shard boundary — every pyramid row a band
// needs beyond itself is recomputed from them) and ONE all-to-all gather of the coarse level jr; both are NCCL
// point-to-point groups on the compute stream.  Everything else is the single-GPU kernels on this rank's rows.
struct ShardPlan {  // per geometry: every rank's band (gathered once), reused call after call
    int key[11];
    bool valid = false;
    std::vector<int> bands;  // [lo, hi] per rank
};
thread_local ShardPlan g_shard;  // (per thread: the ranks of an in-process loopback group are threads of one process)

int run_local_laplacian_sharded(halide_buffer_t *input, int levels, float alpha, float beta, halide_buffer_t *output,
                                int frame_y_min, int frame_y_extent) {
    int r;
    bool done;
    hb::Arg args[2] = {{input, kArgs[0]}, {output, kArgs[4]}};
    if ((r = check_and_query(args, levels, &done)) || done) return r;
    if (!hbdist::active()) {
        return hb::fail(halide_error_code_generic_error, "local_laplacian_sharded: call halide_b200_dist_init first");
    }
    const int rank = hbdist::rank(), nranks = hbdist::size();
    Span band = {output->dim[1].min, output->dim[1].min + output->dim[1].extent - 1};
    if (input->dim[1].min != band.lo || input->dim[1].extent != band.n()) {
        return hb::fail(halide_error_code_constraint_violated,
                        "local_laplacian_sharded: input rows [%d,%d) must equal the output band [%d,%d)", input->dim[1].min,
                        input->dim[1].min + input->dim[1].extent, band.lo, band.hi + 1);
    }
    const bool first = rank == 0, last = rank == nranks - 1;
    Span frame_y = {frame_y_min, frame_y_min + frame_y_extent - 1};
    if ((first && band.lo != frame_y.lo) || (last && band.hi != frame_y.hi) || band.lo < frame_y.lo || band.hi > frame_y.hi) {
        return hb::fail(halide_error_code_constraint_violated, "local_laplacian_sharded: band [%d,%d] inconsistent with frame rows [%d,%d] on rank %d/%d",
                        band.lo, band.hi, frame_y.lo, frame_y.hi, rank, nranks);
    }
    if (input->dim[0].min != output->dim[0].min || input->dim[0].extent != output->dim[0].extent) {
        return hb::fail(halide_error_code_constraint_violated, "local_laplacian_sharded: input and output bands must span the same columns");
    }
    if ((r = hb::acquire(args, 2))) return r;

    Plan p;
    fill_frame(p, args, levels, alpha, beta);
    const int W = p.f.W, C = p.f.in_c;
    Span outx = {p.f.out_x0, p.f.out_x0 + W - 1};
    Span inx = {p.f.in_x0, p.f.in_x0 + p.f.in_w - 1};
    const ll::Geom whole = ll::make_geom(outx, frame_y, inx, frame_y, ll::kMaxJ);
    const int jr = choose_coarse_level(whole, nranks, ll::kMaxJ, p.f.levels);

    // every rank's band: gathered once per geometry (collective on first use / change) and per communicator (a rank
    // that kept its plan from an earlier group would skip the gather its new peers enter)
    const int key[11] = {W, band.lo, band.hi, frame_y.lo, frame_y.hi, rank, nranks, C, jr, levels, hbdist::epoch()};
    if (!g_shard.valid || memcmp(g_shard.key, key, sizeof(key)) != 0) {
        int mine[2] = {band.lo, band.hi};
        g_shard.valid = false;  // (until the gather succeeds)
        g_shard.bands.assign(2 * (size_t)nranks, 0);
        if ((r = hbdist::allgather_bytes(mine, g_shard.bands.data(), sizeof(mine)))) return r;
        for (int q = 0; q + 1 < nranks; q++) {
            if (g_shard.bands[2 * q + 1] + 1 != g_shard.bands[2 * q + 2]) {
                return hb::fail(halide_error_code_constraint_violated,
                                "local_laplacian_sharded: rank %d's band ends at row %d but rank %d's starts at %d", q,
                                g_shard.bands[2 * q + 1], q + 1, g_shard.bands[2 * q + 2]);
            }
        }
        memcpy(g_shard.key, key, sizeof(key));
        g_shard.valid = true;
    }
    auto band_of = [&](int q) { return Span{g_shard.bands[2 * q], g_shard.bands[2 * q + 1]}; };
    auto rows_of = [&](int q, ll::ShardLevel *sl, Span *need) {
        ll::compute_shard_rows(whole, frame_y, band_of(q), q == 0, q == nranks - 1, jr, sl, need);
    };
    // Bands too thin to shard: checked for every rank, not only this one, so that all ranks refuse the same frame
    // (a rank refusing alone would leave its neighbours waiting in the exchange).  need[q]: input rows rank q reads.
    std::vector<Span> need(nranks);
    for (int q = 0; q < nranks; q++) {
        ll::ShardLevel t[ll::kMaxJ];
        rows_of(q, t, &need[q]);
        for (int j = 1; j <= jr && j < ll::kMaxJ; j++) {
            if (t[j].own.n() < 1) {
                return hb::fail(halide_error_code_constraint_violated,
                                "local_laplacian_sharded: rank %d's band of %d rows is too small for %d ranks (level %d owns no row)", q,
                                band_of(q).n(), nranks, j);
            }
        }
        const int above = band_of(q).lo - need[q].lo, below = need[q].hi - band_of(q).hi;
        if (above > (q == 0 ? 0 : band_of(q - 1).n()) || below > (q == nranks - 1 ? 0 : band_of(q + 1).n())) {
            return hb::fail(halide_error_code_constraint_violated,
                            "local_laplacian_sharded: rank %d's input halo (%d rows above, %d below) is larger than the bands next to it", q,
                            above, below);
        }
    }
    ll::ShardLevel sl[ll::kMaxJ];
    Span in_need;
    rows_of(rank, sl, &in_need);
    p.f.clamp_y0 = frame_y.lo;
    p.f.clamp_h = frame_y.n();
    hb::Scratch scratch;
    if ((r = alloc_levels(p, ll::make_shard_geom(whole, sl, jr), scratch))) return r;

    // ---- input halo: rows [in_need.lo, band.lo) from the rank above, (band.hi, in_need.hi] from the rank below ----
    const int ht = band.lo - in_need.lo, hbn = in_need.hi - band.hi;
    const size_t rowb = (size_t)p.f.in_w * sizeof(uint16_t);
    uint16_t *halo_top = nullptr, *halo_bot = nullptr, *send_up = nullptr, *send_dn = nullptr;
    // rows the rank above needs from my top (its bottom halo) / the rank below needs from my bottom (its top halo)
    const int up_need = first ? 0 : need[rank - 1].hi - band_of(rank - 1).hi;
    const int dn_need = last ? 0 : band_of(rank + 1).lo - need[rank + 1].lo;
    if (ht) halo_top = scratch.get<uint16_t>((size_t)C * ht * p.f.in_w);
    if (hbn) halo_bot = scratch.get<uint16_t>((size_t)C * hbn * p.f.in_w);
    if (up_need) send_up = scratch.get<uint16_t>((size_t)C * up_need * p.f.in_w);
    if (dn_need) send_dn = scratch.get<uint16_t>((size_t)C * dn_need * p.f.in_w);
    if ((ht && !halo_top) || (hbn && !halo_bot) || (up_need && !send_up) || (dn_need && !send_dn)) {
        return hb::fail(halide_error_code_device_malloc_failed, "local_laplacian_sharded: scratch allocation failed");
    }
    p.f.halo_pitch = p.f.in_w;
    p.f.halo_top = halo_top; p.f.halo_bot = halo_bot;
    p.f.halo_top_rows = ht; p.f.halo_bot_rows = hbn;

    cudaStream_t s = hb::stream();
    LutHold lut;  // (held through the exchanges too: this rank waits there for its peers before it launches)
    if ((r = get_lut(p, s, lut))) return r;
    // A halo pack that fails is reported only once the call is over: every rank still enters each exchange of the call,
    // so that no neighbour is left waiting for this one.
    cudaError_t pack_err = cudaSuccess;
    {
        hb::CallTimer timer(s);
        // pack my boundary rows per channel ([c][row][w], the layout of the receiver's halo arrays) and exchange — on a
        // second stream, so that the level-1 kernel's interior rows (every source row inside the band) run meanwhile;
        // only the few level-1 rows at the band's edges wait for the halo (HALIDE_B200_SHARD_OVERLAP=0: one stream)
        static const bool overlap = [] {
            const char *e = getenv("HALIDE_B200_SHARD_OVERLAP");
            return !(e && e[0] == '0');
        }();
        static thread_local cudaStream_t comm_stream = nullptr;
        static thread_local cudaEvent_t ev_in = nullptr, ev_halo = nullptr;
        if (overlap && !comm_stream) {
            cudaStreamCreateWithFlags(&comm_stream, cudaStreamNonBlocking);
            cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming);
            cudaEventCreateWithFlags(&ev_halo, cudaEventDisableTiming);
        }
        bool exchanged_async = false;
        {
            cudaStream_t xs = overlap ? comm_stream : s;
            if (overlap) {  // the input (and the previous call's use of the scratch blocks) is ordered on s
                cudaEventRecord(ev_in, s);
                cudaStreamWaitEvent(xs, ev_in, 0);
            }
            // `rows` rows from `src` on, packed [row][w]: one 2-D copy when they run forward at least a row apart, else row
            // by row (a flipped or zero row stride, which cudaMemcpy2D's unsigned pitch cannot express; a few rows each)
            auto pack = [&](uint16_t *dst, const uint16_t *src, int rows) {
                if (p.f.in_sy >= p.f.in_w) {
                    return cudaMemcpy2DAsync(dst, rowb, src, (size_t)p.f.in_sy * sizeof(uint16_t), rowb, rows, cudaMemcpyDeviceToDevice, xs);
                }
                for (int i = 0; i < rows; i++) {
                    cudaError_t e = cudaMemcpyAsync(dst + (size_t)i * p.f.in_w, src + (int64_t)i * p.f.in_sy, rowb, cudaMemcpyDeviceToDevice, xs);
                    if (e != cudaSuccess) return e;
                }
                return cudaSuccess;
            };
            hbdist::Msg msgs[4];
            int n = 0;
            auto keep_first = [&](cudaError_t e) {
                if (pack_err == cudaSuccess) pack_err = e;
            };
            for (int c = 0; c < C; c++) {
                const uint16_t *plane = p.f.in + (int64_t)c * p.f.in_sc;
                if (up_need) keep_first(pack(send_up + (size_t)c * up_need * p.f.in_w, plane, up_need));
                if (dn_need) keep_first(pack(send_dn + (size_t)c * dn_need * p.f.in_w, plane + (int64_t)(p.f.in_h - dn_need) * p.f.in_sy, dn_need));
            }
            if (up_need) msgs[n++] = {send_up, (size_t)C * up_need * rowb, rank - 1, true};
            if (dn_need) msgs[n++] = {send_dn, (size_t)C * dn_need * rowb, rank + 1, true};
            if (ht) msgs[n++] = {halo_top, (size_t)C * ht * rowb, rank - 1, false};
            if (hbn) msgs[n++] = {halo_bot, (size_t)C * hbn * rowb, rank + 1, false};
            if (n) {
                hb::profile_begin("nccl_input_halo", xs);  // (event-bracketed in profile mode like a kernel launch; not counted as one)
                r = hbdist::exchange(msgs, n, xs);
                hb::after_launch(xs);
                if (r) return r;
                if (overlap) {
                    cudaEventRecord(ev_halo, xs);
                    exchanged_async = true;
                }
            }
        }
        LevelBuf *lb = p.ls.lv;
        if (exchanged_async && fast_down(p)) {
            // levels 1 and 2 in up to three launches: the interior rows (every source row inside the band) now, with the
            // halo rows hidden from the kernel, and the rows at each edge after the halo
            const Span cy = lb[1].cy, cy2 = lb[2].cy;
            const int i_lo = std::max(cy.lo, (p.f.in_y0 + 2) >> 1);                // smallest y with 2y-1 >= in_y0
            const int i_hi = std::min(cy.hi, (p.f.in_y0 + p.f.in_h - 3) >> 1);      // largest y with 2y+2 <= in_y0 + in_h - 1
            if (i_lo > i_hi) {  // (band too thin to have interior rows)
                cudaStreamWaitEvent(s, ev_halo, 0);
                launch_down(p, 1, s);
            } else {
                // level-2 rows whose taps 2y-1 .. 2y+2 are all interior level-1 rows
                const Span c2 = {std::max(cy2.lo, (i_lo + 2) >> 1), std::min(cy2.hi, (i_hi - 2) >> 1)};
                const Span top2 = {cy2.lo, std::min(cy2.hi, c2.lo - 1)};
                const Span bot2 = {std::max(c2.hi, top2.hi) + 1, cy2.hi};
                LLFrame fi = p.f;
                fi.halo_top = fi.halo_bot = nullptr;
                fi.halo_top_rows = fi.halo_bot_rows = 0;
                launch_level12(p, fi, {i_lo, i_hi}, c2, s);
                cudaStreamWaitEvent(s, ev_halo, 0);
                if (cy.lo < i_lo || top2.n() > 0) launch_level12(p, p.f, {cy.lo, i_lo - 1}, top2, s);
                if (i_hi < cy.hi || bot2.n() > 0) launch_level12(p, p.f, {i_hi + 1, cy.hi}, bot2, s);
            }
        } else {
            if (exchanged_async) cudaStreamWaitEvent(s, ev_halo, 0);
            launch_down(p, 1, s);
        }
        for (int j = 2; j <= jr; j++) launch_down(p, j, s);  // (level jr: only the rows this rank owns)
        // ---- gather level jr: my rows to every rank, every rank's rows into my whole-frame copy ----
        {
            std::vector<hbdist::Msg> msgs;
            const size_t gp_row = (size_t)lb[jr].nq * lb[jr].gpitch * 2 * sizeof(float), ing_row = (size_t)lb[jr].gpitch * sizeof(float);
            auto rows_msg = [&](Span rows, int peer, bool send) {
                if (rows.n() <= 0) return;
                const size_t off = (size_t)(rows.lo - lb[jr].sy.lo);
                msgs.push_back({(char *)lb[jr].gp + off * gp_row, (size_t)rows.n() * gp_row, peer, send});
                msgs.push_back({(char *)lb[jr].ing + off * ing_row, (size_t)rows.n() * ing_row, peer, send});
            };
            for (int q = 0; q < nranks; q++) {
                if (q == rank) continue;
                Span own_q[ll::kMaxJ];
                ll::compute_band_own(whole, band_of(q), q == 0, q == nranks - 1, own_q);
                rows_msg(sl[jr].own, q, true);
                rows_msg(own_q[jr], q, false);
            }
            if (!msgs.empty()) {
                hb::profile_begin("nccl_level_gather", s);
                r = hbdist::exchange(msgs.data(), (int)msgs.size(), s);
                hb::after_launch(s);
                if (r) return r;
            }
        }
        lb[jr].cy = lb[jr].sy;   // from here on level jr is complete
        run_coarse_sweep(p, jr, s);          // levels jr+1.. down, ..jr+1 up, whole frame, on every rank
        launch_up(p, jr, s);
        for (int j = jr - 1; j >= first_up_level(p); j--) launch_up(p, j, s);
        launch_final(p, s);
    }
    if (pack_err != cudaSuccess) {
        cudaGetLastError();  // (the copy's error, reported here instead)
        return hb::check_cuda(pack_err, "local_laplacian_sharded halo pack", halide_error_code_device_run_failed);
    }
    return hb::finish(args, 2, "local_laplacian_sharded launch");
}

}  // namespace

// Test hook: route K == 8 calls through the generic (any `levels`) kernels so both paths stay covered.
extern "C" void halide_b200_ll_force_generic(int enable) {
    g_force_naive = enable;
}

// Test hook: take (hold = 1) or drop (hold = 0) one hold on the remap table of (levels, alpha) on the current device, as a
// call does between its lookup and its last launch; taking builds the table (on the calling thread's stream) if it is
// missing.  A held table survives evictions.  0, or a negative halide_error_code_t.
extern "C" int halide_b200_ll_lut_hold(int32_t levels, float alpha, int32_t hold) {
    if (levels < 2 || levels > 32) {
        return hb::fail(levels < 2 ? halide_error_code_param_too_small : halide_error_code_param_too_large,
                        "Parameter levels is %d but must be in [2, 32]", levels);
    }
    float *lut = nullptr;
    if (hold) return lut_acquire(levels, alpha, hb::stream(), &lut);
    int dev = 0;
    cudaGetDevice(&dev);
    {
        std::lock_guard<std::mutex> lock(g_lut_mu);
        for (const LutEntry &e : g_luts) {
            if (e.device == dev && e.levels == levels && memcmp(&e.alpha, &alpha, sizeof(float)) == 0) lut = e.lut;
        }
    }
    if (!lut || !lut_release(lut)) {
        return hb::fail(halide_error_code_generic_error, "halide_b200_ll_lut_hold: the remap table of levels %d, alpha %g is not held",
                        levels, (double)alpha);
    }
    return 0;
}

// Row-sharded path: which pyramid level is gathered all-to-all (see run_local_laplacian_sharded).  Collective
// setting: every rank must use the same value.  0 = choose by size (default), n >= 2 = level n.
extern "C" void halide_b200_ll_shard_coarse_level(int level) {
    g_shard_coarse_level = level < 0 ? 0 : level;
}

// Probe for the CPU-side tests (no CUDA calls): the level halide_b200_local_laplacian_sharded gathers for a
// frame of frame_w x frame_h split over nranks ranks.
extern "C" int halide_b200_ll_shard_plan_level(int32_t frame_w, int32_t frame_h, int32_t nranks) {
    Span fx = {0, frame_w - 1}, fy = {0, frame_h - 1};
    return choose_coarse_level(ll::make_geom(fx, fy, fx, fy, ll::kMaxJ), nranks, ll::kMaxJ, 8);
}

// Probe for the CPU-side tests (no CUDA calls): the last pyramid level that halide_b200_local_laplacian_pyramid_levels
// gives launches of its own on a frame_w x frame_h frame (input == output region); the levels above it share the fused
// coarse tail.
extern "C" int halide_b200_ll_last_own_level(int32_t frame_w, int32_t frame_h, int32_t pyramid_levels) {
    if (frame_w < 1 || frame_h < 1 || pyramid_levels < 1 || pyramid_levels > ll::kMaxLevels) return -1;
    Span fx = {0, frame_w - 1}, fy = {0, frame_h - 1};
    const ll::Geom g = ll::make_geom(fx, fy, fx, fy, pyramid_levels);
    Plan p;
    p.J = pyramid_levels;
    p.N = 1;
    for (int j = 0; j < p.J; j++) p.ls.lv[j].sx = g.lv[j].sx, p.ls.lv[j].sy = g.lv[j].sy;
    return last_own_level(p, 0);
}

// Row-sharded entry point (library extension; see run_local_laplacian_sharded).
extern "C" int halide_b200_local_laplacian_sharded(halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                   halide_buffer_t *output, int32_t frame_y_min, int32_t frame_y_extent) {
    return run_local_laplacian_sharded(input, levels, alpha, beta, output, frame_y_min, frame_y_extent);
}

// Band geometry probe for the CPU-side tests of the sharding logic (no CUDA calls): for a band [band_lo, band_hi] of a
// frame_w x frame_h frame and gathered level jr, fills out[j*8 .. j*8+7] = {own.lo, own.hi, d.lo, d.hi, u.lo, u.hi,
// S_j.lo, S_j.hi} (ll_geom.h: ShardLevel; S_j = the level's stored rows on the whole frame) for j = 0..7 and
// out[64..65] = the input rows [lo, hi] the band's level-1 rows read.
extern "C" int halide_b200_ll_band_geometry(int32_t frame_w, int32_t frame_h, int32_t band_lo, int32_t band_hi, int32_t first,
                                            int32_t last, int32_t jr, int32_t *out) {
    Span fx = {0, frame_w - 1}, fy = {0, frame_h - 1};
    ll::Geom whole = ll::make_geom(fx, fy, fx, fy, ll::kMaxJ);
    ll::ShardLevel sl[ll::kMaxJ];
    Span need;
    ll::compute_shard_rows(whole, fy, Span{band_lo, band_hi}, first != 0, last != 0, jr, sl, &need);
    for (int j = 0; j < ll::kMaxJ; j++) {
        int32_t *o = out + j * 8;
        o[0] = sl[j].own.lo; o[1] = sl[j].own.hi; o[2] = sl[j].d.lo; o[3] = sl[j].d.hi;
        o[4] = sl[j].u.lo; o[5] = sl[j].u.hi; o[6] = whole.lv[j].sy.lo; o[7] = whole.lv[j].sy.hi;
    }
    out[64] = need.lo;
    out[65] = need.hi;
    return 0;
}

// Device self-test of the arithmetic shortcuts used by the fast kernels (shared-reciprocal division, magic-number
// conversions): returns the number of mismatches against div.rn / cvt over n pseudo-random operand sets, or -1.
extern "C" long long halide_b200_selftest_arith(unsigned long long n, unsigned long long seed) {
    unsigned long long *bad = nullptr, host = 0;
    if (cudaMalloc(&bad, sizeof(*bad)) != cudaSuccess) return -1;
    cudaMemset(bad, 0, sizeof(*bad));
    cudaStream_t s = hb::stream();
    HB_LAUNCH("ll_selftest", ll_selftest_kernel, 132 * 8, 256, 0, s, n, seed, bad);
    if (cudaMemcpyAsync(&host, bad, sizeof(host), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
        cudaFree(bad);
        return -1;
    }
    cudaFree(bad);
    return (long long)host;
}
