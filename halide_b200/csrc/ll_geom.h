// ll_geom.h — pyramid geometry of local_laplacian shared by the host FFI code and the kernels.
//
// Halide evaluates every pyramid level as a pure function on an ENLARGED region derived by bounds
// inference (only the input is edge-clamped, SURVEY.md finding 5; generator
// apps/local_laplacian/local_laplacian_generator.cpp:28,266-282).  Because the input is constant
// outside its own bounds, each level is constant beyond a small border: if level j is constant
// for x <= L_j and for x >= R_j then level j+1 (which reads 2x-1 .. 2x+2) is constant for
// x <= floor((L_j-2)/2) and x >= ceil((R_j+1)/2).  The kernels therefore store level j only on
// S_j = G_j ∩ [L_j, R_j] and clamp coordinates into S_j when reading — bit-identical to the
// enlarged-region evaluation (the oracle evaluates the enlarged regions literally and the parity
// tests compare the two), at ~W/2^j + 3 columns per level instead of W/2^j + 2^(J-j+1).
#pragma once
#include <stdint.h>

namespace ll {

constexpr int kMaxJ = 8;  // pyramid_levels GeneratorParam of the shipped app (generator :10): the level slots of the kernels'
                          // LevelSet / FrameStrides, and J of every entry point but halide_b200_local_laplacian_pyramid_levels
constexpr int kMaxLevels = 20;  // the generator's largest pyramid_levels (maxJ, generator :6): sizes the host-side geometry

struct Span {
    int lo, hi;  // inclusive
    __host__ __device__ int n() const { return hi - lo + 1; }
};

__host__ __device__ inline int fdiv2(int a) { return a >> 1; }  // Euclidean /2 on signed ints

struct Level {
    Span sx, sy;   // stored region of the Gaussian-side planes (gPyramid[j] K planes + inGPyramid[j])
    Span ox, oy;   // region of outGPyramid[j], stored and computed here (oy: the rank's rows when row-sharded)
    Span cy;       // Gaussian-side rows this device COMPUTES (== sy on one GPU; the owned band when row-sharded)
    Span gy;       // rows of the whole frame's S_j (== sy on one GPU): the clamp range
    int xo;        // even column origin of the Gaussian-side arrays: column x lives at index x - xo
    int gpitch;    // pixels per row of the Gaussian-side planes
    int opitch;    // pixels per row of the outG plane
};

struct Geom {
    int J;
    Level lv[kMaxLevels];
};

// out_[xy]: output region; in_[xy]: bounds of the input buffer (for the clamp / constant borders).
inline void compute_axis(Span out, Span in, int J, Span *S, Span *O) {
    Span G[kMaxLevels];
    O[0] = out;
    for (int j = 1; j < J; j++) O[j] = {fdiv2(O[j - 1].lo - 1), fdiv2(O[j - 1].hi + 1)};
    G[J - 1] = O[J - 1];
    for (int j = J - 2; j >= 0; j--) {
        int lo = 2 * G[j + 1].lo - 1, hi = 2 * G[j + 1].hi + 2;
        G[j] = {O[j].lo < lo ? O[j].lo : lo, O[j].hi > hi ? O[j].hi : hi};
    }
    int L = in.lo, R = in.hi;
    for (int j = 0; j < J; j++) {
        if (j > 0) {
            L = fdiv2(L - 2);
            R = fdiv2(R + 2);  // ceil((R+1)/2)
        }
        int lo = G[j].lo > L ? G[j].lo : L;
        if (lo > G[j].hi) lo = G[j].hi;
        int hi = G[j].hi < R ? G[j].hi : R;
        if (hi < lo) hi = lo;
        S[j] = {lo, hi};
    }
}

inline Geom make_geom(Span outx, Span outy, Span inx, Span iny, int J) {
    Geom g;
    g.J = J;
    Span SX[kMaxLevels], OX[kMaxLevels], SY[kMaxLevels], OY[kMaxLevels];
    compute_axis(outx, inx, J, SX, OX);
    compute_axis(outy, iny, J, SY, OY);
    for (int j = 0; j < J; j++) {
        g.lv[j].sx = SX[j]; g.lv[j].sy = SY[j];
        g.lv[j].ox = OX[j]; g.lv[j].oy = OY[j];
        g.lv[j].cy = SY[j]; g.lv[j].gy = SY[j];
        g.lv[j].xo = SX[j].lo & ~1;  // (two's complement: rounds toward -inf, also for negative lows)
        g.lv[j].gpitch = (SX[j].hi - g.lv[j].xo + 1 + 3) & ~3;
        g.lv[j].opitch = (OX[j].n() + 3) & ~3;
    }
    return g;
}

// ---- row sharding (multi-GPU) -----------------------------------------------------------------------
// The frame's rows are split into contiguous bands, one per rank (top to bottom).  No pyramid level is exchanged
// row by row: a rank RECOMPUTES the few rows of every level that its band's taps reach beyond the band, from a halo
// of input rows fetched once per call (one exchange where the stencil footprint crosses the shard boundary), and one
// coarse level jr — small enough that its whole-frame copy is a few MB — is gathered all-to-all so that the levels
// above it are computed redundantly on every rank with no further communication.
//   own[j]   partition of level j's stored rows among the ranks: the rows whose first source row (2y) the rank owns,
//            A_{j+1} = ceil(A_j / 2); rows beyond the first / last band belong to the first / last rank.  Level jr is
//            produced by its owners and gathered.
//   u[j]     rows of outGPyramid[j] the rank needs (taps (y-1)/2, (y+1)/2 of u[j-1]; u[0] = the band)
//   d[j]     rows of gPyramid[j] / inGPyramid[j] the rank computes and holds: u[j] plus the 1-3-3-1 taps
//            2y-1 .. 2y+2 of the rows of level j+1 it computes, clipped to the level's stored rows
// Levels >= jr are held for the whole frame on every rank.
struct ShardLevel {
    Span own, d, u;
};

// The `own` partition alone (depends only on the band's ends and the whole-frame geometry).
inline void compute_band_own(const Geom &whole, Span band, bool first, bool last, Span *own) {
    int a_lo = band.lo, a_hi = band.hi + 1;  // [a_lo, a_hi)
    for (int j = 0; j < whole.J; j++) {
        if (j > 0) {
            a_lo = (a_lo + 1) >> 1;
            a_hi = (a_hi + 1) >> 1;
        }
        const Span S = whole.lv[j].sy;
        own[j].lo = first ? S.lo : (a_lo > S.lo ? a_lo : S.lo);
        own[j].hi = last ? S.hi : (a_hi - 1 < S.hi ? a_hi - 1 : S.hi);
    }
}

// Rows per level for one rank, and the input rows [in_need.lo, in_need.hi] its level-1 rows read (clipped to the frame).
inline void compute_shard_rows(const Geom &whole, Span frame_y, Span band, bool first, bool last, int jr, ShardLevel *sl,
                               Span *in_need) {
    Span own[kMaxJ];
    compute_band_own(whole, band, first, last, own);
    Span u = band;
    for (int j = 0; j < whole.J; j++) {
        if (j > 0) u = {fdiv2(u.lo - 1), fdiv2(u.hi + 1)};
        sl[j].own = own[j];
        sl[j].u = j >= jr ? whole.lv[j].oy : u;
    }
    for (int j = whole.J - 1; j >= 1; j--) {
        const Span S = whole.lv[j].sy;
        if (j >= jr) {
            sl[j].d = S;
            continue;
        }
        const Span next = (j + 1 == jr) ? sl[j + 1].own : sl[j + 1].d;  // rows of level j+1 computed here
        int lo = 2 * next.lo - 1, hi = 2 * next.hi + 2;
        if (sl[j].u.lo < lo) lo = sl[j].u.lo;
        if (sl[j].u.hi > hi) hi = sl[j].u.hi;
        if (lo < S.lo) lo = S.lo;
        if (hi > S.hi) hi = S.hi;
        sl[j].d = {lo, hi};
    }
    sl[0].d = band;
    const Span c1 = jr == 1 ? sl[1].own : sl[1].d;
    int lo = 2 * c1.lo - 1, hi = 2 * c1.hi + 2;
    if (band.lo < lo) lo = band.lo;
    if (band.hi > hi) hi = band.hi;
    if (lo < frame_y.lo) lo = frame_y.lo;
    if (hi > frame_y.hi) hi = frame_y.hi;
    *in_need = {lo, hi};
}

// Geometry of one rank: the whole frame's geometry with the y spans replaced by the rank's rows.
inline Geom make_shard_geom(const Geom &whole, const ShardLevel *sl, int jr) {
    Geom g = whole;
    for (int j = 1; j < whole.J; j++) {
        if (j >= jr) {
            // held for the whole frame; level jr is produced band by band (cy = own) and completed by the gather
            g.lv[j].cy = j == jr ? sl[j].own : whole.lv[j].sy;
            continue;
        }
        g.lv[j].sy = sl[j].d; g.lv[j].cy = sl[j].d;
        // outGPyramid rows: the rank's u rows, clipped to the level's O rows (they are a sub-range by construction)
        Span o = sl[j].u;
        if (o.lo < whole.lv[j].oy.lo) o.lo = whole.lv[j].oy.lo;
        if (o.hi > whole.lv[j].oy.hi) o.hi = whole.lv[j].oy.hi;
        g.lv[j].oy = o;
    }
    return g;
}

}  // namespace ll
