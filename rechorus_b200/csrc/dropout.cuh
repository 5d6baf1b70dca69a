// dropout.cuh -- the dropout mask of NeuMF.py:70-72 and utils/layers.py:113-117 as a pure function of an element's
// logical coordinates, so the forward, the backward, a replayed CUDA graph and SASRec's last-query block all see the same
// mask without storing it.  Element (row r, position t, column j) of dropout site `site` at training step `step`:
//   word = Philox4x32-10(ctr = (r, (t << 16) | (j >> 2), 0x80000000 | site, lo32(step)),
//                        key = (lo32(seed), hi32(seed)))[j & 3]
//   kept iff word >= thr, thr = floor(p * 2^32) (2^32 at p = 1: nothing kept); a kept element is multiplied by
//   s = float(1 / (1 - p)), s = 0 at p = 1.
// (seed, step) come from the 16-byte device snapshot b2r_dropout_tick writes once per training forward.
// oracle: tests/dropout_oracle.py dropout_mask.
#pragma once
#include <math.h>

#include "common.cuh"
#include "philox.cuh"

namespace b2r {

// kernel-side form of b2r_dropout
struct DropK {
    const uint64_t* state;     // {seed, step}
    const int64_t* lengths;    // row mapping, see b2r_dropout
    uint64_t thr;
    float scale;
    uint32_t site;
    int L;
};

// validates a b2r_dropout (0 = ok, else the error code set with its message)
int check_dropout(const b2r_dropout* d, const char* what);

static inline float dropout_scale(double p) { return p >= 1.0 ? 0.f : (float)(1.0 / (1.0 - p)); }

static inline DropK make_dropk(const b2r_dropout& d) {
    DropK k;
    k.state = d.state;
    k.lengths = d.lengths;
    k.thr = (uint64_t)floor(d.p * 4294967296.0);
    k.scale = dropout_scale(d.p);
    k.site = (uint32_t)d.site;
    k.L = d.L;
    return k;
}

struct DropKey {
    uint32_t k0, k1, step;
};

__device__ __forceinline__ DropKey drop_key(const DropK& d) {
    const unsigned long long* s = reinterpret_cast<const unsigned long long*>(d.state);
    const unsigned long long seed = __ldg(s), step = __ldg(s + 1);
    return DropKey{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)step};
}

// the four mask words of columns 4 jq .. 4 jq + 3 of activation row `row`.  Row -> (r, t): L == 0: (row, 0) (NeuMF's
// [B*C, w] activations); lengths == NULL: (row / L, row % L) (a [B, L, d] block); else (row, clamp(lengths[row] - 1, 0,
// L - 1)) (one row per sequence at the position select_last reads)
__device__ __forceinline__ uint4 drop_words(const DropK& d, const DropKey& k, int64_t row, uint32_t jq) {
    uint32_t r, t;
    if (d.L == 0) {
        r = (uint32_t)row;
        t = 0;
    } else if (d.lengths == nullptr) {
        r = (uint32_t)(row / d.L);
        t = (uint32_t)(row % d.L);
    } else {
        const int64_t tl = d.lengths[row] - 1;
        r = (uint32_t)row;
        t = (uint32_t)(tl < 0 ? 0 : (tl > d.L - 1 ? d.L - 1 : tl));
    }
    return philox4x32_10(r, (t << 16) | jq, 0x80000000u | d.site, k.step, k.k0, k.k1);
}

__device__ __forceinline__ uint32_t drop_word(const uint4& w, int i) {
    return i == 0 ? w.x : (i == 1 ? w.y : (i == 2 ? w.z : w.w));
}

__device__ __forceinline__ float drop_apply(const DropK& d, uint32_t word, float v) {
    return (uint64_t)word >= d.thr ? v * d.scale : 0.f;
}

// keep bit of one word
__device__ __forceinline__ uint32_t drop_keep(const DropK& d, uint32_t word) { return (uint64_t)word >= d.thr ? 1u : 0u; }

// The keep bits of one row of d <= 256 columns for the scalar (one warp per row) kernels: bit i of lane l is column
// l + 32 i.  Lane l draws the four words of column groups l and 32 + l (one Philox each, where the group exists) and the
// warp hands them out as 4-bit nibbles, so a row costs the warp one or two Philox evaluations.  Warp-uniform call.
__device__ __forceinline__ uint32_t drop_row_bits(const DropK& d, const DropKey& k, int64_t row, int ncols, int lane) {
    const int ng = (ncols + 3) >> 2;
    uint32_t nib0 = 0, nib1 = 0;
    if (lane < ng) {
        const uint4 w = drop_words(d, k, row, (uint32_t)lane);
        nib0 = drop_keep(d, w.x) | drop_keep(d, w.y) << 1 | drop_keep(d, w.z) << 2 | drop_keep(d, w.w) << 3;
    }
    if (32 + lane < ng) {
        const uint4 w = drop_words(d, k, row, (uint32_t)(32 + lane));
        nib1 = drop_keep(d, w.x) | drop_keep(d, w.y) << 1 | drop_keep(d, w.z) << 2 | drop_keep(d, w.w) << 3;
    }
    uint32_t bits = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {                       // column lane + 32 i is in group 8 i + lane / 4, word lane % 4
        const uint32_t nib = __shfl_sync(B2R_FULL_MASK, i < 4 ? nib0 : nib1, (8 * i + (lane >> 2)) & 31);
        bits |= ((nib >> (lane & 3)) & 1u) << i;
    }
    return bits;
}

__device__ __forceinline__ float drop_apply_bit(const DropK& d, uint32_t bits, int i, float v) {
    return (bits >> i) & 1u ? v * d.scale : 0.f;
}

__device__ __forceinline__ float4 drop_apply4(const DropK& d, const uint4& w, const float4& v) {
    return make_float4(drop_apply(d, w.x, v.x), drop_apply(d, w.y, v.y), drop_apply(d, w.z, v.z), drop_apply(d, w.w, v.w));
}

}  // namespace b2r
