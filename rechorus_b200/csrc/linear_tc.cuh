// linear_tc.cuh -- the pieces of the tensor-core Linear forward that fix its bits: the TF32 hi/lo operand split, the
// swizzled shared-memory store of the split halves and the 3-product wgmma loop.  Shared by linear_tc.cu's k_linear_tc
// and neumf_all.cu's fused NeuMF scorer, so that a 64-row tile holding the same rows gives the same bits in both
// (the scorer's bit-identity with NeuMF's forward rests on it), as rank_tile.cuh is shared by eval.cu and topk.cu.
#pragma once
#include "common.cuh"
#include "wgmma_tf32.cuh"

namespace b2r {

constexpr int TC_M = 64;           // rows per tile == wgmma M
constexpr int TC_THREADS = 128;    // one warpgroup
constexpr int64_t kTcMinRows = 4096;   // the Linear forward takes the tensor cores from this many rows on

// round to the nearest TF32 value (10 explicit mantissa bits): the tensor core ignores the low 13 bits of what it is
// given, so operands are pre-rounded here and arrive exactly representable
__device__ __forceinline__ float tc_rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// hi = rn_tf32(x), lo = rn_tf32(x - hi)  (|x - hi - lo| <= 2^-23 |x|)
__device__ __forceinline__ void tc_split(float x, float& hi, float& lo) {
    hi = tc_rn_tf32(x);
    lo = tc_rn_tf32(x - hi);
}

// byte offset of (row, 16-byte chunk) in a K-major SWIZZLE_128B slab (wgmma_tf32.cuh)
__device__ __forceinline__ uint32_t tc_swz(int row, int chunk) {
    return (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) * 16);
}

// split 4 floats and store both halves at the swizzled chunk position
__device__ __forceinline__ void tc_store_split(char* hi_base, char* lo_base, int row, int chunk, const float4& v) {
    const uint32_t off = tc_swz(row, chunk);
    float4 h, l;
    tc_split(v.x, h.x, l.x); tc_split(v.y, h.y, l.y); tc_split(v.z, h.z, l.z); tc_split(v.w, h.w, l.w);
    *reinterpret_cast<float4*>(hi_base + off) = h;
    *reinterpret_cast<float4*>(lo_base + off) = l;
}

// acc[64 x NW] = A[64 x K] B[NW x K]^T with K = 32 KS, both operands given as hi/lo tiles of KS 128-byte slabs
// (A slabs 64 * 128 bytes apart, B slabs NW * 128): hi*hi, then hi*lo, then lo*hi, each over the slabs in ascending
// order and 4 MMAs of K = 8 per slab, the first one overwriting acc.  Issues the MMAs only: the caller commits and waits.
template <int KS, int NW>
__device__ __forceinline__ void tc_mma_3x(float (&acc)[NW / 2], const char* A_hi, const char* A_lo, const char* B_hi,
                                          const char* B_lo) {
    constexpr size_t a_slab = (size_t)TC_M * 128, b_slab = (size_t)NW * 128;
#pragma unroll
    for (int prod = 0; prod < 3; ++prod) {                  // hi*hi, hi*lo, lo*hi
        const char* Ab = (prod < 2) ? A_hi : A_lo;
        const char* Bb = (prod & 1) ? B_lo : B_hi;
#pragma unroll
        for (int s = 0; s < KS; ++s) {
#pragma unroll
            for (int k = 0; k < 4; ++k)                     // 4 MMAs of K = 8 floats (32 bytes) per slab
                wgmma_tf32<NW>(acc, wg_desc(wg_smem_u32(Ab + s * a_slab) + k * 32),
                               wg_desc(wg_smem_u32(Bb + s * b_slab) + k * 32), (prod | s | k) != 0);
        }
    }
}

// the wgmma width k_linear_tc uses for N output columns (W's rows N..NW-1 are zero)
static inline int tc_width(int N) { return N <= 16 ? 16 : N <= 32 ? 32 : N <= 64 ? 64 : N <= 128 ? 128 : 256; }

// whether k_linear_tc computes Y[M, N] = X[M, K] W^T (pointer alignment and leading dimensions aside): K % 32 == 0 and
// K <= 128, N % 16 == 0 and N <= 256, but not N > 128 with K > 64, whose W tiles alone would take 2 K 256 4 bytes of
// shared memory (linear_tc.cu)
bool linear_tc_shape(int64_t M, int N, int K);

}  // namespace b2r
