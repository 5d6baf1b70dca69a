// linear_tc.cu -- nn.Linear forward on the Hopper tensor cores (wgmma.mma_async, TF32 operands, fp32 accumulator in
// registers) with fp32-class accuracy: every operand is split x = hi + lo (hi = x rounded to TF32, lo = the TF32 rounding of
// the remainder) and three products hi*hi + hi*lo + lo*hi are accumulated in the same registers, which brings the result to
// ~2^-21 relative of the fp32 answer (the 1e-5 parity bar rules out a single TF32 product at trained-scale weights,
// SURVEY.md 7.3.4).
//
// Shape class: the q/k/v and feed-forward Linear layers of utils/layers.py:26-28,106-107 and NeuMF's tower
// (NeuMF.py:70): Y[M,N] = act(X[M,K] W^T + b) with small K (multiple of 32 floats, <= 128) and N (multiple of 16,
// <= 256) and M = B*L in the hundreds of thousands -- each CTA (one warpgroup) owns 64-row tiles of X, W stays resident
// in shared memory for the CTA's lifetime, so the kernel streams X once and Y once (HBM-bound) while the MMAs ride along.
//
// Operand staging: threads load X / W with coalesced 128-bit loads, split hi/lo in registers and store both halves into
// shared memory in the K-major SWIZZLE_128B layout of wgmma_tf32.cuh, then fence.proxy.async + barrier, and the
// warpgroup issues 3 * (K / 8) wgmmas.  The loads of the CTA's next tile are issued before the MMA wait, so they stay in
// flight through the MMAs and the epilogue, which adds the bias, applies ReLU and stores Y straight from the accumulator.
#include "common.cuh"
#include "wgmma_tf32.cuh"

namespace b2r {

constexpr int TC_M = 64;           // rows per tile == wgmma M
constexpr int TC_THREADS = 128;    // one warpgroup

// round to the nearest TF32 value (10 explicit mantissa bits): the tensor core ignores the low 13 bits of what it is
// given, so operands are pre-rounded here and arrive exactly representable
__device__ __forceinline__ float tc_rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// split 4 floats into hi = rn_tf32(x) and lo = rn_tf32(x - hi)  (|x - hi - lo| <= 2^-23 |x|), store both at the
// swizzled chunk position
__device__ __forceinline__ void tc_store_split(char* hi_base, char* lo_base, int row, int chunk, const float4& v) {
    const uint32_t off = (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) * 16);
    float4 h, l;
    h.x = tc_rn_tf32(v.x); h.y = tc_rn_tf32(v.y); h.z = tc_rn_tf32(v.z); h.w = tc_rn_tf32(v.w);
    l.x = tc_rn_tf32(v.x - h.x); l.y = tc_rn_tf32(v.y - h.y); l.z = tc_rn_tf32(v.z - h.z); l.w = tc_rn_tf32(v.w - h.w);
    *reinterpret_cast<float4*>(hi_base + off) = h;
    *reinterpret_cast<float4*>(lo_base + off) = l;
}

// dynamic shared memory (1024-byte aligned): A_hi[KS][64*128B] A_lo[...] B_hi[KS][NW*128B] B_lo[...]; NW >= N is the
// wgmma width, W's rows N..NW-1 are zero and their output columns are not stored
template <int KS, int NW>
__global__ void __launch_bounds__(TC_THREADS)
k_linear_tc(const float* __restrict__ X, int ldx, const float* __restrict__ amask, const float* __restrict__ W,
            const float* __restrict__ bias, float* __restrict__ Y, int ldy, int M, int N, int relu) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr int K = KS * 32;                              // KS 128-byte K slabs
    constexpr int LPT = 8 * KS * TC_M / TC_THREADS;         // 16-byte loads per thread per tile
    constexpr size_t a_slab = (size_t)TC_M * 128, b_slab = (size_t)NW * 128;
    // swizzle-128B operand tiles need 1024-byte aligned bases: align by hand (the launch adds 1 KB of slack)
    char* A_hi = reinterpret_cast<char*>(smem_raw) + ((1024u - (wg_smem_u32(smem_raw) & 1023u)) & 1023u);
    char* A_lo = A_hi + KS * a_slab;
    char* B_hi = A_lo + KS * a_slab;
    char* B_lo = B_hi + KS * b_slab;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    // W -> B_hi / B_lo (once per CTA): element (n, slab s, chunk c) <- W[n*K + s*32 + c*4 ..]
    for (int e = tid; e < NW * KS * 8; e += TC_THREADS) {
        const int c = e % 8, s = (e / 8) % KS, n = e / (8 * KS);
        const float4 v = n < N ? *reinterpret_cast<const float4*>(W + (size_t)n * K + s * 32 + c * 4)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
        tc_store_split(B_hi + s * b_slab, B_lo + s * b_slab, n, c, v);
    }

    const int ntiles = (M + TC_M - 1) / TC_M;
    float4 v[LPT];
    auto issue_loads = [&](int tile) {
        const int m0 = tile * TC_M;
#pragma unroll
        for (int i = 0; i < LPT; ++i) {
            const int e = i * TC_THREADS + tid;
            const int c = e % 8, s = (e / 8) % KS, r = e / (8 * KS);
            v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m0 + r < M) {
                const size_t g = (size_t)(m0 + r) * ldx + s * 32 + c * 4;
                v[i] = ld_row4(X + g);
                if (amask != nullptr) {      // ReLU backward: keep dY where the saved output > 0
                    const float4 mk = ld_row4(amask + g);
                    v[i].x = mk.x > 0.f ? v[i].x : 0.f;
                    v[i].y = mk.y > 0.f ? v[i].y : 0.f;
                    v[i].z = mk.z > 0.f ? v[i].z : 0.f;
                    v[i].w = mk.w > 0.f ? v[i].w : 0.f;
                }
            }
        }
    };
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    int tile = blockIdx.x;
    if (tile < ntiles) issue_loads(tile);
    for (; tile < ntiles; tile += gridDim.x) {
        const int m0 = tile * TC_M;
        __syncthreads();                  // the previous tile's MMAs have completed in every warp before A is overwritten
#pragma unroll
        for (int i = 0; i < LPT; ++i) {
            const int e = i * TC_THREADS + tid;
            const int c = e % 8, s = (e / 8) % KS, r = e / (8 * KS);
            tc_store_split(A_hi + s * a_slab, A_lo + s * a_slab, r, c, v[i]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> async proxy (wgmma)
        __syncthreads();
        wg_fence();
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
        wg_commit();
        if (tile + (int)gridDim.x < ntiles) issue_loads(tile + (int)gridDim.x);
        wg_wait_all();
        wg_fence_regs(acc);
        // epilogue straight from the fragment: each quad of lanes writes 8 consecutive floats (one 32-byte sector) of a row
        const int r0 = m0 + warp * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < NW / 8; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            if (col >= N) continue;
            const float b0 = bias != nullptr ? __ldg(bias + col) : 0.f;
            const float b1 = bias != nullptr ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                if (row >= M) continue;
                float y0 = acc[4 * j + 2 * h] + b0, y1 = acc[4 * j + 2 * h + 1] + b1;
                if (relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
                *reinterpret_cast<float2*>(Y + (size_t)row * ldy + col) = make_float2(y0, y1);
            }
        }
    }
}

template <int KS, int NW>
static int launch_linear_tc(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                            int ldy, int M, int N, int relu, cudaStream_t s) {
    const size_t smem = (size_t)2 * KS * TC_M * 128 + (size_t)2 * KS * NW * 128 + 1024;
    static_assert((size_t)2 * KS * TC_M * 128 + (size_t)2 * KS * NW * 128 + 1024 <= 227 * 1024, "shared memory");
    B2R_CUDA_OK(cudaFuncSetAttribute(k_linear_tc<KS, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2R_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_linear_tc<KS, NW>, TC_THREADS, smem));
    const int ntiles = (M + TC_M - 1) / TC_M;
    int grid = sm_count() * (per_sm < 1 ? 1 : per_sm);
    if (grid > ntiles) grid = ntiles;
    k_linear_tc<KS, NW><<<grid, TC_THREADS, smem, s>>>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu);
    B2R_LAUNCH_OK("k_linear_tc");
    return 0;
}

template <int KS>
static int launch_linear_tc_ks(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                               int ldy, int M, int N, int relu, cudaStream_t s) {
    if (N <= 16) return launch_linear_tc<KS, 16>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, s);
    if (N <= 32) return launch_linear_tc<KS, 32>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, s);
    if (N <= 64) return launch_linear_tc<KS, 64>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, s);
    if (N <= 128) return launch_linear_tc<KS, 128>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, s);
    if constexpr (KS <= 2) return launch_linear_tc<KS, 256>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, s);
    // W's hi/lo tiles alone would take 2 * K * 256 * 4 bytes of shared memory
    return set_error(B2R_E_UNSUPPORTED, "b2r_linear_tc: N=%d with K=%d exceeds the shared memory of one CTA", N, KS * 32);
}

}  // namespace b2r

using namespace b2r;

// returns B2R_E_UNSUPPORTED for shapes outside the tensor-core kernel's class (callers fall back to b2r_linear_fwd)
extern "C" int b2r_linear_fwd_tc(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy, int64_t M,
                                 int N, int K, int relu, b2r_stream_t stream) {
    return b2r_linear_tc(X, ldx, nullptr, W, bias, Y, ldy, M, N, K, relu, stream);
}

extern "C" int b2r_linear_tc(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                             int ldy, int64_t M, int N, int K, int relu, b2r_stream_t stream) {
    B2R_REQUIRE(X && W && Y, B2R_E_BADARG, "b2r_linear_fwd_tc: null pointer");
    if (!(K % 32 == 0 && K >= 32 && K <= 128 && N % 16 == 0 && N >= 16 && N <= 256 && M > 0 && M <= 0x7fffffff &&
          ldx % 4 == 0 && ldy % 4 == 0 && aligned16(X) && aligned16(W) && aligned16(Y) &&
          (x_mask == nullptr || aligned16(x_mask))))
        return set_error(B2R_E_UNSUPPORTED, "b2r_linear_fwd_tc: shape M=%lld N=%d K=%d ldx=%d ldy=%d outside the kernel's class",
                         (long long)M, N, K, ldx, ldy);
    cudaStream_t s = as_stream(stream);
    switch (K / 32) {
        case 1: return launch_linear_tc_ks<1>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, s);
        case 2: return launch_linear_tc_ks<2>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, s);
        case 3: return launch_linear_tc_ks<3>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, s);
        default: return launch_linear_tc_ks<4>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, s);
    }
}
