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
#include "linear_tc.cuh"
#include "dropout.cuh"

namespace b2r {

// dynamic shared memory (1024-byte aligned): A_hi[KS][64*128B] A_lo[...] B_hi[KS][NW*128B] B_lo[...]; NW >= N is the
// wgmma width, W's rows N..NW-1 are zero and their output columns are not stored.  DROP: dropout (dropout.cuh) after
// bias / ReLU in the epilogue, output row = activation row
template <int KS, int NW, bool DROP = false>
__global__ void __launch_bounds__(TC_THREADS)
k_linear_tc(const float* __restrict__ X, int ldx, const float* __restrict__ amask, const float* __restrict__ W,
            const float* __restrict__ bias, float* __restrict__ Y, int ldy, int M, int N, int relu, DropK dk) {
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
    DropKey key;
    if constexpr (DROP) key = drop_key(dk);
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
        tc_mma_3x<KS, NW>(acc, A_hi, A_lo, B_hi, B_lo);
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
            uint2 wd[2];                                        // DROP: mask words of (col, col + 1) in rows r0, r0 + 8
            if constexpr (DROP) {
                // lanes l and l ^ 1 hold the four columns of one group in the same two rows: the even lane draws row r0's
                // words, the odd lane row r0 + 8's, and each hands its partner the half the partner needs
                const int odd = lane & 1;
                const uint4 w = drop_words(dk, key, min(r0 + 8 * odd, M - 1), (uint32_t)col >> 2);
                const uint32_t g0 = __shfl_xor_sync(B2R_FULL_MASK, odd ? w.x : w.z, 1);
                const uint32_t g1 = __shfl_xor_sync(B2R_FULL_MASK, odd ? w.y : w.w, 1);
                wd[0] = odd ? make_uint2(g0, g1) : make_uint2(w.x, w.y);
                wd[1] = odd ? make_uint2(w.z, w.w) : make_uint2(g0, g1);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                if (row >= M) continue;
                float y0 = acc[4 * j + 2 * h] + b0, y1 = acc[4 * j + 2 * h + 1] + b1;
                if (relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
                if constexpr (DROP) {
                    y0 = drop_apply(dk, wd[h].x, y0);
                    y1 = drop_apply(dk, wd[h].y, y1);
                }
                *reinterpret_cast<float2*>(Y + (size_t)row * ldy + col) = make_float2(y0, y1);
            }
        }
    }
}

template <int KS, int NW, bool DROP>
static int launch_linear_tc(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                            int ldy, int M, int N, int relu, const DropK& dk, cudaStream_t s) {
    const size_t smem = (size_t)2 * KS * TC_M * 128 + (size_t)2 * KS * NW * 128 + 1024;
    static_assert((size_t)2 * KS * TC_M * 128 + (size_t)2 * KS * NW * 128 + 1024 <= 227 * 1024, "shared memory");
    B2R_CUDA_OK(cudaFuncSetAttribute(k_linear_tc<KS, NW, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2R_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_linear_tc<KS, NW, DROP>, TC_THREADS, smem));
    const int ntiles = (M + TC_M - 1) / TC_M;
    int grid = sm_count() * (per_sm < 1 ? 1 : per_sm);
    if (grid > ntiles) grid = ntiles;
    k_linear_tc<KS, NW, DROP><<<grid, TC_THREADS, smem, s>>>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, dk);
    B2R_LAUNCH_OK("k_linear_tc");
    return 0;
}

template <int KS, bool DROP>
static int launch_linear_tc_ks(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                               int ldy, int M, int N, int relu, const DropK& dk, cudaStream_t s) {
    if (N <= 16) return launch_linear_tc<KS, 16, DROP>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, dk, s);
    if (N <= 32) return launch_linear_tc<KS, 32, DROP>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, dk, s);
    if (N <= 64) return launch_linear_tc<KS, 64, DROP>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, dk, s);
    if (N <= 128) return launch_linear_tc<KS, 128, DROP>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, dk, s);
    if constexpr (KS <= 2) return launch_linear_tc<KS, 256, DROP>(X, ldx, x_mask, W, bias, Y, ldy, M, N, relu, dk, s);
    // W's hi/lo tiles alone would take 2 * K * 256 * 4 bytes of shared memory
    return set_error(B2R_E_UNSUPPORTED, "b2r_linear_tc: N=%d with K=%d exceeds the shared memory of one CTA", N, KS * 32);
}

bool linear_tc_shape(int64_t M, int N, int K) {
    return K % 32 == 0 && K >= 32 && K <= 128 && N % 16 == 0 && N >= 16 && N <= 256 && M > 0 && M <= 0x7fffffff &&
           !(N > 128 && K > 64);
}

template <bool DROP>
static int linear_tc(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y, int ldy,
                     int64_t M, int N, int K, int relu, const DropK& dk, cudaStream_t s) {
    B2R_REQUIRE(X && W && Y, B2R_E_BADARG, "b2r_linear_fwd_tc: null pointer");
    if (!(linear_tc_shape(M, N, K) && ldx % 4 == 0 && ldy % 4 == 0 && aligned16(X) && aligned16(W) && aligned16(Y) &&
          (x_mask == nullptr || aligned16(x_mask))))
        return set_error(B2R_E_UNSUPPORTED, "b2r_linear_fwd_tc: shape M=%lld N=%d K=%d ldx=%d ldy=%d outside the kernel's class",
                         (long long)M, N, K, ldx, ldy);
    switch (K / 32) {
        case 1: return launch_linear_tc_ks<1, DROP>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, dk, s);
        case 2: return launch_linear_tc_ks<2, DROP>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, dk, s);
        case 3: return launch_linear_tc_ks<3, DROP>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, dk, s);
        default: return launch_linear_tc_ks<4, DROP>(X, ldx, x_mask, W, bias, Y, ldy, (int)M, N, relu, dk, s);
    }
}

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_linear_fwd_uses_tc(int64_t M, int N, int K) {
    return M >= kTcMinRows && linear_tc_shape(M, N, K) ? 1 : 0;
}

// returns B2R_E_UNSUPPORTED for shapes outside the tensor-core kernel's class (callers fall back to b2r_linear_fwd)
extern "C" int b2r_linear_fwd_tc(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy, int64_t M,
                                 int N, int K, int relu, b2r_stream_t stream) {
    return b2r_linear_tc(X, ldx, nullptr, W, bias, Y, ldy, M, N, K, relu, stream);
}

extern "C" int b2r_linear_tc(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                             int ldy, int64_t M, int N, int K, int relu, b2r_stream_t stream) {
    return linear_tc<false>(X, ldx, x_mask, W, bias, Y, ldy, M, N, K, relu, DropK{}, as_stream(stream));
}

extern "C" int b2r_linear_fwd_tc_dropout(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy,
                                         int64_t M, int N, int K, int relu, const b2r_dropout* drop, b2r_stream_t stream) {
    const int rc = check_dropout(drop, "b2r_linear_fwd_tc_dropout");
    if (rc != 0) return rc;
    return linear_tc<true>(X, ldx, nullptr, W, bias, Y, ldy, M, N, K, relu, make_dropk(*drop), as_stream(stream));
}
