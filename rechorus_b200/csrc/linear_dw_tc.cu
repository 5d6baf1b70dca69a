// linear_dw_tc.cu -- the weight gradient of nn.Linear on the Hopper tensor cores (wgmma.mma_async, TF32 operands, fp32
// accumulator in registers): dW[n, k] = sum_m dY[m, n] * X[m, k], dbias[n] = sum_m dY[m, n], the autograd of
// utils/layers.py:26-28,106-107 and NeuMF.py:70 behind loss.backward() (helpers/BaseRunner.py:205).
//
// In a SASRec step the weight gradients are contractions over M = B*L rows (hundreds of thousands) with a small result
// (64 x 64), which on the CUDA cores cost more than the attention.  As a tensor-core problem they are an outer-product
// accumulation: D[64 x NB] += A[64 x 8] * B[NB x 8]^T per 8 batch rows, where A's rows are output features n (warpgroup g
// owns features 64 g .. 64 g + 63; rows >= N stay zero), B's rows the K input features plus one row of ones (its column of
// D is dbias) and zero rows up to the wgmma width NB, and the MMA's reduction dimension is the batch-row index m.  The
// operands are therefore the TRANSPOSES of the row-major activations; they are transposed on the way into shared memory
// (each lane owns one batch row of a 32-row slab and writes its elements down a column of the K-major SWIZZLE_128B tile:
// 32 lanes, 32 distinct banks), split x = hi + lo (both TF32-exact) as in linear_tc.cu, and four products hi*hi + hi*lo +
// lo*hi + lo*lo accumulate in registers across the CTA's whole row range.  Each CTA writes one partial [N x (K+1)] tile;
// a second kernel adds the CTAs' partials in CTA order (fixed order -> deterministic).
#include "common.cuh"
#include "wgmma_tf32.cuh"
#include "dropout.cuh"

namespace b2r {

constexpr int DW_SLABS = 2;          // 32-row slabs staged per iteration
constexpr int DW_MAX_WG = 2;         // warpgroups per CTA (N <= 128)
constexpr int DW_MAX_CTAS_PER_SM = 4;

__device__ __forceinline__ float dw_rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// element (feature row `row`, reduction column `col` in [0, 32)) of a 128-byte-row swizzled slab
__device__ __forceinline__ uint32_t dw_off(int row, int col) {
    return (uint32_t)row * 128u + (uint32_t)((((col >> 2) ^ (row & 7)) << 4) + ((col & 3) << 2));
}

// blockDim.x = 128 * ceil(N / 64); dynamic shared memory (1024-byte aligned):
// A_hi[SLABS][64 WG rows * 128B] A_lo[...] B_hi[SLABS][NB * 128B] B_lo[...]
template <int NB>
__global__ void __launch_bounds__(128 * DW_MAX_WG)
k_linear_dw_tc(const float* __restrict__ dY, int lddy, const float* __restrict__ relu_out, const float* __restrict__ X,
               int ldx, float* __restrict__ part, int M, int N, int K, int rows_per_cta) {
    extern __shared__ __align__(1024) unsigned char dw_raw[];
    const int nwg = blockDim.x / 128, nwarps = blockDim.x / 32;
    const size_t a_slab = (size_t)nwg * 64 * 128, b_slab = (size_t)NB * 128;
    char* A_hi = reinterpret_cast<char*>(dw_raw) + ((1024u - (wg_smem_u32(dw_raw) & 1023u)) & 1023u);
    char* A_lo = A_hi + DW_SLABS * a_slab;
    char* B_hi = A_lo + DW_SLABS * a_slab;
    char* B_lo = B_hi + DW_SLABS * b_slab;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;

    // zero every operand tile once: A's rows N.., B's rows K+1.. and the lo half of the ones row never change
    {
        const size_t total16 = (2 * DW_SLABS * (a_slab + b_slab)) / 16;
        float4* z = reinterpret_cast<float4*>(A_hi);
        for (size_t i = tid; i < total16; i += blockDim.x) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    // the row of ones (hi = 1, lo = 0): row K of B.  Batch rows beyond the range have dY = 0 and add nothing to dbias.
    for (int e = tid; e < DW_SLABS * 32; e += blockDim.x)
        *reinterpret_cast<float*>(B_hi + (e / 32) * b_slab + dw_off(K, e % 32)) = 1.f;

    float acc[NB / 2];
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) acc[i] = 0.f;
    const int m_begin = blockIdx.x * rows_per_cta;
    const int m_end = min(M, m_begin + rows_per_cta);
    // staging jobs: (dY | X) x slab; the warps of one job split its features in groups of 32
    const int job = warp % (2 * DW_SLABS), jpart = warp / (2 * DW_SLABS), jparts = nwarps / (2 * DW_SLABS);
    const bool isA = job < DW_SLABS;
    const int slab = job % DW_SLABS;
    const int nf = isA ? N : K;
    char* hi = isA ? A_hi + slab * a_slab : B_hi + slab * b_slab;
    char* lo = isA ? A_lo + slab * a_slab : B_lo + slab * b_slab;
    for (int m0 = m_begin; m0 < m_end; m0 += DW_SLABS * 32) {
        __syncthreads();                   // every warp's MMAs of the previous iteration completed before the tiles change
        {
            const int m = m0 + slab * 32 + lane;
            const bool live = m < m_end;
            const float* src = isA ? dY + (size_t)m * lddy : X + (size_t)m * ldx;
            const float* msk = (isA && relu_out != nullptr) ? relu_out + (size_t)m * lddy : nullptr;
            // 8 x 128-bit loads (32 features) of the lane's batch row in flight before the first use
            for (int f0 = jpart * 32; f0 < nf; f0 += jparts * 32) {
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (live && f0 + 4 * u < nf) v[u] = ld4(src + f0 + 4 * u);
                }
                if (msk != nullptr) {                                // ReLU backward: dY counts where the saved output > 0
                    float4 mk[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        mk[u] = make_float4(1.f, 1.f, 1.f, 1.f);
                        if (live && f0 + 4 * u < nf) mk[u] = ld4(msk + f0 + 4 * u);
                    }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        v[u].x = mk[u].x > 0.f ? v[u].x : 0.f;
                        v[u].y = mk[u].y > 0.f ? v[u].y : 0.f;
                        v[u].z = mk[u].z > 0.f ? v[u].z : 0.f;
                        v[u].w = mk[u].w > 0.f ? v[u].w : 0.f;
                    }
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    if (f0 + 4 * u < nf) {
                        const float pv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float h = dw_rn_tf32(pv[i]);
                            const uint32_t off = dw_off(f0 + 4 * u + i, lane);
                            *reinterpret_cast<float*>(hi + off) = h;
                            *reinterpret_cast<float*>(lo + off) = dw_rn_tf32(pv[i] - h);
                        }
                    }
                }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> async proxy (wgmma)
        __syncthreads();
        wg_fence();
#pragma unroll
        for (int prod = 0; prod < 4; ++prod) {
            const char* Ab = ((prod < 2) ? A_hi : A_lo) + (size_t)wg * 64 * 128;   // hi*hi, hi*lo, lo*hi, lo*lo
            const char* Bb = (prod & 1) ? B_lo : B_hi;
#pragma unroll
            for (int s = 0; s < DW_SLABS; ++s) {
#pragma unroll
                for (int k = 0; k < 4; ++k)                    // 4 MMAs of 8 batch rows (32 bytes) per slab
                    wgmma_tf32<NB>(acc, wg_desc(wg_smem_u32(Ab + s * a_slab) + k * 32),
                                   wg_desc(wg_smem_u32(Bb + s * b_slab) + k * 32), 1);
            }
        }
        wg_commit();
        wg_wait_all();
        wg_fence_regs(acc);
    }
    // epilogue from the fragment: feature row n, column c of [dW | dbias]
    float* out = part + (size_t)blockIdx.x * N * (K + 1);
    const int n0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int n = n0 + 8 * h, col = 8 * j + 2 * (lane & 3) + c;
                if (n < N && col <= K) out[(size_t)n * (K + 1) + col] = acc[4 * j + 2 * h + c];   // 0 for an empty range
            }
        }
    }
}

// dW[n, k] = sum_c part[c][n][k], dbias[n] = sum_c part[c][n][K]  (c ascending); SCALED: times `scale` (the 1 / (1 - p)
// of a dropout after the layer)
template <bool SCALED = false>
__global__ void __launch_bounds__(256)
k_linear_dw_reduce(const float* __restrict__ part, int ctas, int N, int K, float* __restrict__ dW, float* __restrict__ dbias,
                   float scale) {
    // 8 lanes per output element: lane l adds CTAs l, l+8, ... (ascending), then a fixed shuffle tree -> deterministic
    const int total = N * (K + 1);
    const int cl = threadIdx.x & 7;
    const int span = ((total + 31) / 32) * 32;
    for (int i = blockIdx.x * 32 + (threadIdx.x >> 3); i < span; i += gridDim.x * 32) {
        float a = 0.f;
        if (i < total)
            for (int c = cl; c < ctas; c += 8) a += part[(size_t)c * total + i];
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 1);
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 2);
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 4);
        if constexpr (SCALED) a *= scale;
        if (cl == 0 && i < total) {
            const int n = i / (K + 1), k = i % (K + 1);
            if (k < K) dW[(size_t)n * K + k] = a;
            else if (dbias != nullptr) dbias[n] = a;
        }
    }
}

template <int NB>
static int launch_linear_dw_tc(const float* dY, int lddy, const float* relu_out, const float* X, int ldx, float* dW,
                               float* dbias, int M, int N, int K, float* part, const float* scale, cudaStream_t s) {
    const int nwg = (N + 63) / 64;
    const size_t smem = (size_t)2 * DW_SLABS * nwg * 64 * 128 + (size_t)2 * DW_SLABS * NB * 128 + 1024;
    B2R_CUDA_OK(cudaFuncSetAttribute(k_linear_dw_tc<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2R_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_linear_dw_tc<NB>, 128 * nwg, smem));
    if (per_sm > DW_MAX_CTAS_PER_SM) per_sm = DW_MAX_CTAS_PER_SM;
    if (per_sm < 1) per_sm = 1;
    const int64_t slabs = ((int64_t)M + DW_SLABS * 32 - 1) / (DW_SLABS * 32);
    int ctas = sm_count() * per_sm;
    if (ctas > slabs) ctas = (int)slabs;
    const int rows_per_cta = (int)((slabs + ctas - 1) / ctas) * DW_SLABS * 32;
    k_linear_dw_tc<NB><<<ctas, 128 * nwg, smem, s>>>(dY, lddy, relu_out, X, ldx, part, M, N, K, rows_per_cta);
    B2R_LAUNCH_OK("k_linear_dw_tc");
    const int total = N * (K + 1);
    if (scale != nullptr) k_linear_dw_reduce<true><<<(total + 31) / 32, 256, 0, s>>>(part, ctas, N, K, dW, dbias, *scale);
    else k_linear_dw_reduce<<<(total + 31) / 32, 256, 0, s>>>(part, ctas, N, K, dW, dbias, 1.f);
    B2R_LAUNCH_OK("k_linear_dw_reduce");
    return 0;
}

static int linear_bwd_weight_tc(const float* dY, int lddy, const float* relu_out, const float* X, int ldx, float* dW,
                                float* dbias, int64_t M, int N, int K, void* ws, size_t ws_bytes, const float* scale,
                                cudaStream_t s) {
    B2R_REQUIRE(dY && X && dW && ws, B2R_E_BADARG, "b2r_linear_bwd_weight_tc: null pointer");
    if (!(N % 4 == 0 && N >= 4 && N <= 64 * DW_MAX_WG && K % 16 == 0 && K >= 16 && K <= 240 && M > 0 &&
          M <= 0x7fffffff && lddy % 4 == 0 && ldx % 4 == 0 && lddy >= N && ldx >= K && aligned16(dY) && aligned16(X) &&
          (relu_out == nullptr || aligned16(relu_out))))
        return set_error(B2R_E_UNSUPPORTED, "b2r_linear_bwd_weight_tc: shape M=%lld N=%d K=%d outside the kernel's class",
                         (long long)M, N, K);
    B2R_REQUIRE(ws_bytes >= b2r_linear_bwd_weight_tc_workspace_bytes(M, N, K), B2R_E_WORKSPACE,
                "b2r_linear_bwd_weight_tc: workspace too small");
    float* part = static_cast<float*>(ws);
    // wgmma width: K features + the ones row, rounded up to the instantiated widths
    if (K + 1 <= 48) return launch_linear_dw_tc<48>(dY, lddy, relu_out, X, ldx, dW, dbias, (int)M, N, K, part, scale, s);
    if (K + 1 <= 80) return launch_linear_dw_tc<80>(dY, lddy, relu_out, X, ldx, dW, dbias, (int)M, N, K, part, scale, s);
    return launch_linear_dw_tc<256>(dY, lddy, relu_out, X, ldx, dW, dbias, (int)M, N, K, part, scale, s);
}

}  // namespace b2r

using namespace b2r;

extern "C" size_t b2r_linear_bwd_weight_tc_workspace_bytes(int64_t M, int N, int K) {
    if (M <= 0 || N <= 0 || K <= 0) return 0;
    // one partial tile per CTA, at most DW_MAX_CTAS_PER_SM CTAs per SM
    return align_up((size_t)DW_MAX_CTAS_PER_SM * sm_count() * N * (K + 1) * 4, 256);
}

// returns B2R_E_UNSUPPORTED for shapes outside the tensor-core kernel's class (callers fall back to b2r_linear_bwd_weight)
extern "C" int b2r_linear_bwd_weight_tc(const float* dY, int lddy, const float* relu_out, const float* X, int ldx, float* dW,
                                        float* dbias, int64_t M, int N, int K, void* ws, size_t ws_bytes,
                                        b2r_stream_t stream) {
    return linear_bwd_weight_tc(dY, lddy, relu_out, X, ldx, dW, dbias, M, N, K, ws, ws_bytes, nullptr, as_stream(stream));
}

extern "C" int b2r_linear_bwd_weight_tc_dropout(const float* dY, int lddy, const float* relu_out, const float* X, int ldx,
                                                float* dW, float* dbias, int64_t M, int N, int K, const b2r_dropout* drop,
                                                void* ws, size_t ws_bytes, b2r_stream_t stream) {
    const int rc = check_dropout(drop, "b2r_linear_bwd_weight_tc_dropout");
    if (rc != 0) return rc;
    const float scale = dropout_scale(drop->p);
    return linear_bwd_weight_tc(dY, lddy, relu_out, X, ldx, dW, dbias, M, N, K, ws, ws_bytes, &scale, as_stream(stream));
}
