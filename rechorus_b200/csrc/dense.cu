// dense.cu -- fp32 building blocks for the dense parts of NeuMF (NeuMF.py:69-75) and SASRec
// (utils/layers.py:26-28,106-118): a register-tiled SGEMM with fused bias / ReLU / ReLU-mask epilogues in
// the three layouts a Linear layer needs (forward, dX, dW with a deterministic split over the batch
// dimension), residual + LayerNorm forward/backward, and fixed-order partial reductions.
//
// fp32 FMA on the CUDA cores keeps the 1e-5 parity bar of the north star; linear_tc.cu and linear_dw_tc.cu are the
// tensor-core (3xTF32 / 4xTF32 wgmma) versions for long batches.
#include "common.cuh"

namespace b2r {

constexpr int BM = 64, BN = 64, BK = 16, GT = 256;   // CTA tile 64x64, k-step 16, 256 threads x (4x4) outputs

// A_MODE 0: A is [M, Kr] row-major (reduce along the contiguous dim)   1: A is [Kr, M] row-major
// B_MODE 0: B is [N, Kr] row-major (a Linear weight)                   1: B is [Kr, N] row-major
// amask (A_MODE-shaped, same ld): A element is used only where amask > 0 (ReLU backward)
// ones_col: B has a virtual extra column N-1 == 1.0 (bias gradient rides along with dW)
// blockIdx.z splits the reduction range into chunks of kchunk; chunk z writes C + z * c_chunk_stride
template <int A_MODE, int B_MODE>
__global__ void __launch_bounds__(GT)
k_gemm(const float* __restrict__ A, int lda, const float* __restrict__ amask, const float* __restrict__ B, int ldb,
       float* __restrict__ C, int ldc, int M, int N, int Kr, int kchunk, int64_t c_chunk_stride,
       const float* __restrict__ bias, int relu, int ones_col) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int kbeg = blockIdx.z * kchunk;
    const int kend = min(Kr, kbeg + kchunk);
    const int n_real = ones_col ? N - 1 : N;       // columns of B that exist in memory
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = kbeg; k0 < kend; k0 += BK) {
        // ---- A tile -> As[k][m]
        if (A_MODE == 0) {
            const int r = tid / 4, kq = (tid % 4) * 4;            // 64 rows x 4 quads of k
            const int m = m0 + r;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int k = k0 + kq + i;
                float v = 0.f;
                if (m < M && k < kend) {
                    v = A[(int64_t)m * lda + k];
                    if (amask != nullptr && !(amask[(int64_t)m * lda + k] > 0.f)) v = 0.f;
                }
                As[kq + i][r] = v;
            }
        } else {
            const int kk = tid / 16, mq = (tid % 16) * 4;         // 16 k-rows x 16 quads of m
            const int k = k0 + kk;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int m = m0 + mq + i;
                float v = 0.f;
                if (m < M && k < kend) {
                    v = A[(int64_t)k * lda + m];
                    if (amask != nullptr && !(amask[(int64_t)k * lda + m] > 0.f)) v = 0.f;
                }
                As[kk][mq + i] = v;
            }
        }
        // ---- B tile -> Bs[k][n]
        if (B_MODE == 0) {
            const int r = tid / 4, kq = (tid % 4) * 4;
            const int n = n0 + r;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int k = k0 + kq + i;
                Bs[kq + i][r] = (n < n_real && k < kend) ? B[(int64_t)n * ldb + k] : 0.f;
            }
        } else {
            const int kk = tid / 16, nq = (tid % 16) * 4;
            const int k = k0 + kk;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int n = n0 + nq + i;
                float v = 0.f;
                if (k < kend) {
                    if (n < n_real) v = B[(int64_t)k * ldb + n];
                    else if (ones_col && n == n_real) v = 1.f;
                }
                Bs[kk][nq + i] = v;
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* Cz = C + (int64_t)blockIdx.z * c_chunk_stride;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j];
            if (bias != nullptr) v += bias[n];
            if (relu) v = fmaxf(v, 0.f);
            Cz[(int64_t)m * ldc + n] = v;
        }
    }
}

// out[i] = sum over chunks of part[c][i] in a fixed order: 8 lanes per output element each add chunks c, c+8, ...
// (ascending), then the 8 lane sums are combined by a fixed shuffle tree -> deterministic and 8x more parallel than
// one thread per element
__global__ void __launch_bounds__(256)
k_reduce_chunks(const float* __restrict__ part, int64_t size, int chunks, float* __restrict__ out0, int64_t n0,
                float* __restrict__ out1) {
    // element i of a [rows, cols+1]-shaped partial: column cols (the ones column) goes to out1 (bias grad)
    const int cl = threadIdx.x & 7;
    for (int64_t i = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3); i < ((size + 31) / 32) * 32; i += (int64_t)gridDim.x * 32) {
        float a = 0.f;
        if (i < size)
            for (int c = cl; c < chunks; c += 8) a += part[(int64_t)c * size + i];
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 1);
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 2);
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 4);
        if (cl == 0 && i < size) {
            if (out1 == nullptr) {
                out0[i] = a;
            } else {
                const int64_t cols1 = n0 + 1;               // n0 = real columns
                const int64_t r = i / cols1, cidx = i % cols1;
                if (cidx < n0) out0[r * n0 + cidx] = a;
                else out1[r] = a;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// y = LayerNorm(x + res) * gamma + beta  (utils/layers.py:113,117; eps 1e-5, biased variance), one warp per row
// saves mean / rstd for the backward
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_add_layernorm_fwd(const float* __restrict__ x, const float* __restrict__ res, const float* __restrict__ gamma,
                    const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ mean_out,
                    float* __restrict__ rstd_out, int64_t rows, int d, float eps) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * 8) {
        const float* xr = x + r * d;
        const float* rr = res + r * d;
        float s = 0.f;
        for (int k = lane; k < d; k += 32) s += xr[k] + rr[k];
        const float mu = warp_sum(s) / (float)d;
        float q = 0.f;
        for (int k = lane; k < d; k += 32) {
            const float z = xr[k] + rr[k] - mu;
            q = fmaf(z, z, q);
        }
        const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
        for (int k = lane; k < d; k += 32) y[r * d + k] = (xr[k] + rr[k] - mu) * rstd * gamma[k] + beta[k];
        if (lane == 0) {
            mean_out[r] = mu;
            rstd_out[r] = rstd;
        }
    }
}

// the same forward for d = 4 * LPR: one 128-bit load per operand per lane, 32 / LPR rows per warp pass
template <int LPR>
__global__ void __launch_bounds__(256)
k_add_layernorm_fwd_v(const float* __restrict__ x, const float* __restrict__ res, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ mean_out,
                      float* __restrict__ rstd_out, int64_t rows, float eps) {
    constexpr int d = 4 * LPR, RPW = 32 / LPR;
    const int lane = threadIdx.x & 31, sub = lane / LPR, cl = lane % LPR;
    const float4 gm = ld4(gamma + cl * 4), bt = ld4(beta + cl * 4);
    const float invd = 1.f / (float)d;
    for (int64_t r0 = ((int64_t)blockIdx.x * 8 + (threadIdx.x >> 5)) * RPW; r0 < rows; r0 += (int64_t)gridDim.x * 8 * RPW) {
        const int64_t r = r0 + sub;
        const bool valid = r < rows;
        const int64_t rr = valid ? r : rows - 1;
        const float4 a = ld_row4(x + rr * d + cl * 4), b = ld_row4(res + rr * d + cl * 4);
        float4 z = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        const float mu = group_sum<LPR>((z.x + z.y) + (z.z + z.w)) * invd;
        z.x -= mu; z.y -= mu; z.z -= mu; z.w -= mu;
        const float rstd = rsqrtf(group_sum<LPR>(dot4(z, z)) * invd + eps);
        if (valid) {
            st4(y + r * d + cl * 4, make_float4(fmaf(z.x * rstd, gm.x, bt.x), fmaf(z.y * rstd, gm.y, bt.y),
                                                fmaf(z.z * rstd, gm.z, bt.z), fmaf(z.w * rstd, gm.w, bt.w)));
            if (cl == 0) {
                mean_out[r] = mu;
                rstd_out[r] = rstd;
            }
        }
    }
}

// backward of y = LN(z), z = x + res: dz (same for x and res) per row; dgamma/dbeta as per-CTA partials
// xhat = (z - mean) * rstd is recomputed from y: xhat = (y - beta) / gamma would divide by gamma -> recompute from z
__global__ void __launch_bounds__(256)
k_add_layernorm_bwd(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ res,
                    const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                    float* __restrict__ dz, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta,
                    int64_t rows, int d, int64_t rows_per_cta) {
    // CTA c owns rows [c*rows_per_cta, ...): its 8 warps take rows round-robin; dgamma/dbeta partials are
    // accumulated per warp in registers (column k = lane, lane+32, ...; d <= 256) and combined in warp order.
    __shared__ float sg[8][256];
    __shared__ float sb[8][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float ag[8], ab[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) ag[i] = ab[i] = 0.f;
    const int64_t rbeg = (int64_t)blockIdx.x * rows_per_cta;
    const int64_t rend = min(rows, rbeg + rows_per_cta);
    for (int64_t r = rbeg + warp; r < rend; r += 8) {
        const float mu = mean[r], rs = rstd[r];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int k = lane + 32 * i;
            if (k < d) {
                const float xh = (x[r * d + k] + res[r * d + k] - mu) * rs;
                const float g = dy[r * d + k] * gamma[k];
                s1 += g;
                s2 = fmaf(g, xh, s2);
                ag[i] = fmaf(dy[r * d + k], xh, ag[i]);
                ab[i] += dy[r * d + k];
            }
        }
        s1 = warp_sum(s1) / (float)d;
        s2 = warp_sum(s2) / (float)d;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int k = lane + 32 * i;
            if (k < d) {
                const float xh = (x[r * d + k] + res[r * d + k] - mu) * rs;
                dz[r * d + k] = (dy[r * d + k] * gamma[k] - s1 - xh * s2) * rs;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int k = lane + 32 * i;
        if (k < 256) {
            sg[warp][k] = ag[i];
            sb[warp][k] = ab[i];
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < d; k += 256) {
        float g = 0.f, b = 0.f;
        for (int w = 0; w < 8; ++w) {
            g += sg[w][k];
            b += sb[w][k];
        }
        part_dgamma[(int64_t)blockIdx.x * d + k] = g;
        part_dbeta[(int64_t)blockIdx.x * d + k] = b;
    }
}

// the same backward for d = 4 * LPR (LPR = 8, 16, 32 lanes per row): 128-bit loads, every value read once and kept in
// registers between the two row passes, 32 / LPR rows per warp pass (the scalar kernel above reads 4 bytes per lane, holds one
// 256-byte row per warp in flight and re-reads its inputs for the second pass: 2.8x its HBM time at d = 64)
template <int LPR>
__global__ void __launch_bounds__(256)
k_add_layernorm_bwd_v(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ res,
                      const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                      float* __restrict__ dz, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta,
                      int64_t rows, int64_t rows_per_cta) {
    constexpr int d = 4 * LPR, RPW = 32 / LPR;
    __shared__ float sg[8][d];
    __shared__ float sb[8][d];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / LPR, cl = lane % LPR;
    const float4 gm = ld4(gamma + cl * 4);
    float4 ag = make_float4(0.f, 0.f, 0.f, 0.f), ab = ag;
    const int64_t rbeg = (int64_t)blockIdx.x * rows_per_cta;
    const int64_t rend = min(rows, rbeg + rows_per_cta);
    const float invd = 1.f / (float)d;
    for (int64_t r0 = rbeg + warp * RPW; r0 < rend; r0 += 8 * RPW) {
        const int64_t r = r0 + sub;
        const bool valid = r < rend;
        const int64_t rr = valid ? r : rend - 1;
        const float4 xv = ld_row4(x + rr * d + cl * 4), rv = ld_row4(res + rr * d + cl * 4), g = ld_row4(dy + rr * d + cl * 4);
        const float mu = mean[rr], rs = rstd[rr];
        const float4 xh = make_float4((xv.x + rv.x - mu) * rs, (xv.y + rv.y - mu) * rs, (xv.z + rv.z - mu) * rs, (xv.w + rv.w - mu) * rs);
        const float4 gg = make_float4(g.x * gm.x, g.y * gm.y, g.z * gm.z, g.w * gm.w);
        const float s1 = group_sum<LPR>((gg.x + gg.y) + (gg.z + gg.w)) * invd;
        const float s2 = group_sum<LPR>(dot4(gg, xh)) * invd;
        if (valid) {
            st4(dz + r * d + cl * 4, make_float4((gg.x - s1 - xh.x * s2) * rs, (gg.y - s1 - xh.y * s2) * rs,
                                                 (gg.z - s1 - xh.z * s2) * rs, (gg.w - s1 - xh.w * s2) * rs));
            ag.x = fmaf(g.x, xh.x, ag.x); ag.y = fmaf(g.y, xh.y, ag.y); ag.z = fmaf(g.z, xh.z, ag.z); ag.w = fmaf(g.w, xh.w, ag.w);
            ab.x += g.x; ab.y += g.y; ab.z += g.z; ab.w += g.w;
        }
    }
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {                      // the warp's row slots, fixed order
        ag.x += __shfl_xor_sync(B2R_FULL_MASK, ag.x, o); ag.y += __shfl_xor_sync(B2R_FULL_MASK, ag.y, o);
        ag.z += __shfl_xor_sync(B2R_FULL_MASK, ag.z, o); ag.w += __shfl_xor_sync(B2R_FULL_MASK, ag.w, o);
        ab.x += __shfl_xor_sync(B2R_FULL_MASK, ab.x, o); ab.y += __shfl_xor_sync(B2R_FULL_MASK, ab.y, o);
        ab.z += __shfl_xor_sync(B2R_FULL_MASK, ab.z, o); ab.w += __shfl_xor_sync(B2R_FULL_MASK, ab.w, o);
    }
    if (sub == 0) {
        st4(&sg[warp][cl * 4], ag);
        st4(&sb[warp][cl * 4], ab);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < d; k += 256) {
        float g = 0.f, b = 0.f;
        for (int w = 0; w < 8; ++w) {
            g += sg[w][k];
            b += sb[w][k];
        }
        part_dgamma[(int64_t)blockIdx.x * d + k] = g;
        part_dbeta[(int64_t)blockIdx.x * d + k] = b;
    }
}

static int gemm_launch(int a_mode, int b_mode, const float* A, int lda, const float* amask, const float* B, int ldb,
                       float* C, int ldc, int M, int N, int Kr, int kchunk, int64_t cstride, const float* bias,
                       int relu, int ones_col, cudaStream_t s) {
    const int chunks = (Kr + kchunk - 1) / kchunk;
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, chunks);
    if (a_mode == 0 && b_mode == 0)
        k_gemm<0, 0><<<grid, GT, 0, s>>>(A, lda, amask, B, ldb, C, ldc, M, N, Kr, kchunk, cstride, bias, relu, ones_col);
    else if (a_mode == 0 && b_mode == 1)
        k_gemm<0, 1><<<grid, GT, 0, s>>>(A, lda, amask, B, ldb, C, ldc, M, N, Kr, kchunk, cstride, bias, relu, ones_col);
    else if (a_mode == 1 && b_mode == 1)
        k_gemm<1, 1><<<grid, GT, 0, s>>>(A, lda, amask, B, ldb, C, ldc, M, N, Kr, kchunk, cstride, bias, relu, ones_col);
    else
        return set_error(B2R_E_UNSUPPORTED, "gemm layout %d/%d", a_mode, b_mode);
    B2R_LAUNCH_OK("k_gemm");
    return 0;
}

constexpr int kDwChunk = 512;    // rows of the batch dimension per dW partial (>= 400 CTAs at B*L = 204,800)

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_linear_fwd(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy,
                              int64_t M, int N, int K, int relu, b2r_stream_t stream) {
    B2R_REQUIRE(X && W && Y, B2R_E_BADARG, "b2r_linear_fwd: null pointer");
    B2R_REQUIRE(M >= 0 && M <= 0x7fffffff && N > 0 && K > 0 && ldx >= K && ldy >= N, B2R_E_BADARG,
                "b2r_linear_fwd: bad shape M=%lld N=%d K=%d ldx=%d ldy=%d", (long long)M, N, K, ldx, ldy);
    if (M == 0) return 0;
    return gemm_launch(0, 0, X, ldx, nullptr, W, K, Y, ldy, (int)M, N, K, K, 0, bias, relu, 0, as_stream(stream));
}

extern "C" int b2r_linear_bwd_input(const float* dY, int lddy, const float* relu_out, const float* W, float* dX,
                                    int lddx, int64_t M, int N, int K, b2r_stream_t stream) {
    B2R_REQUIRE(dY && W && dX, B2R_E_BADARG, "b2r_linear_bwd_input: null pointer");
    B2R_REQUIRE(M >= 0 && M <= 0x7fffffff && N > 0 && K > 0 && lddy >= N && lddx >= K, B2R_E_BADARG,
                "b2r_linear_bwd_input: bad shape");
    if (M == 0) return 0;
    // dX[M,K] = (dY * [relu_out > 0]) [M,N] x W[N,K]
    return gemm_launch(0, 1, dY, lddy, relu_out, W, K, dX, lddx, (int)M, K, N, N, 0, nullptr, 0, 0, as_stream(stream));
}

extern "C" size_t b2r_linear_bwd_weight_workspace_bytes(int64_t M, int N, int K) {
    if (M <= 0 || N <= 0 || K <= 0) return 0;
    const int64_t chunks = (M + kDwChunk - 1) / kDwChunk;
    return (size_t)chunks * N * (K + 1) * sizeof(float);
}

extern "C" int b2r_linear_bwd_weight(const float* dY, int lddy, const float* relu_out, const float* X, int ldx,
                                     float* dW, float* dbias, int64_t M, int N, int K, void* ws, size_t ws_bytes,
                                     b2r_stream_t stream) {
    B2R_REQUIRE(dY && X && dW && ws, B2R_E_BADARG, "b2r_linear_bwd_weight: null pointer");
    B2R_REQUIRE(M > 0 && M <= 0x7fffffff && N > 0 && K > 0 && lddy >= N && ldx >= K, B2R_E_BADARG,
                "b2r_linear_bwd_weight: bad shape");
    B2R_REQUIRE(ws_bytes >= b2r_linear_bwd_weight_workspace_bytes(M, N, K), B2R_E_WORKSPACE,
                "b2r_linear_bwd_weight: workspace too small");
    cudaStream_t s = as_stream(stream);
    const int chunks = (int)((M + kDwChunk - 1) / kDwChunk);
    const int ones = dbias != nullptr ? 1 : 0;
    const int Kc = K + ones;
    float* part = static_cast<float*>(ws);
    // part[z][N][Kc] = sum_{m in chunk z} (dY*mask)[m,n] * [X | 1][m,k]
    int rc = gemm_launch(1, 1, dY, lddy, relu_out, X, ldx, part, Kc, N, Kc, (int)M, kDwChunk, (int64_t)N * Kc, nullptr,
                         0, ones, s);
    if (rc != 0) return rc;
    const int64_t size = (int64_t)N * Kc;
    k_reduce_chunks<<<(int)((size + 31) / 32), 256, 0, s>>>(part, size, chunks, dW, K, ones ? dbias : nullptr);
    B2R_LAUNCH_OK("k_reduce_chunks");
    return 0;
}

extern "C" int b2r_add_layernorm_fwd(const float* x, const float* res, const float* gamma, const float* beta,
                                     float* y, float* mean, float* rstd, int64_t rows, int d, float eps,
                                     b2r_stream_t stream) {
    B2R_REQUIRE(x && res && gamma && beta && y && mean && rstd, B2R_E_BADARG, "b2r_add_layernorm_fwd: null pointer");
    B2R_REQUIRE(rows >= 0 && d > 0, B2R_E_BADARG, "b2r_add_layernorm_fwd: bad shape");
    if (rows == 0) return 0;
    int64_t need = (rows + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 16;
    const int grid = (int)(need < cap ? need : cap);
    const bool vec = aligned16(x) && aligned16(res) && aligned16(y) && aligned16(gamma) && aligned16(beta);
    if (vec && d == 64) k_add_layernorm_fwd_v<16><<<grid, 256, 0, as_stream(stream)>>>(x, res, gamma, beta, y, mean, rstd, rows, eps);
    else if (vec && d == 128) k_add_layernorm_fwd_v<32><<<grid, 256, 0, as_stream(stream)>>>(x, res, gamma, beta, y, mean, rstd, rows, eps);
    else if (vec && d == 32) k_add_layernorm_fwd_v<8><<<grid, 256, 0, as_stream(stream)>>>(x, res, gamma, beta, y, mean, rstd, rows, eps);
    else k_add_layernorm_fwd<<<grid, 256, 0, as_stream(stream)>>>(x, res, gamma, beta, y, mean, rstd, rows, d, eps);
    B2R_LAUNCH_OK("k_add_layernorm_fwd");
    return 0;
}

static int ln_bwd_ctas(int64_t rows) {
    int64_t c = (rows + 255) / 256;           // >= 256 rows per CTA
    const int64_t cap = (int64_t)sm_count() * 4;
    if (c > cap) c = cap;
    return (int)(c < 1 ? 1 : c);
}

extern "C" size_t b2r_add_layernorm_bwd_workspace_bytes(int64_t rows, int d) {
    if (rows <= 0 || d <= 0) return 0;
    return (size_t)2 * ln_bwd_ctas(rows) * d * sizeof(float);
}

extern "C" int b2r_add_layernorm_bwd(const float* dy, const float* x, const float* res, const float* gamma,
                                     const float* mean, const float* rstd, float* dz, float* dgamma, float* dbeta,
                                     int64_t rows, int d, void* ws, size_t ws_bytes, b2r_stream_t stream) {
    B2R_REQUIRE(dy && x && res && gamma && mean && rstd && dz && dgamma && dbeta && ws, B2R_E_BADARG,
                "b2r_add_layernorm_bwd: null pointer");
    B2R_REQUIRE(rows > 0 && d > 0 && d <= 256, B2R_E_UNSUPPORTED, "b2r_add_layernorm_bwd: need 0 < d <= 256 (d=%d)", d);
    B2R_REQUIRE(ws_bytes >= b2r_add_layernorm_bwd_workspace_bytes(rows, d), B2R_E_WORKSPACE,
                "b2r_add_layernorm_bwd: workspace too small");
    cudaStream_t s = as_stream(stream);
    const int ctas = ln_bwd_ctas(rows);
    const int64_t rpc = (rows + ctas - 1) / ctas;
    float* pg = static_cast<float*>(ws);
    float* pb = pg + (size_t)ctas * d;
    const bool vec = aligned16(dy) && aligned16(x) && aligned16(res) && aligned16(dz) && aligned16(gamma);
    if (vec && d == 64) k_add_layernorm_bwd_v<16><<<ctas, 256, 0, s>>>(dy, x, res, gamma, mean, rstd, dz, pg, pb, rows, rpc);
    else if (vec && d == 128) k_add_layernorm_bwd_v<32><<<ctas, 256, 0, s>>>(dy, x, res, gamma, mean, rstd, dz, pg, pb, rows, rpc);
    else if (vec && d == 32) k_add_layernorm_bwd_v<8><<<ctas, 256, 0, s>>>(dy, x, res, gamma, mean, rstd, dz, pg, pb, rows, rpc);
    else k_add_layernorm_bwd<<<ctas, 256, 0, s>>>(dy, x, res, gamma, mean, rstd, dz, pg, pb, rows, d, rpc);
    B2R_LAUNCH_OK("k_add_layernorm_bwd");
    k_reduce_chunks<<<(d + 31) / 32, 256, 0, s>>>(pg, d, ctas, dgamma, 0, nullptr);
    B2R_LAUNCH_OK("k_reduce_chunks");
    k_reduce_chunks<<<(d + 31) / 32, 256, 0, s>>>(pb, d, ctas, dbeta, 0, nullptr);
    B2R_LAUNCH_OK("k_reduce_chunks");
    return 0;
}
