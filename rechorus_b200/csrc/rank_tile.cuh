// rank_tile.cuh -- the register-blocked fp32 score tile shared by the test_all kernels (eval.cu's k_rank_all and
// topk.cu's k_score_chunk): acc[i][j] = <Q[q0 + ty*8 + i], I[j0 + tx*8 + j]>, accumulated s = fmaf(q_k, i_k, s) for k
// ascending, so both kernels produce the same bits for the same (query, item) as k_target_score's scalar loop.
#pragma once
#include "common.cuh"

namespace b2r {

// 128 queries x 128 items per CTA, 256 threads, 8 x 8 scores per thread, the reduction dimension in chunks of 16.
constexpr int kTQ = 128, kTI = 128, kTK = 16, kAT = 256;

__device__ __forceinline__ void rank_tile_accumulate(const float* __restrict__ Q, int ldq, const float* __restrict__ I,
                                                     int B, int64_t n_items, int d, int q0, int64_t j0,
                                                     float (&Qs)[kTK][kTQ + 4], float (&Is)[kTK][kTI + 4],
                                                     float (&acc)[8][8]) {
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;        // tx -> items, ty -> queries
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    // loader mapping: thread -> (row = tid % 128, 8 consecutive k of the 16-wide chunk): a warp stores 32 consecutive
    // columns of one shared-memory row (conflict-free) and reads one full 32-byte sector per lane
    const int lr = tid % kTQ, lk = (tid / kTQ) * 8;
    for (int k0 = 0; k0 < d; k0 += kTK) {
        {
            const int q = q0 + lr;
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = 0.f;
            if (q < B) {
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if (k0 + lk + i < d) v[i] = Q[(int64_t)q * ldq + k0 + lk + i];
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) Qs[lk + i][lr] = v[i];
        }
        {
            const int64_t j = j0 + lr;
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = 0.f;
            if (j < n_items) {
                if (k0 + lk + 8 <= d) {
                    const float4 a = ld_row4(I + j * d + k0 + lk);
                    const float4 c = ld_row4(I + j * d + k0 + lk + 4);
                    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
                    v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (k0 + lk + i < d) v[i] = I[j * d + k0 + lk + i];
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) Is[lk + i][lr] = v[i];
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kTK; ++kk) {
            // k beyond d contributes fmaf(0, 0, acc) == acc exactly, so a ragged last chunk does not change the bits
            const float4 a0 = *reinterpret_cast<const float4*>(&Qs[kk][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&Qs[kk][ty * 8 + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Is[kk][tx * 8]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Is[kk][tx * 8 + 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
}

}  // namespace b2r
