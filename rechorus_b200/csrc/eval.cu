// eval.cu -- the evaluation half of the path (SURVEY.md §8 row f2): integer ranks of the ground-truth item computed
// on the device, so neither the [N, C] prediction matrix nor (for test_all) the [B, n_items] score matrix has to
// travel to the host or even exist.
//
//   k_gt_rank        rank[r] = #{c : pred[r,c] >= pred[r,0]}            helpers/BaseRunner.py:63
//   k_rank_hist      hist[min(rank, kmax+1)] += 1                        (HR@k / NDCG@k are sums over this histogram, :66-74)
//   k_target_score   s0[b] = <q_b, I[target_b]>, rank[b] = 1            column 0 of the test_all candidate list
//   k_rank_all       rank[b] += #{1 <= j < n_items : <q_b, I[j]> >= s0[b]}   BaseModel.py:194-198 (candidates =
//                    [target] + arange(1, n_items)) scored by BPRMF.py:42 / SASRec.py:81, as a register-blocked
//                    fp32 GEMM whose epilogue compares and counts instead of storing
//   k_rank_unmask    rank[b] -= 1 for every listed (b, j) with <q_b, I[j]> >= s0[b]   the clicked-item masking
//                    preds[rows, cols] = -inf of BaseRunner.py:244-251
//   k_rank_unmask_clicked  the same masking read from the clicked-item CSR (b2r_mask_clicked's): one warp per batch row
//                    walks users[b]'s slice, one lane scores one clicked item
//
// Every score on the test_all path is accumulated as s = fmaf(q_k, i_k, s) for k ascending -- in the GEMM tile, in
// k_target_score and in both unmask kernels alike -- so the same (b, j) always yields the same bits and the comparison
// against s0 is consistent between the three kernels.  Counts are integers: atomics do not affect determinism.
// The GEMM tile itself (rank_tile.cuh) is shared with topk.cu's b2r_topk_all_items.
#include "common.cuh"
#include "rank_tile.cuh"

namespace b2r {

constexpr int kRT = 128;          // threads per CTA of the small kernels

__global__ void __launch_bounds__(kRT)
k_gt_rank(const float* __restrict__ pred, int64_t N, int64_t C, int64_t ld, int64_t* __restrict__ rank) {
    __shared__ int warp_cnt[kRT / 32];
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    if (C <= 1024) {                               // one warp per row
        for (int64_t r = (int64_t)blockIdx.x * (kRT / 32) + warp; r < N; r += (int64_t)gridDim.x * (kRT / 32)) {
            const float* p = pred + r * ld;
            const float t = p[0];
            int cnt = 0;
            for (int64_t c = lane; c < C; c += 32) cnt += (p[c] >= t) ? 1 : 0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(B2R_FULL_MASK, cnt, o);
            if (lane == 0) rank[r] = cnt;
        }
    } else {                                       // one CTA per row (test_all predictions that were materialised)
        for (int64_t r = blockIdx.x; r < N; r += gridDim.x) {
            const float* p = pred + r * ld;
            const float t = p[0];
            int cnt = 0;
            for (int64_t c = threadIdx.x; c < C; c += kRT) cnt += (p[c] >= t) ? 1 : 0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(B2R_FULL_MASK, cnt, o);
            if (lane == 0) warp_cnt[warp] = cnt;
            __syncthreads();
            if (threadIdx.x == 0) {
                int tot = 0;
                for (int w = 0; w < kRT / 32; ++w) tot += warp_cnt[w];
                rank[r] = tot;
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(kRT)
k_rank_hist(const int64_t* __restrict__ rank, int64_t N, int kmax, unsigned long long* __restrict__ hist) {
    for (int64_t r = (int64_t)blockIdx.x * kRT + threadIdx.x; r < N; r += (int64_t)gridDim.x * kRT) {
        int64_t k = rank[r];
        if (k < 0) k = 0;
        if (k > kmax) k = (int64_t)kmax + 1;
        atomicAdd(hist + k, 1ULL);
    }
}

__global__ void __launch_bounds__(kRT)
k_target_score(const float* __restrict__ Q, int ldq, const float* __restrict__ I, const int64_t* __restrict__ target,
               int B, int64_t n_items, int d, float* __restrict__ s0, int64_t* __restrict__ rank,
               int32_t* __restrict__ err_flag) {
    const int b = blockIdx.x * kRT + threadIdx.x;
    if (b >= B) return;
    int64_t t = target[b];
    if (t < 0 || t >= n_items) {
        if (err_flag) atomicAdd(err_flag, 1);
        t = 0;
    }
    const float* q = Q + (int64_t)b * ldq;
    const float* it = I + t * d;
    float s = 0.f;
    for (int k = 0; k < d; ++k) s = fmaf(q[k], it[k], s);
    s0[b] = s;
    rank[b] = 1;                                   // the candidate list's column 0 is the target itself
}

__global__ void __launch_bounds__(kAT)
k_rank_all(const float* __restrict__ Q, int ldq, const float* __restrict__ I, const float* __restrict__ s0, int B,
           int64_t n_items, int d, unsigned long long* __restrict__ rank) {
    __shared__ float Qs[kTK][kTQ + 4];
    __shared__ float Is[kTK][kTI + 4];
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;        // tx -> items, ty -> queries
    const int q0 = blockIdx.y * kTQ;
    const int64_t j0 = (int64_t)blockIdx.x * kTI;
    float acc[8][8];
    rank_tile_accumulate(Q, ldq, I, B, n_items, d, q0, j0, Qs, Is, acc);
    // epilogue: compare against the target's score and count; item 0 is not a candidate (ids are 1-based)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int q = q0 + ty * 8 + i;
        const float t = q < B ? s0[q] : 0.f;
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int64_t item = j0 + tx * 8 + j;
            cnt += (item >= 1 && item < n_items && acc[i][j] >= t) ? 1 : 0;
        }
        // the 16 threads sharing this query are the 16 consecutive lanes of a half warp
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) cnt += __shfl_xor_sync(B2R_FULL_MASK, cnt, o);
        if (tx == 0 && q < B && cnt != 0) atomicAdd(rank + q, (unsigned long long)cnt);
    }
}

__global__ void __launch_bounds__(kRT)
k_rank_unmask(const float* __restrict__ Q, int ldq, const float* __restrict__ I, const float* __restrict__ s0,
              const int64_t* __restrict__ mask_row, const int64_t* __restrict__ mask_item, int64_t E, int B,
              int64_t n_items, int d, unsigned long long* __restrict__ rank, int32_t* __restrict__ err_flag) {
    for (int64_t e = (int64_t)blockIdx.x * kRT + threadIdx.x; e < E; e += (int64_t)gridDim.x * kRT) {
        const int64_t b = mask_row[e], j = mask_item[e];
        if (b < 0 || b >= B) {
            if (err_flag) atomicAdd(err_flag, 1);
            continue;
        }
        if (j < 1 || j >= n_items) continue;       // not a column of the candidate list
        const float* q = Q + b * ldq;
        const float* it = I + j * d;
        float s = 0.f;
        for (int k = 0; k < d; ++k) s = fmaf(q[k], it[k], s);
        if (s >= s0[b]) atomicAdd(rank + b, ~0ULL);  // -1
    }
}

// One warp per batch row.  Each clicked item is scored by ONE lane with the scalar fmaf chain of k_target_score (k
// ascending; the float4 loads only fetch four consecutive k at once), so its bits equal the GEMM tile's and s0's.  The
// CSR holds each item once per user, so the count equals k_rank_unmask's over the same (row, item) pairs.  The warp is
// the only writer of rank[b] here (k_rank_all has finished: same stream), so no atomic is needed.
__global__ void __launch_bounds__(kRT)
k_rank_unmask_clicked(const float* __restrict__ Q, int ldq, const float* __restrict__ I, const float* __restrict__ s0,
                      const int64_t* __restrict__ users, const int64_t* __restrict__ clicked_ptr,
                      const int64_t* __restrict__ clicked_items, int64_t n_users, int B, int64_t n_items, int d,
                      int64_t* __restrict__ rank, int32_t* __restrict__ err_flag) {
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    for (int64_t b = (int64_t)blockIdx.x * (kRT / 32) + warp; b < B; b += (int64_t)gridDim.x * (kRT / 32)) {
        const int64_t u = users[b];
        if (u < 0 || u >= n_users) {               // counted once; the row stays unmasked
            if (lane == 0 && err_flag) atomicAdd(err_flag, 1);
            continue;
        }
        const int64_t beg = clicked_ptr[u], end = clicked_ptr[u + 1];
        const float* q = Q + b * ldq;
        const float t = s0[b];
        int cnt = 0;
        for (int64_t e = beg + lane; e < end; e += 32) {
            const int64_t j = clicked_items[e];
            if (j < 1 || j >= n_items) continue;   // not a column of the candidate list
            const float* it = I + j * d;
            float s = 0.f;
            for (int k = 0; k < d; k += 4) {
                const float4 v = ld_row4(it + k);
                s = fmaf(q[k], v.x, s);
                s = fmaf(q[k + 1], v.y, s);
                s = fmaf(q[k + 2], v.z, s);
                s = fmaf(q[k + 3], v.w, s);
            }
            cnt += (s >= t) ? 1 : 0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(B2R_FULL_MASK, cnt, o);
        if (lane == 0 && cnt != 0) rank[b] -= cnt;
    }
}

}  // namespace b2r

using namespace b2r;

// s0 and the unmasked ranks: k_target_score, then k_rank_all over the whole catalogue
static int rank_all_unmasked(const float* Q, int ldq, const float* I, const int64_t* target, int B, int64_t n_items, int d,
                             float* s0, int64_t* rank, int32_t* err_flag, cudaStream_t s) {
    k_target_score<<<(B + kRT - 1) / kRT, kRT, 0, s>>>(Q, ldq, I, target, B, n_items, d, s0, rank, err_flag);
    B2R_LAUNCH_OK("k_target_score");
    const int64_t tiles_i = (n_items + kTI - 1) / kTI;
    B2R_REQUIRE(tiles_i <= 0x7fffffff && (B + kTQ - 1) / kTQ <= 65535, B2R_E_UNSUPPORTED, "b2r_rank_all_items: grid");
    dim3 grid((unsigned)tiles_i, (unsigned)((B + kTQ - 1) / kTQ));
    k_rank_all<<<grid, kAT, 0, s>>>(Q, ldq, I, s0, B, n_items, d, reinterpret_cast<unsigned long long*>(rank));
    B2R_LAUNCH_OK("k_rank_all");
    return 0;
}

extern "C" int b2r_gt_rank(const float* pred, int64_t N, int64_t C, int64_t ld, int64_t* rank, b2r_stream_t stream) {
    B2R_REQUIRE(pred && rank, B2R_E_BADARG, "b2r_gt_rank: null pointer");
    B2R_REQUIRE(N >= 0 && C >= 1 && ld >= C, B2R_E_BADARG, "b2r_gt_rank: bad shape N=%lld C=%lld ld=%lld", (long long)N,
                (long long)C, (long long)ld);
    if (N == 0) return 0;
    int64_t grid = C <= 1024 ? (N + kRT / 32 - 1) / (kRT / 32) : N;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    k_gt_rank<<<(int)grid, kRT, 0, as_stream(stream)>>>(pred, N, C, ld, rank);
    B2R_LAUNCH_OK("k_gt_rank");
    return 0;
}

extern "C" int b2r_rank_histogram(const int64_t* rank, int64_t N, int kmax, int64_t* hist, b2r_stream_t stream) {
    B2R_REQUIRE(rank && hist, B2R_E_BADARG, "b2r_rank_histogram: null pointer");
    B2R_REQUIRE(N >= 0 && kmax >= 1, B2R_E_BADARG, "b2r_rank_histogram: bad shape");
    cudaStream_t s = as_stream(stream);
    B2R_CUDA_OK(cudaMemsetAsync(hist, 0, sizeof(int64_t) * ((size_t)kmax + 2), s));
    if (N == 0) return 0;
    int64_t grid = (N + kRT - 1) / kRT;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    k_rank_hist<<<(int)grid, kRT, 0, s>>>(rank, N, kmax, reinterpret_cast<unsigned long long*>(hist));
    B2R_LAUNCH_OK("k_rank_hist");
    return 0;
}

extern "C" int b2r_rank_all_items(const float* Q, int ldq, const float* I, const int64_t* target, int B, int64_t n_items,
                                  int d, const int64_t* mask_row, const int64_t* mask_item, int64_t n_mask, float* s0,
                                  int64_t* rank, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(Q && I && target && s0 && rank, B2R_E_BADARG, "b2r_rank_all_items: null pointer");
    B2R_REQUIRE(B >= 0 && n_items >= 1 && d >= 1 && ldq >= d, B2R_E_BADARG, "b2r_rank_all_items: bad shape");
    B2R_REQUIRE(d % 4 == 0 && aligned16(I), B2R_E_UNSUPPORTED, "b2r_rank_all_items: d=%d must be a multiple of 4", d);
    B2R_REQUIRE(n_mask == 0 || (mask_row && mask_item), B2R_E_BADARG, "b2r_rank_all_items: mask arrays missing");
    if (B == 0) return 0;
    cudaStream_t s = as_stream(stream);
    const int rc = rank_all_unmasked(Q, ldq, I, target, B, n_items, d, s0, rank, err_flag, s);
    if (rc != 0) return rc;
    if (n_mask > 0) {
        int64_t g = (n_mask + kRT - 1) / kRT;
        const int64_t cap = (int64_t)sm_count() * 16;
        if (g > cap) g = cap;
        k_rank_unmask<<<(int)g, kRT, 0, s>>>(Q, ldq, I, s0, mask_row, mask_item, n_mask, B, n_items, d,
                                             reinterpret_cast<unsigned long long*>(rank), err_flag);
        B2R_LAUNCH_OK("k_rank_unmask");
    }
    return 0;
}

extern "C" int b2r_rank_all_items_clicked(const float* Q, int ldq, const float* I, int64_t n_items, int d,
                                          const int64_t* target, const int64_t* users, int B, const int64_t* clicked_ptr,
                                          const int64_t* clicked_items, int64_t n_users, float* s0, int64_t* rank,
                                          int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(Q && I && target && users && clicked_ptr && clicked_items && s0 && rank, B2R_E_BADARG,
                "b2r_rank_all_items_clicked: null pointer");
    B2R_REQUIRE(B >= 0 && n_items >= 1 && d >= 1 && ldq >= d && n_users >= 1, B2R_E_BADARG,
                "b2r_rank_all_items_clicked: bad shape");
    B2R_REQUIRE(d % 4 == 0 && aligned16(I), B2R_E_UNSUPPORTED, "b2r_rank_all_items_clicked: d=%d must be a multiple of 4",
                d);
    if (B == 0) return 0;
    cudaStream_t s = as_stream(stream);
    const int rc = rank_all_unmasked(Q, ldq, I, target, B, n_items, d, s0, rank, err_flag, s);
    if (rc != 0) return rc;
    int64_t g = (B + kRT / 32 - 1) / (kRT / 32);
    const int64_t cap = (int64_t)sm_count() * 16;
    if (g > cap) g = cap;
    k_rank_unmask_clicked<<<(int)g, kRT, 0, s>>>(Q, ldq, I, s0, users, clicked_ptr, clicked_items, n_users, B, n_items, d,
                                                 rank, err_flag);
    B2R_LAUNCH_OK("k_rank_unmask_clicked");
    return 0;
}
