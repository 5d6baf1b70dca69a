// sampler.cu -- SURVEY.md §8 row f3, batch production on the device (opt-in: --device_sampler / --device_batches):
// the per-epoch negative sampling of models/BaseModel.py:206-214 and the collate of models/BaseModel.py:192-203,135-152.
//
// Reference semantics: for every training row i (user u_i) and every j < K draw an item uniformly from [1, n_items)
// and redraw while it is in the user's training clicks -- the result is uniform over the user's non-clicked items,
// duplicates across j allowed.  The reference does this with NumPy's global Mersenne Twister in a Python loop, a
// stream that is sequential and data dependent, so it cannot be reproduced in parallel; this kernel keeps the
// distribution and gives up the stream (documented in DESIGN.md).  No rejection loop either: with the clicks as a
// sorted CSR row c[0..m) the allowed items are the "missing numbers" of that row, so one uniform r in [0, A),
// A = n_items - 1 - m, selects the (r+1)-th allowed item directly: p = first position with c[p] - 1 - p > r (binary
// search; c[p] - 1 - p allowed items lie below c[p]), item = r + 1 + p.  r = floor(x * A / 2^32) with x = word 0 of
// Philox4x32-10(counter = (lo32(i*K+j), hi32(i*K+j), 0, epoch), key = seed).  The same definition is restated in
// oracle.device_sampler_reference, so the GPU output is checked bit for bit.
#include "common.cuh"
#include "philox.cuh"

namespace b2r {

__global__ void __launch_bounds__(256)
k_sample_negatives(const int64_t* __restrict__ user_ids, int64_t N, int K, const int64_t* __restrict__ clicked_ptr,
                   const int64_t* __restrict__ clicked_items, int64_t n_users, int64_t n_items, uint32_t seed_lo,
                   uint32_t seed_hi, uint32_t epoch, int64_t* __restrict__ out, int32_t* __restrict__ err_flag) {
    const int64_t total = N * K;
    for (int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 256) {
        const int64_t i = idx / K;
        int64_t u = user_ids[i];
        if (u < 0 || u >= n_users) {
            if (err_flag) atomicAdd(err_flag, 1);
            u = 0;
        }
        const int64_t beg = clicked_ptr[u];
        const int64_t m = clicked_ptr[u + 1] - beg;
        const int64_t A = n_items - 1 - m;                 // allowed items
        if (A <= 0) {                                      // the user clicked the whole catalogue: nothing to draw
            if (err_flag) atomicAdd(err_flag, 1);
            out[idx] = 1;
            continue;
        }
        const uint32_t x = philox4x32_10((uint32_t)idx, (uint32_t)((uint64_t)idx >> 32), 0u, epoch, seed_lo, seed_hi).x;
        const int64_t r = (int64_t)(((uint64_t)x * (uint64_t)A) >> 32);
        int64_t lo = 0, hi = m;                            // p = first position with c[p] - 1 - p > r
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (clicked_items[beg + mid] - 1 - mid > r) hi = mid; else lo = mid + 1;
        }
        out[idx] = r + 1 + lo;
    }
}

// One training batch of a GeneralModel assembled on the device: what GeneralModel.Dataset._get_feed_dict
// (models/BaseModel.py:192-203) + collate_batch (:135-152) build on the host sample by sample.  Row t of the batch is
// training row perm[start + t] (perm NULL: identity): user_id[t] = users[row], item_id[t] = [items[row], neg[row, 0..K)].
__global__ void __launch_bounds__(256)
k_collate_general(const int64_t* __restrict__ users, const int64_t* __restrict__ items, const int64_t* __restrict__ neg,
                  const int64_t* __restrict__ perm, int64_t start, int Bn, int K, int64_t* __restrict__ out_uid,
                  int64_t* __restrict__ out_iid) {
    const int C = K + 1;
    const int64_t total = (int64_t)Bn * C;
    for (int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 256) {
        const int t = (int)(idx / C), c = (int)(idx - (int64_t)t * C);
        const int64_t row = perm ? perm[start + t] : start + t;
        if (c == 0) {
            out_uid[t] = users[row];
            out_iid[idx] = items[row];
        } else {
            out_iid[idx] = neg[row * K + (c - 1)];
        }
    }
}

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_collate_general(const int64_t* users, const int64_t* items, const int64_t* neg, const int64_t* perm,
                                   int64_t start, int Bn, int K, int64_t* out_uid, int64_t* out_iid, b2r_stream_t stream) {
    B2R_REQUIRE(users && items && neg && out_uid && out_iid, B2R_E_BADARG, "b2r_collate_general: null pointer");
    B2R_REQUIRE(Bn >= 0 && K >= 1 && start >= 0, B2R_E_BADARG, "b2r_collate_general: Bn=%d K=%d", Bn, K);
    if (Bn == 0) return 0;
    const int64_t total = (int64_t)Bn * (K + 1);
    int64_t grid = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    k_collate_general<<<(int)grid, 256, 0, as_stream(stream)>>>(users, items, neg, perm, start, Bn, K, out_uid, out_iid);
    B2R_LAUNCH_OK("k_collate_general");
    return 0;
}

extern "C" int b2r_sample_negatives(const int64_t* user_ids, int64_t N, int K, const int64_t* clicked_ptr,
                                    const int64_t* clicked_items, int64_t n_users, int64_t n_items, uint64_t seed,
                                    uint32_t epoch, int64_t* out, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(user_ids && clicked_ptr && out, B2R_E_BADARG, "b2r_sample_negatives: null pointer");
    B2R_REQUIRE(N >= 0 && K >= 1 && n_users > 0 && n_items >= 2 && n_items - 1 <= 0xffffffffLL, B2R_E_BADARG,
                "b2r_sample_negatives: bad sizes N=%lld K=%d n_items=%lld", (long long)N, K, (long long)n_items);
    if (N == 0) return 0;
    const int64_t total = N * K;
    int64_t grid = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    k_sample_negatives<<<(int)grid, 256, 0, as_stream(stream)>>>(user_ids, N, K, clicked_ptr, clicked_items, n_users,
                                                                 n_items, (uint32_t)seed, (uint32_t)(seed >> 32), epoch,
                                                                 out, err_flag);
    B2R_LAUNCH_OK("k_sample_negatives");
    return 0;
}
