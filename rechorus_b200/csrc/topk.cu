// topk.cu -- the final top-k recommendation lists on the device (SURVEY.md §8 row a11 / f2): the TopK branch of
// main.py:117-132 (save_rec_results), which sorts every row of runner.predict's [N, C] matrix in Python and keeps the
// top 100.
//
//   k_mask_clicked      pred[b, j] = -inf for j in the user's clicked CSR slice, 1 <= j < C   BaseRunner.py:244-251
//   k_topk_scan         top-k of one column range of one row (scores or, when merging, keys of earlier passes)
//   k_topk_all_init     column 0 of the test_all list (the target, scored as k_target_score does) opens each row's list
//   k_score_chunk       rank_tile.cuh's GEMM tile, scores of one item chunk into the [B, W] chunk buffer
//   k_topk_all_merge    the chunk's masked scores merged into each row's running top-k list
//   k_topk_all_out      running lists -> item ids and scores
//
// Ordering (include/b200rec.h): Python's stable sorted(..., reverse=True) -- score descending, ties by column
// ascending -- as the ascending order of the 64-bit key (~mono(score) << 32) | column, -0.0 folded onto +0.0, NaN
// last.  Keys are unique within a row, so the result is one total order whatever the grid or the arrival order.
//
// Selection: a CTA keeps a shared-memory buffer of keys and a threshold (the current k-th key, or "accept all" while
// fewer than k are held).  Candidates below the threshold are appended; when the buffer could overflow in the next
// round it is bitonic-sorted, cut to k and the threshold tightened.  After the first few rounds almost nothing passes
// the threshold, so a range is read once at memory speed.
#include "common.cuh"
#include "rank_tile.cuh"

namespace b2r {

constexpr int kKT = 256;                  // threads per selection CTA
constexpr int kKTSmall = 32;              // b2r_topk_rows on rows of <= kSmallC columns: one warp per row
constexpr int64_t kSmallC = 1024;
constexpr int kEPT = 8;                   // candidates per thread per load round
constexpr int kMaxTopK = 1024;
constexpr int64_t kRangeMin = 4096;       // b2r_topk_rows: a row is split into ranges of at least this many columns,
constexpr int64_t kRangeCtas = 1024;      // into at most ceil(1024 / N) of them
constexpr size_t kChunkBytes = 32u << 20; // b2r_topk_all_items: the [B, W] score buffer of one item chunk
constexpr int kChunkMax = 8192;           // widest chunk (its mask bitmap lives in shared memory)
constexpr uint64_t kNoKey = ~0ull;

__host__ __device__ __forceinline__ int select_cap(int k) {      // buffer keys: room for k kept + one round
    int p = 1;
    while (p < k) p <<= 1;
    return 2 * p > 512 ? 2 * p : 512;
}

__device__ __forceinline__ uint64_t order_key(float s, uint32_t col) {
    uint32_t u = __float_as_uint(s);
    if (u == 0x80000000u) u = 0u;                                   // -0.0 == +0.0
    uint32_t hi;
    if ((u & 0x7fffffffu) > 0x7f800000u) {
        hi = 0xffffffffu;                                           // NaN: after -inf
    } else {
        const uint32_t mono = (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // ascending with the float
        hi = ~mono;                                                 // descending score first
    }
    return ((uint64_t)hi << 32) | col;
}

__device__ __forceinline__ float key_score(uint64_t key) {
    const uint32_t hi = (uint32_t)(key >> 32);
    if (hi == 0xffffffffu) return __uint_as_float(0x7fc00000u);
    const uint32_t mono = ~hi;
    return __uint_as_float((mono & 0x80000000u) ? (mono & 0x7fffffffu) : ~mono);
}

// Sort buf[0, *cnt) ascending (bitonic over the next power of two, padded with kNoKey), keep the first k and tighten the
// threshold.  Called by the whole CTA after a barrier; ends with one.
__device__ __forceinline__ void select_flush(uint64_t* buf, int* cnt, uint64_t* thr, int k) {
    const int n = *cnt;
    int P = 1;
    while (P < n) P <<= 1;
    for (int i = n + threadIdx.x; i < P; i += blockDim.x) buf[i] = kNoKey;
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < P / 2; i += blockDim.x) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const uint64_t a = buf[lo], b = buf[hi];
                if ((a > b) == ((lo & size) == 0)) {
                    buf[lo] = b;
                    buf[hi] = a;
                }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        const int m = n < k ? n : k;
        *cnt = m;
        *thr = m == k ? buf[k - 1] : kNoKey;
    }
    __syncthreads();
}

// append the warp's taken keys (one atomic per warp)
__device__ __forceinline__ void select_offer(uint64_t* buf, int* cnt, uint64_t key, bool take) {
    const unsigned m = __ballot_sync(B2R_FULL_MASK, take);
    if (m == 0) return;
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(cnt, __popc(m));
    base = __shfl_sync(B2R_FULL_MASK, base, leader);
    if (take) buf[base + __popc(m & ((1u << lane) - 1u))] = key;
}

// Offer the keys key_at(0 .. n) to the CTA's selection (buf / cnt / thr in shared memory; NT threads).  `prime` (may
// be a no-op) is called once, by the whole CTA, before the first key that passes the threshold is appended:
// b2r_topk_all_items loads the row's running list there only when the chunk changes it.  Ends with the buffer sorted
// and cut to k.
//
// Each round offers at most NT keys, so a buffer of cap keys is flushed once it holds more than cap - NT.  That
// decision must be the same in every thread: the first barrier of a round orders it after every append of the previous
// round, and the count is evaluated as the predicate of a second barrier (__syncthreads_or), which no thread passes --
// and so no thread appends -- before every thread has read it.  *thr changes only inside select_flush, which ends with
// a barrier.
template <int NT, class KeyAt, class Prime>
__device__ void select_scan(uint64_t* buf, int* cnt, uint64_t* thr, int k, int cap, int64_t n, KeyAt key_at,
                            Prime prime) {
    bool primed = false;
    for (int64_t base = 0; base < n; base += (int64_t)NT * kEPT) {
        uint64_t key[kEPT];
#pragma unroll
        for (int e = 0; e < kEPT; ++e) {
            const int64_t i = base + (int64_t)e * NT + threadIdx.x;
            key[e] = i < n ? key_at(i) : kNoKey;
        }
#pragma unroll
        for (int e = 0; e < kEPT; ++e) {
            __syncthreads();
            if (__syncthreads_or(*cnt > cap - NT)) select_flush(buf, cnt, thr, k);
            const bool take = key[e] < *thr;
            if (!primed && __syncthreads_or(take)) {
                prime();
                primed = true;
            }
            if (primed) select_offer(buf, cnt, key[e], take);
        }
    }
    __syncthreads();
    select_flush(buf, cnt, thr, k);
}

struct NoPrime {
    __device__ void operator()() const {}
};

// One CTA of NT threads per (row, column range).  Source: scores pred[r*ld + c] (keys built here) or, for a merge
// pass, the kNoKey-padded key lists of the previous pass (keys_in, `per_row` keys per row).  Output: when `last_pass`,
// the top-kk of the row as columns + the scores read back from pred; otherwise the range's k keys (kNoKey padded) into
// keys_out.
template <int NT>
__global__ void __launch_bounds__(NT)
k_topk_scan(const float* __restrict__ pred, int64_t ld, const uint64_t* __restrict__ keys_in, int64_t per_row,
            int64_t ranges, int64_t range_len, int k, int kk, bool last_pass, uint64_t* __restrict__ keys_out,
            int64_t* __restrict__ out_idx, float* __restrict__ out_score) {
    extern __shared__ uint64_t buf[];
    __shared__ int cnt;
    __shared__ uint64_t thr;
    const int64_t r = (int64_t)blockIdx.x / ranges, g = (int64_t)blockIdx.x - r * ranges;
    const int64_t c0 = g * range_len;
    const int64_t c1 = c0 + range_len < per_row ? c0 + range_len : per_row;
    const int64_t n = c1 > c0 ? c1 - c0 : 0;
    if (threadIdx.x == 0) {
        cnt = 0;
        thr = kNoKey;
    }
    const int cap = select_cap(k);
    if (keys_in) {
        const uint64_t* src = keys_in + r * per_row + c0;
        select_scan<NT>(buf, &cnt, &thr, k, cap, n, [&](int64_t i) { return src[i]; }, NoPrime());
    } else {
        const float* src = pred + r * ld + c0;
        select_scan<NT>(buf, &cnt, &thr, k, cap, n,
                    [&](int64_t i) { return order_key(src[i], (uint32_t)(c0 + i)); }, NoPrime());
    }
    if (last_pass) {
        for (int t = threadIdx.x; t < kk; t += NT) {
            const int64_t col = (int64_t)(uint32_t)buf[t];
            out_idx[r * kk + t] = col;
            out_score[r * kk + t] = pred[r * ld + col];
        }
    } else {
        uint64_t* dst = keys_out + (r * ranges + g) * k;
        for (int t = threadIdx.x; t < k; t += NT) dst[t] = t < cnt ? buf[t] : kNoKey;
    }
}

__global__ void __launch_bounds__(128)
k_mask_clicked(float* __restrict__ pred, int64_t N, int64_t C, int64_t ld, const int64_t* __restrict__ users,
               const int64_t* __restrict__ clicked_ptr, const int64_t* __restrict__ clicked_items, int64_t n_users,
               int32_t* __restrict__ err_flag) {
    for (int64_t b = blockIdx.x; b < N; b += gridDim.x) {
        const int64_t u = users[b];
        if (u < 0 || u >= n_users) {
            if (threadIdx.x == 0 && err_flag) atomicAdd(err_flag, 1);
            continue;
        }
        const int64_t beg = clicked_ptr[u], end = clicked_ptr[u + 1];
        for (int64_t e = beg + threadIdx.x; e < end; e += blockDim.x) {
            const int64_t j = clicked_items[e];
            if (j >= 1 && j < C) pred[b * ld + j] = __int_as_float(0xff800000);
        }
    }
}

// ---- b2r_topk_all_items ------------------------------------------------------------------------------------------
// Per row b the workspace holds a running list keys[b, 0..k) (ascending, kNoKey padded) and its threshold thr[b].  The
// list opens with column 0 (the target); every item chunk [jc, jc + Wc) is scored by k_score_chunk and merged by
// k_topk_all_merge.  Items are columns: column j >= 1 is item j.

__global__ void __launch_bounds__(128)
k_topk_all_init(const float* __restrict__ Q, int ldq, const float* __restrict__ I, const int64_t* __restrict__ target,
                const int64_t* __restrict__ users, int B, int64_t n_items, int64_t n_users, int d, int k,
                uint64_t* __restrict__ keys, uint64_t* __restrict__ thr, int32_t* __restrict__ err_flag) {
    const int b = blockIdx.x * 128 + threadIdx.x;
    if (b >= B) return;
    int64_t t = target[b];
    const int64_t u = users[b];
    if (t < 0 || t >= n_items) {
        if (err_flag) atomicAdd(err_flag, 1);
        t = 0;
    }
    if ((u < 0 || u >= n_users) && err_flag) atomicAdd(err_flag, 1);
    const float* q = Q + (int64_t)b * ldq;
    const float* it = I + t * d;
    float s = 0.f;
    for (int kk = 0; kk < d; ++kk) s = fmaf(q[kk], it[kk], s);
    const uint64_t k0 = order_key(s, 0u);
    uint64_t* row = keys + (int64_t)b * k;
    row[0] = k0;
    for (int i = 1; i < k; ++i) row[i] = kNoKey;
    thr[b] = k == 1 ? k0 : kNoKey;
}

__global__ void __launch_bounds__(kAT)
k_score_chunk(const float* __restrict__ Q, int ldq, const float* __restrict__ I, int B, int64_t n_items, int d,
              int64_t jc, int W, float* __restrict__ S) {
    __shared__ float Qs[kTK][kTQ + 4];
    __shared__ float Is[kTK][kTI + 4];
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    const int q0 = blockIdx.y * kTQ;
    const int off = blockIdx.x * kTI + tx * 8;                       // column inside the chunk
    float acc[8][8];
    rank_tile_accumulate(Q, ldq, I, B, n_items, d, q0, jc + (int64_t)blockIdx.x * kTI, Qs, Is, acc);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int q = q0 + ty * 8 + i;
        if (q < B) {
            float* dst = S + (int64_t)q * W + off;
            st4(dst, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
            st4(dst + 4, make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]));
        }
    }
}

__global__ void __launch_bounds__(kKT)
k_topk_all_merge(const float* __restrict__ S, int W, int64_t jc, int Wc, const int64_t* __restrict__ users,
                 const int64_t* __restrict__ clicked_ptr, const int64_t* __restrict__ clicked_items, int64_t n_users,
                 int k, uint64_t* __restrict__ keys, uint64_t* __restrict__ thr_g) {
    extern __shared__ uint64_t buf[];
    __shared__ int cnt;
    __shared__ uint64_t thr;
    __shared__ uint32_t masked[kChunkMax / 32];
    __shared__ int64_t mlo, mhi;
    __shared__ int loaded;                                          // the running list was read (and must be written)
    const int b = blockIdx.x;
    for (int i = threadIdx.x; i < (Wc + 31) / 32; i += kKT) masked[i] = 0u;
    if (threadIdx.x == 0) {
        cnt = 0;
        loaded = 0;
        thr = thr_g[b];
        int64_t u = users[b];
        if (u < 0 || u >= n_users) u = 0;                          // counted by k_topk_all_init
        // the user's sorted slice, cut to [jc, jc + Wc)
        int64_t lo = clicked_ptr[u], hi = clicked_ptr[u + 1];
        int64_t a = lo, z = hi;
        while (a < z) {
            const int64_t m = (a + z) >> 1;
            if (clicked_items[m] < jc) a = m + 1; else z = m;
        }
        mlo = a;
        z = hi;
        while (a < z) {
            const int64_t m = (a + z) >> 1;
            if (clicked_items[m] < jc + Wc) a = m + 1; else z = m;
        }
        mhi = a;
    }
    __syncthreads();
    for (int64_t e = mlo + threadIdx.x; e < mhi; e += kKT) {
        const int c = (int)(clicked_items[e] - jc);
        atomicOr(&masked[c >> 5], 1u << (c & 31));
    }
    __syncthreads();
    uint64_t* row = keys + (int64_t)b * k;
    const float* src = S + (int64_t)b * W;
    auto key_at = [&](int64_t i) {
        const float s = (masked[i >> 5] >> (i & 31)) & 1u ? __int_as_float(0xff800000) : src[i];
        return order_key(s, (uint32_t)(jc + i));
    };
    auto prime = [&]() {                                            // the running list joins the selection
        for (int i = threadIdx.x; i < k; i += kKT) {
            const uint64_t v = row[i];
            buf[i] = v;
            if (v != kNoKey && (i + 1 == k || row[i + 1] == kNoKey)) cnt = i + 1;
        }
        if (threadIdx.x == 0) loaded = 1;
        __syncthreads();
    };
    select_scan<kKT>(buf, &cnt, &thr, k, select_cap(k), Wc, key_at, prime);
    if (loaded) {
        for (int i = threadIdx.x; i < k; i += kKT) row[i] = i < cnt ? buf[i] : kNoKey;
        if (threadIdx.x == 0) thr_g[b] = thr;
    }
}

__global__ void __launch_bounds__(128)
k_topk_all_out(const uint64_t* __restrict__ keys, const int64_t* __restrict__ target, int B, int64_t n_items, int k,
               int kk, int64_t* __restrict__ out_items, float* __restrict__ out_scores) {
    const int64_t total = (int64_t)B * kk;
    for (int64_t idx = (int64_t)blockIdx.x * 128 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 128) {
        const int64_t b = idx / kk, t = idx - b * kk;
        const uint64_t key = keys[b * k + t];
        const int64_t col = (int64_t)(uint32_t)key;
        int64_t item = col;
        if (col == 0) {
            item = target[b];
            if (item < 0 || item >= n_items) item = 0;
        }
        out_items[idx] = item;
        out_scores[idx] = key_score(key);
    }
}

// ---- host-side shapes ---------------------------------------------------------------------------------------------

static int64_t rows_ranges(int64_t N, int64_t C) {
    if (C <= kRangeMin) return 1;
    const int64_t by_len = (C + kRangeMin - 1) / kRangeMin;
    int64_t want = (kRangeCtas + N - 1) / N;
    if (want < 1) want = 1;
    return want < by_len ? want : by_len;
}

static int all_chunk_width(int B, int64_t n_items) {
    int64_t w = (int64_t)(kChunkBytes / (4 * (size_t)(B > 0 ? B : 1))) / kTI * kTI;
    if (w < kTI) w = kTI;
    if (w > kChunkMax) w = kChunkMax;
    const int64_t need = (n_items - 1 + kTI - 1) / kTI * kTI;     // candidates 1 .. n_items - 1
    if (need >= kTI && w > need) w = need;
    return (int)w;
}

struct AllLayout {
    size_t scores, keys, thr, total;
    int W;
};

static AllLayout all_layout(int B, int64_t n_items, int k) {
    AllLayout L;
    L.W = all_chunk_width(B, n_items);
    L.scores = 0;
    L.keys = align_up((size_t)B * L.W * sizeof(float), 256);
    L.thr = L.keys + align_up((size_t)B * k * sizeof(uint64_t), 256);
    L.total = L.thr + align_up((size_t)B * sizeof(uint64_t), 256);
    return L;
}

}  // namespace b2r

using namespace b2r;

extern "C" size_t b2r_topk_rows_workspace_bytes(int64_t N, int64_t C, int k) {
    if (N <= 0 || C <= 0 || k < 1 || k > kMaxTopK) return 0;
    const int64_t ranges = rows_ranges(N, C);
    return ranges > 1 ? (size_t)N * ranges * k * sizeof(uint64_t) : 0;
}

extern "C" int b2r_topk_rows(const float* pred, int64_t N, int64_t C, int64_t ld, int k, int64_t* out_idx,
                             float* out_score, void* workspace, size_t workspace_bytes, b2r_stream_t stream) {
    B2R_REQUIRE(pred && out_idx && out_score, B2R_E_BADARG, "b2r_topk_rows: null pointer");
    B2R_REQUIRE(N >= 0 && C >= 1 && ld >= C && k >= 1, B2R_E_BADARG, "b2r_topk_rows: bad shape N=%lld C=%lld ld=%lld k=%d",
                (long long)N, (long long)C, (long long)ld, k);
    B2R_REQUIRE(k <= kMaxTopK, B2R_E_UNSUPPORTED, "b2r_topk_rows: k=%d above %d", k, kMaxTopK);
    B2R_REQUIRE(C < 0x7fffffffLL, B2R_E_UNSUPPORTED, "b2r_topk_rows: C=%lld columns", (long long)C);
    const size_t need = b2r_topk_rows_workspace_bytes(N, C, k);
    B2R_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), B2R_E_WORKSPACE,
                "b2r_topk_rows: workspace %zu < %zu bytes", workspace_bytes, need);
    if (N == 0) return 0;
    cudaStream_t s = as_stream(stream);
    const int kk = (int)(C < k ? C : k);
    const size_t smem = (size_t)select_cap(k) * sizeof(uint64_t);
    const int64_t ranges = rows_ranges(N, C);
    B2R_REQUIRE(N * ranges <= 0x7fffffffLL, B2R_E_UNSUPPORTED, "b2r_topk_rows: grid");
    if (ranges == 1) {
        if (C <= kSmallC)        // short rows: a 256-thread CTA would leave most of its threads idle
            k_topk_scan<kKTSmall><<<(unsigned)N, kKTSmall, smem, s>>>(pred, ld, nullptr, C, 1, C, k, kk, true, nullptr,
                                                                     out_idx, out_score);
        else
            k_topk_scan<kKT><<<(unsigned)N, kKT, smem, s>>>(pred, ld, nullptr, C, 1, C, k, kk, true, nullptr, out_idx,
                                                           out_score);
        B2R_LAUNCH_OK("k_topk_scan");
        return 0;
    }
    uint64_t* partial = static_cast<uint64_t*>(workspace);
    const int64_t range_len = (C + ranges - 1) / ranges;
    k_topk_scan<kKT><<<(unsigned)(N * ranges), kKT, smem, s>>>(pred, ld, nullptr, C, ranges, range_len, k, kk, false,
                                                               partial, nullptr, nullptr);
    B2R_LAUNCH_OK("k_topk_scan");
    k_topk_scan<kKT><<<(unsigned)N, kKT, smem, s>>>(pred, ld, partial, ranges * k, 1, ranges * k, k, kk, true, nullptr,
                                                    out_idx, out_score);
    B2R_LAUNCH_OK("k_topk_scan");
    return 0;
}

extern "C" int b2r_mask_clicked(float* pred, int64_t N, int64_t C, int64_t ld, const int64_t* users,
                                const int64_t* clicked_ptr, const int64_t* clicked_items, int64_t n_users,
                                int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(pred && users && clicked_ptr && clicked_items, B2R_E_BADARG, "b2r_mask_clicked: null pointer");
    B2R_REQUIRE(N >= 0 && C >= 1 && ld >= C && n_users >= 1, B2R_E_BADARG, "b2r_mask_clicked: bad shape");
    if (N == 0) return 0;
    int64_t grid = N;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    k_mask_clicked<<<(int)grid, 128, 0, as_stream(stream)>>>(pred, N, C, ld, users, clicked_ptr, clicked_items, n_users,
                                                            err_flag);
    B2R_LAUNCH_OK("k_mask_clicked");
    return 0;
}

extern "C" size_t b2r_topk_all_items_workspace_bytes(int B, int64_t n_items, int k) {
    if (B <= 0 || n_items < 1 || k < 1 || k > kMaxTopK) return 0;
    return all_layout(B, n_items, k).total;
}

extern "C" int b2r_topk_all_items(const float* Q, int ldq, const float* I, int64_t n_items, int d,
                                  const int64_t* target, const int64_t* users, int B, const int64_t* clicked_ptr,
                                  const int64_t* clicked_items, int64_t n_users, int k, int64_t* out_items,
                                  float* out_scores, int32_t* err_flag, void* workspace, size_t workspace_bytes,
                                  b2r_stream_t stream) {
    B2R_REQUIRE(Q && I && target && users && clicked_ptr && clicked_items && out_items && out_scores, B2R_E_BADARG,
                "b2r_topk_all_items: null pointer");
    B2R_REQUIRE(B >= 0 && n_items >= 1 && d >= 1 && ldq >= d && n_users >= 1 && k >= 1, B2R_E_BADARG,
                "b2r_topk_all_items: bad shape B=%d n_items=%lld d=%d k=%d", B, (long long)n_items, d, k);
    B2R_REQUIRE(k <= kMaxTopK, B2R_E_UNSUPPORTED, "b2r_topk_all_items: k=%d above %d", k, kMaxTopK);
    B2R_REQUIRE(d % 4 == 0 && aligned16(I), B2R_E_UNSUPPORTED, "b2r_topk_all_items: d=%d must be a multiple of 4", d);
    B2R_REQUIRE(n_items < 0x7fffffffLL && (B + kTQ - 1) / kTQ <= 65535, B2R_E_UNSUPPORTED, "b2r_topk_all_items: shape");
    if (B == 0) return 0;
    const AllLayout L = all_layout(B, n_items, k);
    B2R_REQUIRE(workspace && workspace_bytes >= L.total && aligned16(workspace), B2R_E_WORKSPACE,
                "b2r_topk_all_items: workspace %zu < %zu bytes", workspace_bytes, L.total);
    cudaStream_t s = as_stream(stream);
    char* ws = static_cast<char*>(workspace);
    float* S = reinterpret_cast<float*>(ws + L.scores);
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + L.keys);
    uint64_t* thr = reinterpret_cast<uint64_t*>(ws + L.thr);
    k_topk_all_init<<<(B + 127) / 128, 128, 0, s>>>(Q, ldq, I, target, users, B, n_items, n_users, d, k, keys, thr,
                                                   err_flag);
    B2R_LAUNCH_OK("k_topk_all_init");
    const size_t smem = (size_t)select_cap(k) * sizeof(uint64_t);
    for (int64_t jc = 1; jc < n_items; jc += L.W) {
        const int Wc = (int)(n_items - jc < L.W ? n_items - jc : L.W);
        dim3 grid((unsigned)((Wc + kTI - 1) / kTI), (unsigned)((B + kTQ - 1) / kTQ));
        k_score_chunk<<<grid, kAT, 0, s>>>(Q, ldq, I, B, n_items, d, jc, L.W, S);
        B2R_LAUNCH_OK("k_score_chunk");
        k_topk_all_merge<<<B, kKT, smem, s>>>(S, L.W, jc, Wc, users, clicked_ptr, clicked_items, n_users, k, keys, thr);
        B2R_LAUNCH_OK("k_topk_all_merge");
    }
    const int kk = (int)(n_items < k ? n_items : k);
    int64_t grid = ((int64_t)B * kk + 127) / 128;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    k_topk_all_out<<<(int)grid, 128, 0, s>>>(keys, target, B, n_items, k, kk, out_items, out_scores);
    B2R_LAUNCH_OK("k_topk_all_out");
    return 0;
}
