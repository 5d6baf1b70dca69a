// bucket.cu -- the hot-path form of the row-sparse embedding backward + optimizer (K2b).
//   plan side (depends only on the ids; runs on the step context's side stream, one step ahead; plan_direct.cuh):
//     k_direct_scatter_pair  drops the batch's (row id, position) pairs into fixed-capacity regions of buckets of
//         2^shift consecutive table rows (~200 pairs each) with one L2 atomic per pair on a line-padded cursor;
//     k_bucket_sort_warp  one warp per bucket sorts its pairs by (row, position) (register bitonic network for small
//         buckets, counting sort in warp-private shared memory otherwise) and writes them back in place;
//     k_bucket_sort_deferred  one CTA per bucket the warps could not take (spilled, too wide, a row with many
//         contributions): counting sort or bitonic network in shared memory, chunked merge beyond it.  Buckets
//         cover ascending disjoint row ranges, so the whole array ends up sorted exactly as a device-wide radix sort
//         would leave it, at a fraction of the cost; rows with many contributions are listed for the cooperative
//         reduction; buckets beyond the shared-memory capacity are chunk-sorted and merged.
//         The sort also lists every touched row once: (row, first position, index of its first pair, run length).
//   apply side (main stream):
//     k_apply_sorted  one lane group per touched row (head list): requests w (m, v), sums the row's contributions in
//         ascending position, applies SGD/Adam/Adagrad in place (mode 2) or adds into a dense gradient (mode 1).
//         No barriers, no atomics.  Rows with >= kLong contributions (listed by the sort) are then reduced by whole
//         CTAs in a fixed order.  A launch can carry two independent tables (jobs).
// Every sum has a fixed order whatever order the partition's atomics produced -> same bits on every run.
// Replaces ATen embedding_dense_backward + the dense grad zero-fill + the embedding part of optimizer.step()
// (helpers/BaseRunner.py:193,205,206).
#include "common.cuh"
#include "plan_direct.cuh"

namespace b2r {

struct BSrc {
    const float* src;
    const float* coef;
    const int64_t* src_id;
    int64_t n;
    int32_t ld;
    FastDiv div;
};

constexpr int kCap = 2048;        // pairs a CTA sorts in shared memory (16 KB)
constexpr int kLong = 48;         // rows with at least this many contributions are reduced by the whole CTA
constexpr int kBT = 256;
constexpr int kCountShift = 12;   // counting-sort candidate: buckets of at most 4096 rows ...
constexpr int kCountRows = 1 << kCountShift;
constexpr int kRunMax = 32;       // ... whose longest row has at most this many contributions

__device__ __forceinline__ void b_contribution(const BSrc& s0, const BSrc& s1, uint32_t p, const float*& base,
                                               int& ld, int64_t& row, float& c) {
    const bool first = (int64_t)p < s0.n;
    const int64_t pp = first ? (int64_t)p : (int64_t)p - s0.n;
    const int64_t* sid = first ? s0.src_id : s1.src_id;
    const float* cf = first ? s0.coef : s1.coef;
    int64_t r = (int64_t)fastdiv((uint32_t)pp, first ? s0.div : s1.div);
    if (sid != nullptr) r = sid[r];
    row = r;
    c = (cf != nullptr) ? cf[pp] : 1.f;
    base = first ? s0.src : s1.src;
    ld = first ? s0.ld : s1.ld;
}

__device__ __forceinline__ void b_optim(const b2r_optim& o, float4& w, float4& m, float4& v, const float4& gin) {
    float* wp = &w.x;
    float* mp = &m.x;
    float* vp = &v.x;
    const float* gp = &gin.x;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float g = fmaf(o.weight_decay, wp[i], gp[i]);
        if (o.kind == 0) {
            wp[i] = fmaf(-o.lr, g, wp[i]);
        } else if (o.kind == 1) {
            mp[i] = fmaf(o.beta1, mp[i], (1.f - o.beta1) * g);
            vp[i] = fmaf(o.beta2, vp[i], (1.f - o.beta2) * g * g);
            const float denom = sqrtf(vp[i]) / sqrtf(o.bc2) + o.eps;
            wp[i] = wp[i] - (o.lr / o.bc1) * (mp[i] / denom);
        } else {
            vp[i] = fmaf(g, g, vp[i]);
            wp[i] = wp[i] - o.lr * g / (sqrtf(vp[i]) + o.eps);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// per-bucket sort + segment reduce + optimizer
// ---------------------------------------------------------------------------------------------------
template <int LPR>
struct RowIO {
    static constexpr int D = LPR * 4;
    // MODE 0: rows -> grad_rows[out_base + u], uniq_rows; MODE 1: dense += ; MODE 2: optimizer in place
    template <int MODE>
    __device__ static __forceinline__ void finish(int64_t row, const float4& acc, int sub, float4 w, float4 m, float4 v,
                                                  float* W, float* M, float* V, float* dense, const OptK& opt) {
        if (MODE == 1) {
            w.x += acc.x; w.y += acc.y; w.z += acc.z; w.w += acc.w;
            st4(dense + row * D + sub * 4, w);
        } else {
            optk_update4_fast(opt, w, m, v, acc);
            st4(W + row * D + sub * 4, w);
            if (opt.kind == 1) st4(M + row * (opt.state_ld ? opt.state_ld : D) + sub * 4, m);
            if (opt.kind != 0) st4(V + row * (opt.state_ld ? opt.state_ld : D) + sub * 4, v);
        }
    }
};

__device__ __forceinline__ void bitonic_sort_smem(uint64_t* s, int P) {
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (P >> 1); t += kBT) {
                const int i = ((t / j) * (j << 1)) + (t % j);
                const int l = i + j;
                const bool up = (i & k) == 0;
                const uint64_t a = s[i], b = s[l];
                if ((a > b) == up) {
                    s[i] = b;
                    s[l] = a;
                }
            }
            __syncthreads();
        }
    }
}

// first index in the sorted run a[0..n) whose value is >= v (ties cannot occur: (row, position) pairs are unique)
__device__ __forceinline__ int lower_bound64(const uint64_t* a, int n, uint64_t v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// After a bucket is sorted (a = its pairs, in shared or global memory): list every row's first pair as
// (row, position of the first pair, index of the first pair, run length) for k_apply_sorted, which then never has to
// discover run boundaries itself.  Rows with >= kLong contributions go to the cooperative list instead (their head
// entry carries length 0).  Slots are reserved with one global atomic per bucket; the order of the list does not
// influence any result (each row is reduced by exactly one lane group, in ascending position).
__device__ __forceinline__ void emit_row_heads(const uint64_t* a, int cnt, int beg, int* n_long, uint2* longs,
                                               int long_cap, int* n_heads, uint4* heads, int* head_cnt,
                                               int* head_base) {
    __syncthreads();                                   // a[] complete, *head_cnt == 0
    int mine = 0;
    for (int i = threadIdx.x; i < cnt; i += kBT)
        mine += (i == 0 || (uint32_t)(a[i - 1] >> 32) != (uint32_t)(a[i] >> 32)) ? 1 : 0;
    if (mine) atomicAdd(head_cnt, mine);
    __syncthreads();
    if (threadIdx.x == 0) {
        *head_base = atomicAdd(n_heads, *head_cnt);
        *head_cnt = 0;
    }
    __syncthreads();
    const int base = *head_base;
    for (int i = threadIdx.x; i < cnt; i += kBT) {
        const uint64_t v = a[i];
        const uint32_t key = (uint32_t)(v >> 32);
        if (i == 0 || (uint32_t)(a[i - 1] >> 32) != key) {
            const int len = lower_bound64(a, cnt, ((uint64_t)key + 1) << 32) - i;
            const bool is_long = len >= kLong;
            if (is_long) {
                const int q = atomicAdd(n_long, 1);
                if (q < long_cap) longs[q] = make_uint2((uint32_t)(beg + i), (uint32_t)len);
            }
            const int slot = base + atomicAdd(head_cnt, 1);
            heads[slot] = make_uint4(key, (uint32_t)v, (uint32_t)(beg + i), is_long ? 0u : (uint32_t)len);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) *head_cnt = 0;
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// Counting sort of a bucket.  The bitonic network costs 36-45 barrier-separated stages per bucket; a bucket's keys span
// only R = 2^shift rows, so one shared-memory histogram over the rows gives every pair its row's start, an arrival-order
// slot inside the row, and -- for free -- the row heads.  Rows with several contributions (a minority) are put in
// ascending position by one thread each (insertion sort, at most kRunMax elements).  Returns false, having written
// nothing, when a row has more than kRunMax contributions: the caller then runs the bitonic path.  Output is identical
// to the bitonic path (same sorted array; the head list is a permutation of the same entries).
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool bucket_sort_counting(uint64_t* __restrict__ g, int cnt, int beg, uint32_t row0, int R,
                                                     uint64_t* s, int* hist, int* scratch, int* n_heads,
                                                     uint4* heads) {
    constexpr int PER = kCap / kBT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int r = tid; r <= R; r += kBT) hist[r] = 0;
    if (tid == 0) {
        scratch[32] = 0;     // largest row count
        scratch[33] = 0;     // head counter
    }
    __syncthreads();
    uint64_t v[PER];
    int rk[PER];
#pragma unroll
    for (int q = 0; q < PER; ++q) {
        const int i = tid + q * kBT;
        v[q] = 0;
        rk[q] = 0;
        if (i < cnt) {
            v[q] = g[i];
            rk[q] = atomicAdd(&hist[(uint32_t)(v[q] >> 32) - row0], 1);
        }
    }
    __syncthreads();
    // thread t owns rows [t * RP, (t + 1) * RP): largest count, then an exclusive scan across the CTA
    const int RP = (R + kBT - 1) / kBT;
    int local = 0, mx = 0;
    for (int x = 0; x < RP; ++x) {
        const int r = tid * RP + x;
        if (r < R) {
            const int c = hist[r];
            local += c;
            mx = max(mx, c);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(B2R_FULL_MASK, mx, o));
    if (lane == 0) atomicMax(&scratch[32], mx);
    int inc = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(B2R_FULL_MASK, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) scratch[warp] = inc;
    __syncthreads();
    if (scratch[32] > kRunMax) return false;             // same value in every thread
    int run = inc - local;
    for (int w = 0; w < warp; ++w) run += scratch[w];
    for (int x = 0; x < RP; ++x) {
        const int r = tid * RP + x;
        if (r < R) {
            const int c = hist[r];
            hist[r] = run;                               // start of row r in the sorted bucket
            run += c;
        }
    }
    if (tid == 0) hist[R] = cnt;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < PER; ++q) {
        const int i = tid + q * kBT;
        if (i < cnt) s[hist[(uint32_t)(v[q] >> 32) - row0] + rk[q]] = v[q];
    }
    __syncthreads();
    int mine = 0;
    for (int r = tid; r < R; r += kBT) {
        const int a = hist[r], b = hist[r + 1];
        for (int x = a + 1; x < b; ++x) {                // insertion sort of the row's run by (row, position)
            const uint64_t val = s[x];
            int y = x - 1;
            while (y >= a && s[y] > val) {
                s[y + 1] = s[y];
                --y;
            }
            s[y + 1] = val;
        }
        mine += (b > a) ? 1 : 0;
    }
    if (mine) atomicAdd(&scratch[33], mine);
    __syncthreads();
    if (tid == 0) {
        scratch[34] = atomicAdd(n_heads, scratch[33]);
        scratch[33] = 0;
    }
    __syncthreads();
    const int base = scratch[34];
    for (int r = tid; r < R; r += kBT) {
        const int a = hist[r], b = hist[r + 1];
        if (b > a) {
            const int slot = base + atomicAdd(&scratch[33], 1);
            heads[slot] = make_uint4(row0 + (uint32_t)r, (uint32_t)s[a], (uint32_t)(beg + a), (uint32_t)(b - a));
        }
    }
    for (int i = tid; i < cnt; i += kBT) g[i] = s[i];
    __syncthreads();
    return true;
}

// sort one bucket's pairs g[0, cnt) in place (beg = index of g[0] in the plan's pair address space, tg = scratch of the
// same extent for the merge path) and list its row heads / long rows
__device__ __forceinline__ void sort_one_bucket(uint64_t* g, uint64_t* tg, int cnt, int beg, uint32_t row0, int shift,
                                                uint64_t* s, int* hist, int* scratch, int* head_cnt, int* head_base,
                                                int* n_long, uint2* longs, int long_cap, int* n_heads, uint4* heads) {
    const int tid = threadIdx.x;
    if (cnt <= kCap && shift <= kCountShift &&
        bucket_sort_counting(g, cnt, beg, row0, 1 << shift, s, hist, scratch, n_heads, heads))
        return;
    if (cnt <= kCap) {
        int P = 32;
        while (P < cnt) P <<= 1;
        for (int i = tid; i < P; i += kBT) s[i] = i < cnt ? g[i] : ~0ull;
        __syncthreads();
        bitonic_sort_smem(s, P);
        for (int i = tid; i < cnt; i += kBT) g[i] = s[i];
        emit_row_heads(s, cnt, beg, n_long, longs, long_cap, n_heads, heads, head_cnt, head_base);
    } else {
        // chunked shared-memory sorts ...
        for (int c0 = 0; c0 < cnt; c0 += kCap) {
            const int m = min(kCap, cnt - c0);
            int P = 32;
            while (P < m) P <<= 1;
            for (int i = tid; i < P; i += kBT) s[i] = i < m ? g[c0 + i] : ~0ull;
            __syncthreads();
            bitonic_sort_smem(s, P);
            for (int i = tid; i < m; i += kBT) g[c0 + i] = s[i];
            __syncthreads();
        }
        // ... then pairwise merges by rank (each element: own index + rank in the sibling run), ping-pong g <-> tg
        uint64_t* src = g;
        uint64_t* dst = tg;
        for (int width = kCap; width < cnt; width <<= 1) {
            for (int i = tid; i < cnt; i += kBT) {
                const int run = i / width;
                const int base = (run & ~1) * width;
                const int a0 = base, a1 = min(cnt, base + width), b1 = min(cnt, base + 2 * width);
                const uint64_t v = src[i];
                int pos;
                if ((run & 1) == 0) pos = (i - a0) + lower_bound64(src + a1, b1 - a1, v);
                else pos = (i - a1) + lower_bound64(src + a0, a1 - a0, v);
                dst[base + pos] = v;
            }
            __syncthreads();
            uint64_t* t2 = src; src = dst; dst = t2;
        }
        if (src != g) {
            for (int i = tid; i < cnt; i += kBT) g[i] = src[i];
            __syncthreads();
        }
        emit_row_heads(g, cnt, beg, n_long, longs, long_cap, n_heads, heads, head_cnt, head_base);
    }
}

// ---------------------------------------------------------------------------------------------------
// The CTA sort of a direct plan's bucket (sort_one_bucket), for the buckets k_bucket_sort_warp defers.  Pairs were
// dropped into fixed-capacity bucket regions by k_direct_scatter_pair (plan_direct.cuh).  A bucket that overflowed its
// region (skewed ids) first collects its spilled pairs from the spill list into the "big" area behind the regions and
// is sorted there.
// ---------------------------------------------------------------------------------------------------
struct DirectSortJob {
    int nb, cap, shift;
    int* cursor;
    uint64_t* region;
    uint64_t* spill;
    int* counters;               // [0] spill count, [1] big cursor, [2] n_long, [3] n_heads, [4] deferred buckets
    int spill_cap;
    uint64_t* big;
    uint64_t* tmp;               // scratch for the merge path, same extent as big
    int big_cap;
    uint2* longs;
    int long_cap;
    uint4* heads;
    int2* deferred;              // [nb] (bucket, pair count) the warp sort left to the CTA pass
};

// one bucket (raw = its cursor's count) by a whole CTA: the region in place, or -- overflow -- region + spilled pairs
// gathered into the big area
__device__ __forceinline__ void direct_sort_bucket(const DirectSortJob& J, int b, int raw, uint64_t* s, int* hist,
                                                   int* scratch, int* head_cnt, int* head_base, int* sh) {
    const int tid = threadIdx.x;
    const uint32_t row0 = (uint32_t)b << J.shift;
    if (raw <= J.cap) {
        const int beg = b * J.cap;
        sort_one_bucket(J.region + (int64_t)beg, J.tmp, raw, beg, row0, J.shift, s, hist, scratch, head_cnt,
                               head_base, J.counters + 2, J.longs, J.long_cap, J.counters + 3, J.heads);
        return;
    }
    // overflow: region (cap pairs) + this bucket's share of the spill list -> contiguous run in the big area
    const int nsp = min(J.counters[0], J.spill_cap);
    int mine = 0;
    for (int i = tid; i < nsp; i += kBT) mine += ((uint32_t)(J.spill[i] >> 32) >> J.shift) == (uint32_t)b ? 1 : 0;
    if (tid == 0) sh[1] = 0;
    __syncthreads();
    if (mine) atomicAdd(&sh[1], mine);
    __syncthreads();
    const int total = J.cap + sh[1];
    if (tid == 0) {
        sh[2] = atomicAdd(&J.counters[1], total);
        sh[3] = 0;
    }
    __syncthreads();
    const int base = sh[2];
    if (base + total > J.big_cap) return;               // cannot happen (big_cap = 2n); never write out of bounds
    uint64_t* g = J.big + base;
    for (int i = tid; i < J.cap; i += kBT) g[i] = J.region[(int64_t)b * J.cap + i];
    for (int i = tid; i < nsp; i += kBT) {
        const uint64_t v = J.spill[i];
        if (((uint32_t)(v >> 32) >> J.shift) == (uint32_t)b) g[J.cap + atomicAdd(&sh[3], 1)] = v;
    }
    __syncthreads();
    // pair indices of the big area continue after the regions: nb * cap + offset
    sort_one_bucket(g, J.tmp + base, total, J.nb * J.cap + base, row0, J.shift, s, hist, scratch, head_cnt,
                           head_base, J.counters + 2, J.longs, J.long_cap, J.counters + 3, J.heads);
}

// the pairs of one or two id arrays into their direct plans (one launch; CTAs [0, grid_a) work on a).  Each thread keeps
// kScatterILP pairs in flight: with the bounded grid of the step context a thread handles many pairs, and one
// returning L2 atomic at a time would leave the launch latency-bound.
constexpr int kScatterILP = 4;

__device__ __forceinline__ void scatter_ids(const DirectPlanDev& P, const int64_t* __restrict__ ids, int64_t n,
                                            int64_t rows, int64_t first, int64_t stride, int32_t* err_flag,
                                            int64_t ignore_id, int64_t ignore_n) {
    for (int64_t i0 = first; i0 < n; i0 += stride * kScatterILP) {
        int64_t id[kScatterILP];
#pragma unroll
        for (int u = 0; u < kScatterILP; ++u) {
            const int64_t i = i0 + u * stride;
            id[u] = i < n ? ids[i] : -1;
        }
#pragma unroll
        for (int u = 0; u < kScatterILP; ++u) {
            const int64_t i = i0 + u * stride;
            if (i >= n || (i < ignore_n && id[u] == ignore_id)) continue;   // padding positions contribute nothing
            direct_scatter(P, (uint32_t)checked_id(id[u], rows, err_flag), (uint32_t)i);
        }
    }
}

__global__ void __launch_bounds__(kBT)
k_direct_scatter_pair(const int64_t* __restrict__ ids_a, int64_t n_a, int64_t rows_a, const __grid_constant__ DirectPlanDev pa,
                      int grid_a, const int64_t* __restrict__ ids_b, int64_t n_b, int64_t rows_b,
                      const __grid_constant__ DirectPlanDev pb, int32_t* err_flag, int64_t ignore_id, int64_t ignore_n) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {           // counters the following sort accumulates into
        pa.counters[1] = pa.counters[2] = pa.counters[3] = pa.counters[4] = 0;
        if (n_b > 0) pb.counters[1] = pb.counters[2] = pb.counters[3] = pb.counters[4] = 0;
    }
    if ((int)blockIdx.x < grid_a) {
        scatter_ids(pa, ids_a, n_a, rows_a, (int64_t)blockIdx.x * kBT + threadIdx.x, (int64_t)grid_a * kBT, err_flag,
                    ignore_id, ignore_n);                 // the padding rule applies to plan a only
    } else {
        const int gb = (int)gridDim.x - grid_a;
        scatter_ids(pb, ids_b, n_b, rows_b, (int64_t)((int)blockIdx.x - grid_a) * kBT + threadIdx.x, (int64_t)gb * kBT,
                    err_flag, -1, 0);
    }
}

// ---------------------------------------------------------------------------------------------------
// k_bucket_sort_warp: one warp per bucket, warp-private shared memory, __syncwarp only.  A bucket of a typical batch
// holds ~200 pairs (items) or ~30 (users): a 256-thread CTA per bucket leaves most of its threads idle and, with 33 KB of
// shared memory and 64 registers a thread, takes the SM slot of a forward or optimizer CTA.  The warp form keeps the
// plan's footprint small (kSortWarps warps and kSortWarps * ~8 KB per CTA) so that it can run underneath the step's
// HBM-bound kernels.  Output is the same as the CTA sort's: the same sorted pair array, the same row heads (the order
// of the head list differs; nothing depends on it) and the same long rows.
//   <= kRegSort pairs (any bucket width): bitonic network in registers (two pairs a lane, shuffles);
//   otherwise, bucket rows <= 2^kWarpShift and pairs <= kWarpCap: counting sort over a warp-private row histogram,
//       rows with several contributions put in ascending position by insertion sort (at most kRunMax each);
//   anything else (overflowed into the spill list, a row with > kRunMax contributions, a bucket too wide or too full)
//       goes on the plan's deferred list for k_bucket_sort_deferred, which runs the CTA sort above.
// ---------------------------------------------------------------------------------------------------
constexpr int kSortWarps = 4;            // warps of a k_bucket_sort_warp CTA
constexpr int kWarpCap = 768;            // pairs a warp sorts in its shared-memory slice (6 KB)
constexpr int kWarpShift = 9;            // widest bucket a warp's histogram covers: 512 rows (2 KB)
constexpr int kRegSort = 64;             // pairs sorted in registers

struct WarpSortSmem {
    uint64_t s[kWarpCap];
    int hist[(1 << kWarpShift) + 1];
};

__device__ __forceinline__ uint64_t bitonic_lane(uint64_t v, int i, int j, int k) {
    const uint64_t p = __shfl_xor_sync(B2R_FULL_MASK, v, j);
    const bool lower = (i & j) == 0, up = (i & k) == 0;
    return (lower == up) ? (v < p ? v : p) : (v < p ? p : v);
}

// cnt <= kRegSort pairs g[0, cnt): sorted in registers (element i in lane i % 32, register i / 32), written back, heads
// (and long rows, >= kLong contributions) listed with one slot reservation per bucket
__device__ __forceinline__ void warp_sort_small(const DirectSortJob& J, uint64_t* g, int cnt, int beg) {
    const int lane = threadIdx.x & 31;
    uint64_t e0 = lane < cnt ? g[lane] : ~0ull;
    uint64_t e1 = lane + 32 < cnt ? g[lane + 32] : ~0ull;
    for (int k = 2; k <= 64; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            if (j == 32) {                               // k == 64: the two registers of a lane, ascending
                const uint64_t lo = e0 < e1 ? e0 : e1, hi = e0 < e1 ? e1 : e0;
                e0 = lo;
                e1 = hi;
            } else {
                e0 = bitonic_lane(e0, lane, j, k);
                e1 = bitonic_lane(e1, lane + 32, j, k);
            }
        }
    }
    const uint32_t k0 = (uint32_t)(e0 >> 32), k1 = (uint32_t)(e1 >> 32);
    const uint32_t p0 = __shfl_up_sync(B2R_FULL_MASK, k0, 1), p1 = __shfl_up_sync(B2R_FULL_MASK, k1, 1);
    const uint32_t last0 = __shfl_sync(B2R_FULL_MASK, k0, 31);
    const bool h0 = lane < cnt && (lane == 0 || p0 != k0);
    const bool h1 = lane + 32 < cnt && (lane == 0 ? last0 != k1 : p1 != k1);
    const uint64_t H = ((uint64_t)__ballot_sync(B2R_FULL_MASK, h1) << 32) | __ballot_sync(B2R_FULL_MASK, h0);
    int base = 0;
    if (lane == 0) base = atomicAdd(J.counters + 3, __popcll(H));
    base = __shfl_sync(B2R_FULL_MASK, base, 0);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int i = lane + 32 * r;
        const uint64_t v = r ? e1 : e0;
        if (i < cnt) g[i] = v;
        if (!(r ? h1 : h0)) continue;
        const uint64_t after = H & ~((2ull << i) - 1);   // heads behind i (i = 63: none)
        const int len = (after ? __ffsll((long long)after) - 1 : cnt) - i;
        const bool is_long = len >= kLong;
        if (is_long) {
            const int q = atomicAdd(J.counters + 2, 1);
            if (q < J.long_cap) J.longs[q] = make_uint2((uint32_t)(beg + i), (uint32_t)len);
        }
        J.heads[base + __popcll(H & ((1ull << i) - 1))] =
            make_uint4((uint32_t)(v >> 32), (uint32_t)v, (uint32_t)(beg + i), is_long ? 0u : (uint32_t)len);
    }
}

// counting sort of g[0, cnt) (cnt <= kWarpCap) over rows [row0, row0 + R) (R <= 2^kWarpShift) by one warp.  Returns
// false, having written nothing, when a row has more than kRunMax contributions.
__device__ __forceinline__ bool warp_sort_counting(const DirectSortJob& J, uint64_t* g, int cnt, int beg, uint32_t row0,
                                                   int R, WarpSortSmem& S) {
    const int lane = threadIdx.x & 31;
    for (int r = lane; r < R; r += 32) S.hist[r] = 0;
    __syncwarp();
    for (int i = lane; i < cnt; i += 32) atomicAdd(&S.hist[(uint32_t)(g[i] >> 32) - row0], 1);
    __syncwarp();
    // lane owns rows [lane * RP, (lane + 1) * RP): longest row, touched rows, then an exclusive scan across the warp
    const int RP = (R + 31) >> 5;
    int local = 0, mx = 0, rows = 0;
    for (int x = 0; x < RP; ++x) {
        const int r = lane * RP + x;
        if (r < R) {
            const int c = S.hist[r];
            local += c;
            mx = max(mx, c);
            rows += c > 0 ? 1 : 0;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(B2R_FULL_MASK, mx, o));
    int inc = local, rinc = rows;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(B2R_FULL_MASK, inc, o), z = __shfl_up_sync(B2R_FULL_MASK, rinc, o);
        if (lane >= o) {
            inc += y;
            rinc += z;
        }
    }
    if (mx > kRunMax) return false;                      // same value in every lane
    int run = inc - local;
    for (int x = 0; x < RP; ++x) {
        const int r = lane * RP + x;
        if (r < R) {
            const int c = S.hist[r];
            S.hist[r] = run;                             // start of row r; the scatter below moves it to the row's end
            run += c;
        }
    }
    int base = 0;
    if (lane == 31) base = atomicAdd(J.counters + 3, rinc);   // rinc of lane 31: the bucket's touched rows
    base = __shfl_sync(B2R_FULL_MASK, base, 31);
    __syncwarp();
    for (int i = lane; i < cnt; i += 32) {
        const uint64_t v = g[i];
        S.s[atomicAdd(&S.hist[(uint32_t)(v >> 32) - row0], 1)] = v;
    }
    __syncwarp();
    // row r now spans [hist[r - 1], hist[r]); rows in chunks of 32 (lane = row), heads in ascending row order
    for (int r0 = 0; r0 < R; r0 += 32) {
        const int r = r0 + lane;
        const int a = r < R ? (r ? S.hist[r - 1] : 0) : 0, b = r < R ? S.hist[r] : 0;
        for (int x = a + 1; x < b; ++x) {                // insertion sort of the row's run by (row, position)
            const uint64_t val = S.s[x];
            int y = x - 1;
            while (y >= a && S.s[y] > val) {
                S.s[y + 1] = S.s[y];
                --y;
            }
            S.s[y + 1] = val;
        }
        const unsigned m = __ballot_sync(B2R_FULL_MASK, b > a);
        if (b > a)
            J.heads[base + __popc(m & ((1u << lane) - 1))] =
                make_uint4(row0 + (uint32_t)r, (uint32_t)S.s[a], (uint32_t)(beg + a), (uint32_t)(b - a));
        base += __popc(m);
    }
    __syncwarp();
    for (int i = lane; i < cnt; i += 32) g[i] = S.s[i];
    __syncwarp();
    return true;
}

// warps of the launch walk the buckets of b (the small plan) and then a, kSortWarps * gridDim.x at a time.  At most 32
// registers a thread (16 CTAs' worth of an SM's register file): a resident sort CTA costs an SM a few percent of its
// registers and ~33 KB of shared memory.
__global__ void __launch_bounds__(kSortWarps * 32, 16)
k_bucket_sort_warp(const __grid_constant__ DirectSortJob a, const __grid_constant__ DirectSortJob b) {
    __shared__ WarpSortSmem smem[kSortWarps];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    WarpSortSmem& S = smem[wl];
    const int total = a.nb + b.nb;
    for (int q = (int)blockIdx.x * kSortWarps + wl; q < total; q += (int)gridDim.x * kSortWarps) {
        const bool in_b = q < b.nb;
        const DirectSortJob& J = in_b ? b : a;
        const int bk = in_b ? q : q - b.nb;
        int raw = 0;
        if (lane == 0) {
            raw = J.cursor[(int64_t)bk * kPadD];
            if (raw) J.cursor[(int64_t)bk * kPadD] = 0;  // left zero for the next plan
        }
        raw = __shfl_sync(B2R_FULL_MASK, raw, 0);
        if (raw == 0) continue;
        const int beg = bk * J.cap;
        if (raw <= kRegSort) {                           // cap >= 128: never an overflowed bucket
            warp_sort_small(J, J.region + beg, raw, beg);
            continue;
        }
        if (raw <= J.cap && raw <= kWarpCap && J.shift <= kWarpShift &&
            warp_sort_counting(J, J.region + beg, raw, beg, (uint32_t)bk << J.shift, 1 << J.shift, S))
            continue;
        if (lane == 0) J.deferred[atomicAdd(J.counters + 4, 1)] = make_int2(bk, raw);
    }
}

// the buckets the warp sort deferred, one CTA each; exits at once when there are none (the usual case).  all_buckets:
// every bucket of both plans instead, straight from the cursors (plans of a few buckets: one launch, no warp pass).
__global__ void __maxnreg__(64)
k_bucket_sort_deferred(const __grid_constant__ DirectSortJob a, const __grid_constant__ DirectSortJob b, int all_buckets) {
    const int nda = all_buckets ? a.nb : a.counters[4], ndb = all_buckets ? b.nb : b.nb ? b.counters[4] : 0;
    if (nda + ndb == 0) return;
    __shared__ uint64_t s[kCap];
    __shared__ int head_cnt, head_base;
    __shared__ int hist[kCountRows + 1];
    __shared__ int scratch[40];
    __shared__ int sh[4];
    if (threadIdx.x == 0) head_cnt = 0;
    __syncthreads();
    for (int q = (int)blockIdx.x; q < nda + ndb; q += (int)gridDim.x) {
        if (all_buckets) {
            const DirectSortJob& J = q < nda ? a : b;
            const int bk = q < nda ? q : q - nda;
            if (threadIdx.x == 0) {
                sh[0] = J.cursor[(int64_t)bk * kPadD];
                J.cursor[(int64_t)bk * kPadD] = 0;
            }
            __syncthreads();
            const int raw = sh[0];
            __syncthreads();
            if (raw != 0) direct_sort_bucket(J, bk, raw, s, hist, scratch, &head_cnt, &head_base, sh);
        } else if (q < nda) {
            const int2 e = a.deferred[q];
            direct_sort_bucket(a, e.x, e.y, s, hist, scratch, &head_cnt, &head_base, sh);
        } else {
            const int2 e = b.deferred[q - nda];
            direct_sort_bucket(b, e.x, e.y, s, hist, scratch, &head_cnt, &head_base, sh);
        }
        __syncthreads();
    }
}

// One table's share of an apply launch: the sorted pairs and row heads of its plan, its contribution sources and
// the arrays to update.  `grid` CTAs of the launch work on it.
struct ApplyJob {
    const uint64_t* pairs;
    const uint4* heads;
    const int* n_heads;
    const int* n_long;
    const uint2* longs;
    int long_cap;
    int grid;
    BSrc s0, s1;
    float* W;
    float* M;
    float* V;
    float* dense;
    int* reset;                  // the plan's spill counter, zeroed here for the next step
};

// ---------------------------------------------------------------------------------------------------
// k_apply_sorted: one lane group per touched row (the head list written by the plan's sort): request the weight/state
// rows, sum the row's contributions in ascending position -- the first one is named by the head entry itself, so a
// row with a single contribution never reads the pair array -- and apply the update.  No barriers, no atomics.
// Rows with >= kLong contributions (listed by the sort; normally none) are then reduced by whole CTAs: contribution
// t goes to group t % GPC, partials are combined in group order -> deterministic.
// A launch can carry two jobs (two tables of one step): CTAs [0, a.grid) work on job a, the rest on job b, so a small
// table's update runs underneath a large one's instead of as a separate, latency-bound launch.
// ---------------------------------------------------------------------------------------------------
template <int LPR, int MODE>
__device__ __forceinline__ void apply_job(const ApplyJob& J, const OptK& opt, int bid, float4 (*part)[LPR]) {
    constexpr int D = LPR * 4;
    constexpr int GPC = kBT / LPR;
    const int sub = threadIdx.x % LPR, grp = threadIdx.x / LPR;
    const int sld = opt.state_ld ? opt.state_ld : D;
    const int n_heads = *J.n_heads;
    if (J.reset != nullptr && bid == 0 && threadIdx.x == 0) *J.reset = 0;
    for (int h = bid * GPC + grp; h < n_heads; h += J.grid * GPC) {
        const uint4 e = __ldg(J.heads + h);
        const int len = (int)e.w;
        if (len == 0) continue;                // long row: handled below
        const int64_t row = (int64_t)e.x;
        float4 w, m, v;
        if (MODE == 2) {
            w = ld4(J.W + row * D + sub * 4);
            if (opt.kind == 1) m = ld4(J.M + row * sld + sub * 4);
            if (opt.kind != 0) v = ld4(J.V + row * sld + sub * 4);
        } else {
            w = ld4(J.dense + row * D + sub * 4);
        }
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        uint32_t pos = e.y;
        for (int t = 0;;) {
            const float* base;
            int ld;
            int64_t r;
            float c;
            b_contribution(J.s0, J.s1, pos, base, ld, r, c);
            fma4(acc, c, ld4(base + r * ld + sub * 4));
            if (++t >= len) break;
            pos = (uint32_t)J.pairs[e.z + t];
        }
        RowIO<LPR>::template finish<MODE>(row, acc, sub, w, m, v, J.W, J.M, J.V, J.dense, opt);
    }
    const int n_long = min(*J.n_long, J.long_cap);
    for (int q = bid; q < n_long; q += J.grid) {
        const uint2 e = J.longs[q];
        const int j0 = (int)e.x, len = (int)e.y;
        const int64_t row = (int64_t)(J.pairs[j0] >> 32);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int t = grp; t < len; t += GPC) {
            const float* base;
            int ld;
            int64_t r;
            float c;
            b_contribution(J.s0, J.s1, (uint32_t)J.pairs[j0 + t], base, ld, r, c);
            fma4(acc, c, ld4(base + r * ld + sub * 4));
        }
        part[grp][sub] = acc;
        __syncthreads();
        if (grp == 0) {
            float4 tot = part[0][sub];
            for (int g2 = 1; g2 < GPC; ++g2) {
                const float4 y = part[g2][sub];
                tot.x += y.x; tot.y += y.y; tot.z += y.z; tot.w += y.w;
            }
            float4 w, m, v;
            if (MODE == 2) {
                w = ld4(J.W + row * D + sub * 4);
                if (opt.kind == 1) m = ld4(J.M + row * sld + sub * 4);
                if (opt.kind != 0) v = ld4(J.V + row * sld + sub * 4);
            } else {
                w = ld4(J.dense + row * D + sub * 4);
            }
            RowIO<LPR>::template finish<MODE>(row, tot, sub, w, m, v, J.W, J.M, J.V, J.dense, opt);
        }
        __syncthreads();
    }
}

template <int LPR, int MODE>
__global__ void __launch_bounds__(kBT)
k_apply_sorted(const __grid_constant__ ApplyJob a, const __grid_constant__ ApplyJob b, const __grid_constant__ OptK opt) {
    __shared__ float4 part[kBT / LPR][LPR];    // only touched when the batch has rows with >= kLong contributions
    OptK o = opt;
    optk_use_clock(o);
    if ((int)blockIdx.x < a.grid) apply_job<LPR, MODE>(a, o, (int)blockIdx.x, part);
    else apply_job<LPR, MODE>(b, o, (int)blockIdx.x - a.grid, part);
}

struct BucketGeom {
    int shift, nb;
};

static BucketGeom bucket_geom(int64_t n, int64_t n_rows) {
    int64_t target = n / 192;                      // ~192 pairs per bucket (measured: 128 equal, 96 and below slower) ...
    if (target < 256) target = n / 32;             // ... but at least a few hundred buckets for small batches
    if (target < 1) target = 1;
    if (target > 32768) target = 32768;
    int64_t rows_per = (n_rows + target - 1) / target;
    int shift = 0;
    while (((int64_t)1 << shift) < rows_per) ++shift;
    BucketGeom g;
    g.shift = shift;
    g.nb = (int)((n_rows + ((int64_t)1 << shift) - 1) >> shift);
    return g;
}

static BSrc to_bsrc(const b2r_grad_source* s, int d) {
    BSrc r{nullptr, nullptr, nullptr, 0, d, make_fastdiv(1)};
    if (s) {
        r.src = s->src;
        r.coef = s->coef;
        r.src_id = s->src_id;
        r.n = s->n;
        r.div = make_fastdiv(s->div < 1 ? 1u : (uint32_t)s->div);
        r.ld = s->ld > 0 ? s->ld : d;
    }
    return r;
}

// ---------------------------------------------------------------------------------------------------
// direct plans (plan_direct.cuh): layout, init, the producer's view, the sort launch, the apply job
// ---------------------------------------------------------------------------------------------------

struct DirectLayout {
    size_t cursor, region, big, tmp, spill, counters, longs, heads, deferred, total;
    int nb, shift, cap, big_cap, spill_cap, long_cap;
};

static DirectLayout direct_layout(int64_t n, int64_t n_rows) {
    const BucketGeom g = bucket_geom(n, n_rows);
    DirectLayout L;
    L.nb = g.nb;
    L.shift = g.shift;
    // region capacity: 3x the uniform share + slack, a multiple of 64, at most what one shared-memory sort takes;
    // more skew than that goes through the spill list
    int64_t cap = (3 * (n / (g.nb > 0 ? g.nb : 1)) + 64 + 63) / 64 * 64;
    if (cap < 128) cap = 128;
    if (cap > kCap) cap = kCap;
    L.cap = (int)cap;
    L.big_cap = (int)(2 * n);
    L.spill_cap = (int)n;
    L.long_cap = (int)(n / kLong + 1);
    size_t o = 0;
    auto take = [&](size_t bytes) {
        size_t r = o;
        o += align_up(bytes, 256);
        return r;
    };
    L.cursor = take((size_t)L.nb * 4 * kPadD);
    L.counters = take(256);
    L.region = take((size_t)L.nb * L.cap * 8);
    L.big = take((size_t)L.big_cap * 8);                   // directly behind the regions: one pair address space
    L.tmp = take((size_t)L.big_cap * 8);
    L.spill = take((size_t)L.spill_cap * 8);
    L.longs = take((size_t)L.long_cap * 8);
    L.heads = take((size_t)n * 16);
    L.deferred = take((size_t)L.nb * 8);
    L.total = o;
    return L;
}

static bool direct_ok(int64_t n, int64_t n_rows) {
    if (n <= 0 || n > 0x3fffffff || n_rows <= 0 || n_rows >= 0xffffffffLL) return false;
    const DirectLayout L = direct_layout(n, n_rows);
    return (int64_t)L.nb * L.cap + L.big_cap < 0x7fffffffLL && L.big == L.region + align_up((size_t)L.nb * L.cap * 8, 256)
           && ((size_t)L.nb * L.cap * 8) % 256 == 0;     // big must start exactly at pair index nb * cap
}

size_t direct_workspace_bytes(int64_t n, int64_t n_rows) {
    return direct_ok(n, n_rows) ? direct_layout(n, n_rows).total : 0;
}

int direct_workspace_init(void* ws, size_t ws_bytes, int64_t n, int64_t n_rows, cudaStream_t s) {
    B2R_REQUIRE(ws && direct_ok(n, n_rows), B2R_E_UNSUPPORTED, "direct plan: n=%lld n_rows=%lld unsupported", (long long)n,
                (long long)n_rows);
    const DirectLayout L = direct_layout(n, n_rows);
    B2R_REQUIRE(ws_bytes >= L.total, B2R_E_WORKSPACE, "direct plan: workspace %zu < %zu", ws_bytes, L.total);
    B2R_CUDA_OK(cudaMemsetAsync(static_cast<char*>(ws) + L.cursor, 0, L.region - L.cursor, s));   // cursors + counters
    return 0;
}

DirectPlanDev direct_plan_dev(void* ws, int64_t n, int64_t n_rows) {
    const DirectLayout L = direct_layout(n, n_rows);
    char* base = static_cast<char*>(ws);
    DirectPlanDev P;
    P.cursor = reinterpret_cast<int*>(base + L.cursor);
    P.region = reinterpret_cast<uint64_t*>(base + L.region);
    P.spill = reinterpret_cast<uint64_t*>(base + L.spill);
    P.counters = reinterpret_cast<int*>(base + L.counters);
    P.cap = L.cap;
    P.shift = L.shift;
    P.spill_cap = L.spill_cap;
    return P;
}

static DirectSortJob direct_sort_job_of(void* ws, int64_t n, int64_t n_rows) {
    const DirectLayout L = direct_layout(n, n_rows);
    char* base = static_cast<char*>(ws);
    DirectSortJob J;
    J.nb = L.nb; J.cap = L.cap; J.shift = L.shift;
    J.cursor = reinterpret_cast<int*>(base + L.cursor);
    J.region = reinterpret_cast<uint64_t*>(base + L.region);
    J.spill = reinterpret_cast<uint64_t*>(base + L.spill);
    J.counters = reinterpret_cast<int*>(base + L.counters);
    J.spill_cap = L.spill_cap;
    J.big = reinterpret_cast<uint64_t*>(base + L.big);
    J.tmp = reinterpret_cast<uint64_t*>(base + L.tmp);
    J.big_cap = L.big_cap;
    J.longs = reinterpret_cast<uint2*>(base + L.longs);
    J.long_cap = L.long_cap;
    J.heads = reinterpret_cast<uint4*>(base + L.heads);
    J.deferred = reinterpret_cast<int2*>(base + L.deferred);
    return J;
}

static int direct_scatter_pair_ex(const int64_t* ids_a, int64_t n_a, int64_t rows_a, void* ws_a, const int64_t* ids_b,
                                  int64_t n_b, int64_t rows_b, void* ws_b, int32_t* err_flag, int64_t ignore_id,
                                  int64_t ignore_n, int ctas, cudaStream_t s);

int direct_scatter_pair(const int64_t* ids_a, int64_t n_a, int64_t rows_a, void* ws_a, const int64_t* ids_b, int64_t n_b,
                        int64_t rows_b, void* ws_b, int32_t* err_flag, int ctas, cudaStream_t s) {
    return direct_scatter_pair_ex(ids_a, n_a, rows_a, ws_a, ids_b, n_b, rows_b, ws_b, err_flag, -1, 0, ctas, s);
}

static int direct_scatter_pair_ex(const int64_t* ids_a, int64_t n_a, int64_t rows_a, void* ws_a, const int64_t* ids_b,
                                  int64_t n_b, int64_t rows_b, void* ws_b, int32_t* err_flag, int64_t ignore_id,
                                  int64_t ignore_n, int ctas, cudaStream_t s) {
    B2R_REQUIRE(ids_a && ws_a && direct_ok(n_a, rows_a), B2R_E_BADARG, "direct_scatter_pair: bad plan a");
    const DirectPlanDev pa = direct_plan_dev(ws_a, n_a, rows_a);
    DirectPlanDev pb = pa;
    int64_t nb = 0;
    if (ids_b != nullptr && ws_b != nullptr) {
        B2R_REQUIRE(direct_ok(n_b, rows_b), B2R_E_BADARG, "direct_scatter_pair: bad plan b");
        pb = direct_plan_dev(ws_b, n_b, rows_b);
        nb = n_b;
    }
    const int cap = sm_count() * 8;
    int ga = (int)((n_a + kBT * 4 - 1) / (kBT * 4));
    if (ga > cap) ga = cap;
    if (ga < 1) ga = 1;
    int gb = nb > 0 ? (int)((nb + kBT * 4 - 1) / (kBT * 4)) : 0;
    if (gb > cap) gb = cap;
    if (ctas > 0 && ga + gb > ctas) {                    // bounded: split the CTAs in proportion to the pairs
        const int want_b = gb;
        gb = nb > 0 ? (int)((int64_t)ctas * nb / (n_a + nb)) : 0;
        if (want_b > 0 && gb < 1) gb = 1;
        ga = ctas - gb;
        if (ga < 1) ga = 1;
    }
    k_direct_scatter_pair<<<ga + gb, kBT, 0, s>>>(ids_a, n_a, rows_a, pa, ga, ids_b, nb, rows_b, pb, err_flag, ignore_id,
                                                  ignore_n);
    B2R_LAUNCH_OK("k_direct_scatter_pair");
    return 0;
}

// the warp sort takes (nearly) every bucket of a typical batch of this plan: its buckets fit a warp's histogram and
// slice, or they hold so few pairs on average (<= 3/4 of kRegSort) that the register sort takes all but a vanishing tail
static bool warp_takes_most(const DirectSortJob& J, int64_t n) {
    return (J.shift <= kWarpShift && J.cap <= kWarpCap) || n <= (int64_t)J.nb * (kRegSort * 3 / 4);
}

int direct_sort_pair(void* ws_a, int64_t n_a, int64_t rows_a, void* ws_b, int64_t n_b, int64_t rows_b, int ctas,
                     cudaStream_t s) {
    B2R_REQUIRE(ws_a && direct_ok(n_a, rows_a), B2R_E_BADARG, "direct_sort_pair: bad plan a");
    DirectSortJob a = direct_sort_job_of(ws_a, n_a, rows_a), b = a;
    b.nb = 0;
    if (ws_b != nullptr) {
        B2R_REQUIRE(direct_ok(n_b, rows_b), B2R_E_BADARG, "direct_sort_pair: bad plan b");
        b = direct_sort_job_of(ws_b, n_b, rows_b);
    }
    if (a.nb + b.nb <= sm_count()) {
        // a few buckets (small batches, e.g. BASELINE config 1): one CTA each in one launch -- the warp pass would only
        // add a launch to a step bound by launch latency
        k_bucket_sort_deferred<<<a.nb + b.nb, kBT, 0, s>>>(a, b, 1);
        B2R_LAUNCH_OK("k_bucket_sort_deferred");
        return 0;
    }
    // a warp per bucket (ctas = 0: as many warps as buckets); the buckets of the small plan come first
    int grid = (a.nb + b.nb + kSortWarps - 1) / kSortWarps;
    if (ctas > 0 && grid > ctas) grid = ctas;
    k_bucket_sort_warp<<<grid, kSortWarps * 32, 0, s>>>(a, b);
    B2R_LAUNCH_OK("k_bucket_sort_warp");
    // deferred buckets: normally none, and the launch's CTAs exit at once.  Plans whose buckets are mostly beyond the
    // warp sort (too wide and too full, e.g. 8,192-row buckets of ~340 pairs) defer nearly all of them: those get a grid
    // sized to their buckets, as the CTA sort always had.
    int dgrid = sm_count();
    if (ctas > 0 && dgrid > ctas) dgrid = ctas;
    if (!warp_takes_most(a, n_a) || (b.nb && !warp_takes_most(b, n_b))) dgrid = min(a.nb + b.nb, sm_count() * 8);
    k_bucket_sort_deferred<<<dgrid, kBT, 0, s>>>(a, b, 0);
    B2R_LAUNCH_OK("k_bucket_sort_deferred");
    return 0;
}

// fills one job from the C-ABI arguments (validated); grid = CTAs it gets
static int make_job(const b2r_apply_job* j, int d, int mode, const b2r_optim& o, int grid_cap, ApplyJob* out) {
    B2R_REQUIRE(j->ws && j->s0 && j->s0->src, B2R_E_BADARG, "direct apply: null pointer");
    B2R_REQUIRE(j->s0->n + (j->s1 ? j->s1->n : 0) == j->n, B2R_E_BADARG, "direct apply: sources do not cover the plan");
    if (mode == 1) {
        B2R_REQUIRE(j->dense, B2R_E_BADARG, "direct apply: mode 1 needs dense");
    } else {
        B2R_REQUIRE(j->W, B2R_E_BADARG, "direct apply: mode 2 needs W");
        B2R_REQUIRE(o.kind != 1 || (j->m && j->v), B2R_E_BADARG, "direct apply: Adam needs m and v");
        B2R_REQUIRE(o.kind != 2 || j->v, B2R_E_BADARG, "direct apply: Adagrad needs v");
    }
    B2R_REQUIRE(direct_ok(j->n, j->n_rows), B2R_E_UNSUPPORTED, "direct apply: n=%lld n_rows=%lld unsupported",
                (long long)j->n, (long long)j->n_rows);
    const DirectLayout L = direct_layout(j->n, j->n_rows);
    const char* base = static_cast<const char*>(j->ws);
    int* counters = reinterpret_cast<int*>(const_cast<char*>(base) + L.counters);
    out->pairs = reinterpret_cast<const uint64_t*>(base + L.region);       // regions, then the big area: one index space
    out->heads = reinterpret_cast<const uint4*>(base + L.heads);
    out->n_heads = counters + 3;
    out->n_long = counters + 2;
    out->longs = reinterpret_cast<const uint2*>(base + L.longs);
    out->long_cap = L.long_cap;
    out->s0 = to_bsrc(j->s0, d);
    out->s1 = to_bsrc(j->s1, d);
    out->W = j->W; out->M = j->m; out->V = j->v; out->dense = j->dense;
    out->reset = counters;                                                  // spill count -> 0 for the next step
    const int gpc = kBT / (d / 4);
    int64_t need = (j->n + gpc - 1) / gpc;
    if (need > grid_cap) need = grid_cap;
    out->grid = (int)(need < 1 ? 1 : need);
    return 0;
}

int direct_apply_pair(const b2r_apply_job* ja, const b2r_apply_job* jb, int d, int mode, const b2r_optim* opt, cudaStream_t s) {
    B2R_REQUIRE(ja, B2R_E_BADARG, "direct apply: null job");
    B2R_REQUIRE(d == 32 || d == 64 || d == 128, B2R_E_UNSUPPORTED, "direct apply: d=%d (have 32, 64, 128)", d);
    B2R_REQUIRE(mode == 1 || mode == 2, B2R_E_BADARG, "direct apply: mode %d (1 = dense +=, 2 = optimizer)", mode);
    b2r_optim o{};
    if (mode == 2) {
        B2R_REQUIRE(opt, B2R_E_BADARG, "direct apply: mode 2 needs opt");
        o = *opt;
        B2R_REQUIRE(o.kind >= 0 && o.kind <= 2, B2R_E_BADARG, "direct apply: optimizer kind %d", o.kind);
    }
    ApplyJob a{}, b{};
    const int cap = sm_count() * 16;             // ~2.7 waves of 6 resident CTAs/SM; x12 and x20 measured slower
    int rc = make_job(ja, d, mode, o, cap, &a);
    if (rc != 0) return rc;
    if (jb != nullptr) {
        // the second job is the small one by convention; its CTAs come first in the grid so that they are placed at once
        rc = make_job(jb, d, mode, o, cap, &b);
        if (rc != 0) return rc;
    } else {
        b = a;
        b.grid = 0;
    }
    const OptK ok = make_optk(o);
    const int grid = a.grid + b.grid;
#define B2R_BK(LPR, MODE) k_apply_sorted<LPR, MODE><<<grid, kBT, 0, s>>>(b.grid ? b : a, b.grid ? a : b, ok)
    if (mode == 1) {
        if (d == 32) B2R_BK(8, 1); else if (d == 64) B2R_BK(16, 1); else B2R_BK(32, 1);
    } else {
        if (d == 32) B2R_BK(8, 2); else if (d == 64) B2R_BK(16, 2); else B2R_BK(32, 2);
    }
#undef B2R_BK
    B2R_LAUNCH_OK("k_apply_sorted");
    return 0;
}

}  // namespace b2r

using namespace b2r;

// ---- C ABI of the direct plans for callers outside a step context (the autograd nodes, the shard owners) -------------
extern "C" size_t b2r_direct_plan_workspace_bytes(int64_t n, int64_t n_rows) { return direct_workspace_bytes(n, n_rows); }

extern "C" int b2r_direct_plan_init(void* ws, size_t ws_bytes, int64_t n, int64_t n_rows, b2r_stream_t stream) {
    return direct_workspace_init(ws, ws_bytes, n, n_rows, as_stream(stream));
}

extern "C" int b2r_direct_plan_build(const int64_t* ids, int64_t n, int64_t n_rows, int64_t ignore_id, int64_t ignore_n,
                                     void* ws, size_t ws_bytes, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(ids && ws, B2R_E_BADARG, "b2r_direct_plan_build: null pointer");
    const size_t need = direct_workspace_bytes(n, n_rows);
    B2R_REQUIRE(need != 0, B2R_E_UNSUPPORTED, "b2r_direct_plan_build: n=%lld n_rows=%lld unsupported", (long long)n,
                (long long)n_rows);
    B2R_REQUIRE(ws_bytes >= need, B2R_E_WORKSPACE, "b2r_direct_plan_build: workspace %zu < %zu", ws_bytes, need);
    cudaStream_t s = as_stream(stream);
    // a plan that was built but never applied leaves its spill counter set: clear the five counters here
    const DirectPlanDev P = direct_plan_dev(ws, n, n_rows);
    B2R_CUDA_OK(cudaMemsetAsync(P.counters, 0, 20, s));
    int rc = direct_scatter_pair_ex(ids, n, n_rows, ws, nullptr, 0, 0, nullptr, err_flag, ignore_id, ignore_n, 0, s);
    if (rc != 0) return rc;
    return direct_sort_pair(ws, n, n_rows, nullptr, 0, 0, 0, s);
}

extern "C" int b2r_direct_plan_apply(const void* ws, int64_t n, int64_t n_rows, int d, const b2r_grad_source* s0,
                                     const b2r_grad_source* s1, int mode, float* dense, float* W, float* m, float* v,
                                     const b2r_optim* opt, b2r_stream_t stream) {
    const b2r_apply_job j{ws, n, n_rows, s0, s1, dense, W, m, v};
    return direct_apply_pair(&j, nullptr, d, mode, opt, as_stream(stream));
}
