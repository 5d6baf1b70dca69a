// impression.cu -- evaluation of the impression models (SURVEY.md §8 row f4, `--model_mode Impression`) on the device:
// the batches of ImpressionModel.Dataset (models/BaseImpressionModel.py:152-184) and the metrics of
// ImpressionRunner.evaluate + evaluate_method (helpers/ImpressionRunner.py:135-171, :74-133), so neither one feed dict
// per impression nor the [N, mp + mn] prediction matrix has to exist on the host.
//
//   k_collate_impression   item_id[t] = [pos[:mp] | 0-pad to mp | neg[:mn] | 0-pad to mn] of phase row
//                          perm[start + t] (start + t without a permutation), from a CSR of the (truncated) positive and
//                          negative lists; user_id[t] = users[row]; for a training batch also ImpressionRunner.fit's
//                          labels (helpers/ImpressionRunner.py:186-189) from the row's pos_num / neg_num
//   k_impression_metrics   one warp per row: the row's float64 sort keys staged in shared memory, every valid positive
//                          ranked by counting the columns the reference's stable argsort puts before it, NDCG / MAP / HR
//                          for every cut-off from those ranks, per-CTA sums, and a last-CTA pass that adds the CTA sums
//                          in CTA order into the caller's accumulator
//
// Why counting is enough (include/b200rec.h has the full restatement): the reference's metrics depend on the sorted
// label row only through the sorted positions of its positives, and a positive's sorted position is the number of
// columns that precede it under the sort's comparator.  Lists are tens to a few hundred long, so the O(P * C) count per
// row costs less than staging the row.  Every sum has a fixed order (lane order inside a warp, warp order inside a CTA,
// CTA order in the final pass), so the result depends on the inputs only and two calls give identical bits.
#include "common.cuh"

namespace b2r {

constexpr int kImpMaxTopk = B2R_IMPRESSION_MAX_TOPK;
constexpr int kImpMaxWarps = 8;                 // rows (warps) per CTA when the staged rows fit 48 KB
constexpr size_t kImpSmemDefault = 48 * 1024;
constexpr size_t kImpSmemMax = 227 * 1024;      // sm_90 opt-in limit of dynamic shared memory per CTA

struct ImpTopk {
    int k[kImpMaxTopk];
};

// shared memory of one warp: C float64 keys, C int32 ranks (only the first mp are used), 3 * kImpMaxTopk row values
__host__ __device__ __forceinline__ size_t imp_rank_bytes(int C) { return ((size_t)C * 4 + 7) / 8 * 8; }
__host__ __device__ __forceinline__ size_t imp_warp_bytes(int C) {
    return (size_t)C * 8 + imp_rank_bytes(C) + (size_t)3 * kImpMaxTopk * 8;
}

// rows per CTA: a function of C alone, so the CTA partition (and with it the summation order) never depends on Bn
static inline int imp_warps(int C) {
    const size_t w = imp_warp_bytes(C);
    int n = (int)(kImpSmemDefault / w);
    return n < 1 ? 1 : (n > kImpMaxWarps ? kImpMaxWarps : n);
}

// One phase batch: rows perm[start + t] (perm NULL: start + t) for t < Bn.  Row `row` has the positive list
// pos_items[pos_ptr[row] .. pos_ptr[row + 1]) and the negative list neg_items[neg_ptr[row] .. neg_ptr[row + 1]);
// only their first mp / mn entries are read, as the slices target_item[:pos_len] / neg_items[:neg_len] of
// _get_feed_dict take them, and the rest of each half is 0 as collate_batch pads it.  With out_lab (a training batch),
// label[t, c] = c < min(pos_num[row], mp) ? 1 : -1 for c < mp and c - mp < min(neg_num[row], mn) ? 0 : -1 after it.
__global__ void __launch_bounds__(256)
k_collate_impression(const int64_t* __restrict__ users, const int64_t* __restrict__ pos_ptr,
                     const int64_t* __restrict__ pos_items, const int64_t* __restrict__ neg_ptr,
                     const int64_t* __restrict__ neg_items, const int64_t* __restrict__ pos_num,
                     const int64_t* __restrict__ neg_num, const int64_t* __restrict__ perm, int64_t n_users,
                     int64_t start, int Bn, int mp, int mn, int64_t* __restrict__ out_uid, int64_t* __restrict__ out_iid,
                     int64_t* __restrict__ out_lab, int32_t* __restrict__ err_flag) {
    const int C = mp + mn;
    const int64_t total = (int64_t)Bn * C;
    for (int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 256) {
        const int t = (int)(idx / C), c = (int)(idx - (int64_t)t * C);
        const int64_t row = perm ? perm[start + t] : start + t;
        if (c == 0) {
            int64_t u = users[row];
            if (u < 0 || u >= n_users) {
                if (err_flag) atomicAdd(err_flag, 1);
                u = 0;
            }
            out_uid[t] = u;
        }
        int64_t v = 0, lab = -1;
        if (c < mp) {
            const int64_t b = pos_ptr[row];
            if (c < pos_ptr[row + 1] - b) v = pos_items[b + c];
            if (out_lab && c < min(pos_num[row], (int64_t)mp)) lab = 1;
        } else {
            const int64_t b = neg_ptr[row];
            if (c - mp < neg_ptr[row + 1] - b) v = neg_items[b + (c - mp)];
            if (out_lab && c - mp < min(neg_num[row], (int64_t)mn)) lab = 0;
        }
        out_iid[idx] = v;
        if (out_lab) out_lab[idx] = lab;
    }
}

// Column c precedes column j in the reference's order: (-key).argsort(kind='mergesort') sorts keys descending, keeps
// ties in column order, and puts NaN after everything (NaNs among themselves in column order).  -0.0 == +0.0.
__device__ __forceinline__ bool imp_before(double kc, int c, double kj, int j) {
    const bool nan_c = isnan(kc), nan_j = isnan(kj);
    if (nan_j) return !nan_c || c < j;
    if (nan_c) return false;
    return kc > kj || (kc == kj && c < j);
}

__global__ void __launch_bounds__(kImpMaxWarps * 32)
k_impression_metrics(const float* __restrict__ pred, int64_t ld, int Bn, int C, int mp,
                     const int64_t* __restrict__ pos_num, const int64_t* __restrict__ neg_num, ImpTopk tk, int nk,
                     unsigned int* __restrict__ counter, double* __restrict__ partials, double* __restrict__ acc) {
    extern __shared__ __align__(16) unsigned char imp_smem[];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int nv = 3 * nk;
    unsigned char* base = imp_smem + (size_t)warp * imp_warp_bytes(C);
    double* keys = reinterpret_cast<double*>(base);
    int* rnk = reinterpret_cast<int*>(base + (size_t)C * 8);
    double* vals = reinterpret_cast<double*>(base + (size_t)C * 8 + imp_rank_bytes(C));
    const int64_t row = (int64_t)blockIdx.x * nw + warp;

    if (row < Bn) {
        // pos_num / neg_num are the raw data columns; evaluate() clips them to the list widths (:162-166, :110-113)
        const int64_t pn = pos_num[row], nn = neg_num[row];
        const int pc = (int)(pn < 0 ? 0 : (pn > mp ? mp : pn));
        const int nc = (int)(nn < 0 ? 0 : (nn > C - mp ? C - mp : nn));
        const int W = pc + nc;                                         // whole_len
        const float* p = pred + row * ld;
        // keys: the masked prediction (invalid slots -inf, :167) promoted to float64, minus eps on the first mp
        // columns (:97-101).  -inf - 1e-6 stays -inf and NaN stays NaN, as in NumPy.
        for (int c = lane; c < C; c += 32) {
            const bool valid = c < pc || (c >= mp && c < mp + nc);
            const double x = valid ? (double)p[c] : -INFINITY;
            keys[c] = c < mp ? x - 1e-6 : x;
        }
        __syncwarp();
        // sorted position of every valid positive: the columns that precede it (all are counted, valid or not)
        for (int j = lane; j < pc; j += 32) {
            const double kj = keys[j];
            int r = 0;
            for (int c = 0; c < C; ++c) r += imp_before(keys[c], c, kj, j) ? 1 : 0;
            rnk[j] = r;
        }
        __syncwarp();
        // labels at sorted positions >= whole_len are zeroed (:20, :36, :55), so only positives with r < W count;
        // P = how many there are.  A counted positive's label prefix sum (AP's precision numerator) is 1 + the
        // number of counted positives before it; positions are distinct, so that is #{q : r_q < r}.
        double dcg[kImpMaxTopk], ap[kImpMaxTopk];
        bool hit[kImpMaxTopk];
#pragma unroll
        for (int i = 0; i < kImpMaxTopk; ++i) { dcg[i] = 0.0; ap[i] = 0.0; hit[i] = false; }
        int P = 0;
        for (int j = lane; j < pc; j += 32) {
            const int r = rnk[j];
            if (r >= W) continue;
            ++P;
            int m = 1;
            for (int q = 0; q < pc; ++q) m += rnk[q] < r ? 1 : 0;
            const double g = 1.0 / log2((double)(r + 2));
            const double a = (double)m / (double)(r + 1);
#pragma unroll
            for (int i = 0; i < kImpMaxTopk; ++i) {
                if (i < nk && r < tk.k[i]) { dcg[i] += g; ap[i] += a; hit[i] = true; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) P += __shfl_xor_sync(B2R_FULL_MASK, P, o);
#pragma unroll
        for (int i = 0; i < kImpMaxTopk; ++i) {
            if (i < nk) {                                              // nk is uniform across the warp
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    dcg[i] += __shfl_xor_sync(B2R_FULL_MASK, dcg[i], o);
                    ap[i] += __shfl_xor_sync(B2R_FULL_MASK, ap[i], o);
                }
                hit[i] = __any_sync(B2R_FULL_MASK, hit[i]);
            }
        }
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < kImpMaxTopk; ++i) {
                if (i < nk) {
                    const int k = tk.k[i];
                    const int lim = P < k ? P : k;
                    double idcg = 0.0;                                 // ideal DCG: the P ones sorted to the front
                    for (int t = 0; t < lim; ++t) idcg += 1.0 / log2((double)(t + 2));
                    if (idcg == 0.0) idcg = 1.0;
                    const int pnum = P < 1 ? 1 : (P > k ? k : P);      // positive_num of AP_at_k
                    vals[i] = dcg[i] / idcg;
                    vals[nk + i] = ap[i] / (double)pnum;
                    vals[2 * nk + i] = hit[i] ? 1.0 : 0.0;
                }
            }
        }
    } else if (lane == 0) {
        for (int v = 0; v < nv; ++v) vals[v] = 0.0;
    }
    __syncthreads();
    // this CTA's sums, warps (rows) in order
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
        double s = 0.0;
        for (int w = 0; w < nw; ++w)
            s += reinterpret_cast<const double*>(imp_smem + (size_t)w * imp_warp_bytes(C) + (size_t)C * 8 +
                                                 imp_rank_bytes(C))[v];
        partials[(size_t)blockIdx.x * nv + v] = s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // the last CTA: one warp per value, lane l sums CTAs l, l + 32, ... in order, then a fixed butterfly
    for (int v = warp; v < nv; v += nw) {
        double s = 0.0;
        for (unsigned int b = lane; b < gridDim.x; b += 32) s += __ldcg(partials + (size_t)b * nv + v);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(B2R_FULL_MASK, s, o);
        if (lane == 0) acc[v] += s;
    }
    if (threadIdx.x == 0) *counter = 0u;                               // ready for the next call on this workspace
}

}  // namespace b2r

using namespace b2r;

static int collate_impression(const char* name, const int64_t* users, const int64_t* pos_ptr, const int64_t* pos_items,
                              const int64_t* neg_ptr, const int64_t* neg_items, const int64_t* pos_num,
                              const int64_t* neg_num, const int64_t* perm, int64_t n_users, int64_t start, int Bn, int mp,
                              int mn, int64_t* out_uid, int64_t* out_iid, int64_t* out_lab, int32_t* err_flag,
                              b2r_stream_t stream) {
    B2R_REQUIRE(users && pos_ptr && pos_items && neg_ptr && neg_items && out_uid && out_iid, B2R_E_BADARG,
                "%s: null pointer", name);
    B2R_REQUIRE(Bn >= 0 && start >= 0 && mp >= 0 && mn >= 0 && mp + mn >= 1 && n_users >= 1, B2R_E_BADARG,
                "%s: Bn=%d start=%lld mp=%d mn=%d n_users=%lld", name, Bn, (long long)start, mp, mn,
                (long long)n_users);
    if (Bn == 0) return 0;
    const int64_t total = (int64_t)Bn * (mp + mn);
    int64_t grid = (total + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    k_collate_impression<<<(int)grid, 256, 0, as_stream(stream)>>>(users, pos_ptr, pos_items, neg_ptr, neg_items, pos_num,
                                                                   neg_num, perm, n_users, start, Bn, mp, mn, out_uid,
                                                                   out_iid, out_lab, err_flag);
    B2R_LAUNCH_OK("k_collate_impression");
    return 0;
}

extern "C" int b2r_collate_impression(const int64_t* users, const int64_t* pos_ptr, const int64_t* pos_items,
                                      const int64_t* neg_ptr, const int64_t* neg_items, int64_t n_users, int64_t start,
                                      int Bn, int mp, int mn, int64_t* out_uid, int64_t* out_iid, int32_t* err_flag,
                                      b2r_stream_t stream) {
    return collate_impression("b2r_collate_impression", users, pos_ptr, pos_items, neg_ptr, neg_items, nullptr, nullptr,
                              nullptr, n_users, start, Bn, mp, mn, out_uid, out_iid, nullptr, err_flag, stream);
}

extern "C" int b2r_collate_impression_train(const int64_t* users, const int64_t* pos_ptr, const int64_t* pos_items,
                                            const int64_t* neg_ptr, const int64_t* neg_items, const int64_t* pos_num,
                                            const int64_t* neg_num, const int64_t* perm, int64_t n_users, int64_t start,
                                            int Bn, int mp, int mn, int64_t* out_uid, int64_t* out_iid,
                                            int64_t* out_labels, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(pos_num && neg_num && out_labels, B2R_E_BADARG, "b2r_collate_impression_train: null pointer");
    return collate_impression("b2r_collate_impression_train", users, pos_ptr, pos_items, neg_ptr, neg_items, pos_num,
                              neg_num, perm, n_users, start, Bn, mp, mn, out_uid, out_iid, out_labels, err_flag, stream);
}

extern "C" size_t b2r_impression_metrics_workspace_bytes(int Bn, int C, int nk) {
    if (Bn <= 0 || C < 1 || nk < 1 || nk > kImpMaxTopk) return 0;
    const int64_t grid = ((int64_t)Bn + imp_warps(C) - 1) / imp_warps(C);
    return 16 + (size_t)grid * 3 * nk * sizeof(double);
}

extern "C" int b2r_impression_metrics(const float* pred, int64_t ld, int Bn, int C, int mp, const int64_t* pos_num,
                                      const int64_t* neg_num, const int* topk, int nk, double* acc, void* workspace,
                                      size_t workspace_bytes, b2r_stream_t stream) {
    B2R_REQUIRE(pred && pos_num && neg_num && topk && acc && workspace, B2R_E_BADARG,
                "b2r_impression_metrics: null pointer");
    B2R_REQUIRE(Bn >= 0 && C >= 1 && mp >= 0 && mp <= C && ld >= C, B2R_E_BADARG,
                "b2r_impression_metrics: Bn=%d C=%d mp=%d ld=%lld", Bn, C, mp, (long long)ld);
    B2R_REQUIRE(nk >= 1 && nk <= kImpMaxTopk, B2R_E_UNSUPPORTED,
                "b2r_impression_metrics: %d cut-offs, at most %d are supported", nk, kImpMaxTopk);
    ImpTopk tk = {};
    for (int i = 0; i < nk; ++i) {
        B2R_REQUIRE(topk[i] >= 1, B2R_E_BADARG, "b2r_impression_metrics: cut-off %d is %d", i, topk[i]);
        tk.k[i] = topk[i];
    }
    const int nw = imp_warps(C);
    const size_t smem = (size_t)nw * imp_warp_bytes(C);
    B2R_REQUIRE(smem <= kImpSmemMax, B2R_E_UNSUPPORTED,
                "b2r_impression_metrics: C=%d candidates do not fit one warp's shared memory", C);
    if (Bn == 0) return 0;
    B2R_REQUIRE(workspace_bytes >= b2r_impression_metrics_workspace_bytes(Bn, C, nk), B2R_E_WORKSPACE,
                "b2r_impression_metrics: workspace of %zu bytes, %zu needed", workspace_bytes,
                b2r_impression_metrics_workspace_bytes(Bn, C, nk));
    if (smem > kImpSmemDefault)
        B2R_CUDA_OK(cudaFuncSetAttribute(k_impression_metrics, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t grid = ((int64_t)Bn + nw - 1) / nw;
    unsigned int* counter = reinterpret_cast<unsigned int*>(workspace);
    double* partials = reinterpret_cast<double*>(static_cast<unsigned char*>(workspace) + 16);
    k_impression_metrics<<<(unsigned)grid, nw * 32, smem, as_stream(stream)>>>(pred, ld, Bn, C, mp, pos_num, neg_num, tk,
                                                                              nk, counter, partials, acc);
    B2R_LAUNCH_OK("k_impression_metrics");
    return 0;
}
