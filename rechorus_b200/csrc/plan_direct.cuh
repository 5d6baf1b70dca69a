// plan_direct.cuh -- the "direct" index plan of a table's row-sparse update (bucket.cu; used by the step context of
// bprmf_step.cu and by the b2r_direct_plan_* entry points).  One scatter launch drops each (row, position) pair of the
// batch into the bucket of its row range: fixed-capacity bucket regions, one L2 atomic per pair on a line-padded cursor,
// pairs beyond a region's capacity (skewed batches) into a spill list.  The sort then orders every bucket -- a warp per
// bucket (k_bucket_sort_warp), a CTA for the few it defers (k_bucket_sort_deferred) -- and lists the row heads for
// k_apply_sorted.  Every launch can carry two tables.
#pragma once
#include "common.cuh"

namespace b2r {

constexpr int kPadD = 32;                 // ints per bucket cursor: one 128-byte line each (L2 atomics serialise per line)

struct DirectPlanDev {                    // what the scatter kernel needs
    int* cursor;                          // [nb * kPadD]
    uint64_t* region;                     // [nb][cap] pairs (row << 32 | position)
    uint64_t* spill;                      // [spill_cap] pairs that did not fit their region
    int* counters;                        // [0] spill count, [1] big-area cursor, [2] long rows, [3] row heads,
                                          // [4] buckets deferred to the CTA sort
    int cap, shift, spill_cap;
};

__device__ __forceinline__ void direct_scatter(const DirectPlanDev& P, uint32_t key, uint32_t pos) {
    const int b = (int)(key >> P.shift);
    const int slot = atomicAdd(&P.cursor[(int64_t)b * kPadD], 1);
    const uint64_t pair = ((uint64_t)key << 32) | (uint64_t)pos;
    if (slot < P.cap) {
        P.region[(int64_t)b * P.cap + slot] = pair;
    } else {
        const int s = atomicAdd(&P.counters[0], 1);
        if (s < P.spill_cap) P.spill[s] = pair;
    }
}

size_t direct_workspace_bytes(int64_t n, int64_t n_rows);
int direct_workspace_init(void* ws, size_t ws_bytes, int64_t n, int64_t n_rows, cudaStream_t s);
DirectPlanDev direct_plan_dev(void* ws, int64_t n, int64_t n_rows);
// drop the pairs of one or two id arrays into their plans in ONE launch (the step context: the NEXT batch's ids on its
// side stream).  ctas > 0 bounds the launch to that many CTAs (a persistent grid looping over the pairs); 0 sizes it to
// the work.
int direct_scatter_pair(const int64_t* ids_a, int64_t n_a, int64_t rows_a, void* ws_a, const int64_t* ids_b, int64_t n_b,
                        int64_t rows_b, void* ws_b, int32_t* err_flag, int ctas, cudaStream_t s);
// sort every bucket of one or two plans (b may be NULL) and list their row heads: a warp per bucket in one launch, then
// one CTA per bucket the warps could not take in a second launch (empty for a typical batch); plans with at most one
// bucket per SM take the CTA sort in a single launch.  ctas > 0 bounds the launches as above.
int direct_sort_pair(void* ws_a, int64_t n_a, int64_t rows_a, void* ws_b, int64_t n_b, int64_t rows_b, int ctas,
                     cudaStream_t s);
// One table's share of an apply launch: its plan, the contribution sources, and the arrays to update (mode 1: dense +=;
// mode 2: W and the optimizer state m, v).
struct b2r_apply_job {
    const void* ws;              // the table's plan: a direct-plan workspace
    int64_t n, n_rows;
    const b2r_grad_source* s0;
    const b2r_grad_source* s1;   // optional second contribution stream (NULL: none)
    float* dense;                // mode 1
    float* W;                    // mode 2
    float* m;
    float* v;
};

// apply one or two tables' updates (jb may be NULL) in ONE launch.  The two updates must be independent -- neither job's
// sources may alias the other job's W -- e.g. the user and the item table of one BPRMF step, the item gradient reading a
// saved copy of the user rows.  The small table's update (jb) then runs underneath the large one's.
int direct_apply_pair(const b2r_apply_job* ja, const b2r_apply_job* jb, int d, int mode, const b2r_optim* opt, cudaStream_t s);

}  // namespace b2r
