// plan.cu -- index plan: stable radix sort of (row id, flat position) + run-head compaction.
//
// The reference's embedding backward (ATen embedding_dense_backward behind nn.Embedding, BPRMF.py:31-32)
// zero-fills a dense [n_rows, d] gradient and accumulates into it.  Here the ids of the batch are sorted once
// (keys only need ceil(log2 n_rows) bits: 20 for 1 M rows, 27 for 100 M) so that each touched row has a
// single owner that sums its contributions in ascending position order: no atomics, no zero-fill, and the
// unique-row list the row-sparse optimizer and the sharded exchange need falls out for free.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "common.cuh"

namespace b2r {

__global__ void __launch_bounds__(256)
k_plan_keys(const int64_t* __restrict__ ids, int64_t n, int64_t n_rows, uint32_t* __restrict__ key,
            uint32_t* __restrict__ pos, int32_t* err_flag, int64_t ignore_id, int64_t ignore_n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t id = ids[i];
        // positions [0, ignore_n) holding ignore_id contribute nothing (e.g. right-padding of a history): they
        // get the sentinel key n_rows, sort to the end, and the segment kernels skip rows >= n_rows
        key[i] = (i < ignore_n && id == ignore_id) ? (uint32_t)n_rows : (uint32_t)checked_id(id, n_rows, err_flag);
        pos[i] = (uint32_t)i;
    }
}

struct RunHead {
    const uint32_t* key;
    __host__ __device__ bool operator()(const int32_t& i) const { return i == 0 || key[i] != key[i - 1]; }
};

static int key_bits(int64_t n_rows) {     // keys are in [0, n_rows] (n_rows itself = the "ignored" sentinel)
    int bits = 1;
    while (bits < 32 && ((int64_t)1 << bits) <= n_rows) ++bits;
    return bits;
}

struct PlanLayout {
    size_t key_in, pos_in, cub_tmp, cub_bytes, total;
};

static int plan_layout(int64_t n, int64_t n_rows, PlanLayout* L) {
    size_t sort_bytes = 0, sel_bytes = 0;
    const int nn = (int)n;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, nn, 0,
                                                    key_bits(n_rows), (cudaStream_t)0);
    if (e != cudaSuccess) return set_error((int)e, "cub sort size query failed: %s", cudaGetErrorString(e));
    cub::CountingInputIterator<int32_t> counting(0);
    RunHead pred{nullptr};
    e = cub::DeviceSelect::If(nullptr, sel_bytes, counting, (int32_t*)nullptr, (int32_t*)nullptr, nn, pred,
                              (cudaStream_t)0);
    if (e != cudaSuccess) return set_error((int)e, "cub select size query failed: %s", cudaGetErrorString(e));
    L->key_in = 0;
    L->pos_in = align_up((size_t)n * sizeof(uint32_t), 256);
    L->cub_tmp = L->pos_in + align_up((size_t)n * sizeof(uint32_t), 256);
    L->cub_bytes = sort_bytes > sel_bytes ? sort_bytes : sel_bytes;
    L->total = L->cub_tmp + align_up(L->cub_bytes, 256);
    return 0;
}

}  // namespace b2r

using namespace b2r;

extern "C" size_t b2r_plan_workspace_bytes(int64_t n, int64_t n_rows) {
    if (n <= 0 || n > 0x7fffffff || n_rows <= 0) return 0;
    PlanLayout L;
    if (plan_layout(n, n_rows, &L) != 0) return 0;
    return L.total;
}

extern "C" int b2r_plan_build_ex(const int64_t* ids, int64_t n, int64_t n_rows, int64_t ignore_id, int64_t ignore_n,
                                 uint32_t* sorted_key, uint32_t* sorted_pos, int32_t* seg_start, int32_t* n_uniq,
                                 void* ws, size_t ws_bytes, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(ids && sorted_key && sorted_pos && seg_start && n_uniq && ws, B2R_E_BADARG,
                "b2r_plan_build_ex: null pointer");
    B2R_REQUIRE(n > 0 && n <= 0x7fffffff, B2R_E_BADARG, "b2r_plan_build_ex: n must be in [1, 2^31) (n=%lld)",
                (long long)n);
    B2R_REQUIRE(n_rows > 0 && n_rows < 0xffffffffLL, B2R_E_UNSUPPORTED,
                "b2r_plan_build_ex: n_rows must fit 32 bits (n_rows=%lld)", (long long)n_rows);
    PlanLayout L;
    int rc = plan_layout(n, n_rows, &L);
    if (rc != 0) return rc;
    B2R_REQUIRE(ws_bytes >= L.total, B2R_E_WORKSPACE, "b2r_plan_build_ex: workspace %zu < required %zu", ws_bytes,
                L.total);
    B2R_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, B2R_E_BADARG,
                "b2r_plan_build_ex: workspace must be 256-byte aligned");
    cudaStream_t s = as_stream(stream);
    char* base = static_cast<char*>(ws);
    uint32_t* key_in = reinterpret_cast<uint32_t*>(base + L.key_in);
    uint32_t* pos_in = reinterpret_cast<uint32_t*>(base + L.pos_in);
    void* cub_tmp = base + L.cub_tmp;
    const int nn = (int)n;

    int grid = (int)((n + 255) / 256);
    const int cap = sm_count() * 8;
    if (grid > cap) grid = cap;
    k_plan_keys<<<grid, 256, 0, s>>>(ids, n, n_rows, key_in, pos_in, err_flag, ignore_id, ignore_n);
    B2R_LAUNCH_OK("k_plan_keys");

    size_t tmp_bytes = L.cub_bytes;
    B2R_CUDA_OK(cub::DeviceRadixSort::SortPairs(cub_tmp, tmp_bytes, (const uint32_t*)key_in, sorted_key,
                                                (const uint32_t*)pos_in, sorted_pos, nn, 0, key_bits(n_rows), s));
    count_launch();
    cub::CountingInputIterator<int32_t> counting(0);
    RunHead pred{sorted_key};
    tmp_bytes = L.cub_bytes;
    B2R_CUDA_OK(cub::DeviceSelect::If(cub_tmp, tmp_bytes, counting, seg_start, n_uniq, nn, pred, s));
    count_launch();
    return 0;
}
