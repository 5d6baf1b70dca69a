// rec_csv.cu -- the rows of save_rec_results' CSV (main.py:117-132, TopK branch) assembled on the device.
//
// A row is "<user><sep><items cell><sep><scores cell>\n": the user a plain decimal in both styles (pandas prints an
// int64 column), a cell "[" + ", ".join(repr(e)) + "]" with NumPy's scalar repr (rec_format.cuh), and a field wrapped
// in '"' exactly when it contains the separator (pandas' QUOTE_MINIMAL; the texts never contain '"', '\r' or '\n', so
// nothing is escaped).  Two passes, one warp per row:
//   1. k_rec_csv_measure formats every field, stores the row's byte length and its three quote flags;
//   2. an exclusive scan of the lengths gives each row's offset (cub::DeviceScan);
//   3. k_rec_csv_write formats the fields again and writes them at the row's offset.
// Every byte's position is a function of the inputs alone, so the text does not depend on scheduling.
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "rec_format.cuh"

namespace b2r {

constexpr int kRowsPerCta = 8;      // one warp per row
constexpr int kMaxK = 1 << 16;

__device__ __forceinline__ bool contains(const char* t, int n, char c) {
    bool hit = false;
    for (int i = 0; i < n; ++i) hit |= t[i] == c;
    return hit;
}

__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(B2R_FULL_MASK, v, o);
    return v;
}

// one list cell's element texts: their total length and whether one contains sep
template <bool FLOAT>
__device__ __forceinline__ void measure_cell(const void* row, int k, int style, char sep, int lane, int& len, bool& quote) {
    char t[recfmt::kMaxText];
    int sum = 0;
    bool hit = false;
    for (int j = lane; j < k; j += 32) {
        const int n = FLOAT ? recfmt::format_f32(__float_as_uint(static_cast<const float*>(row)[j]), style, t)
                            : recfmt::format_i64(static_cast<const int64_t*>(row)[j], style, t);
        sum += n;
        hit |= contains(t, n, sep);
    }
    len = warp_sum_int(sum);
    quote = __any_sync(B2R_FULL_MASK, hit);
}

// writes one list cell at o (quoted when quote); returns its length.  Element j starts after the texts and ", "
// separators of elements 0..j-1: a warp prefix sum per group of 32 elements.
template <bool FLOAT>
__device__ __forceinline__ int64_t write_cell(char* o, const void* row, int k, int style, bool quote, int lane) {
    char t[recfmt::kMaxText];
    int64_t p = 0;
    if (lane == 0) {
        if (quote) o[0] = '"';
        o[quote ? 1 : 0] = '[';
    }
    p = quote ? 2 : 1;
    for (int j0 = 0; j0 < k; j0 += 32) {
        const int j = j0 + lane;
        int n = 0;
        if (j < k) {
            n = FLOAT ? recfmt::format_f32(__float_as_uint(static_cast<const float*>(row)[j]), style, t)
                      : recfmt::format_i64(static_cast<const int64_t*>(row)[j], style, t);
        }
        const int w = j < k ? n + (j + 1 < k ? 2 : 0) : 0;          // text and the ", " that follows it
        int incl = w;
#pragma unroll
        for (int o2 = 1; o2 < 32; o2 <<= 1) {
            const int v = __shfl_up_sync(B2R_FULL_MASK, incl, o2);
            if (lane >= o2) incl += v;
        }
        if (j < k) {
            char* d = o + p + (incl - w);
            for (int i = 0; i < n; ++i) d[i] = t[i];
            if (j + 1 < k) {
                d[n] = ',';
                d[n + 1] = ' ';
            }
        }
        p += __shfl_sync(B2R_FULL_MASK, incl, 31);
    }
    if (lane == 0) {
        o[p] = ']';
        if (quote) o[p + 1] = '"';
    }
    return p + 1 + (quote ? 1 : 0);
}

__device__ __forceinline__ bool cell_fixed_has(char sep, int k) {
    return sep == '[' || sep == ']' || (k >= 2 && (sep == ',' || sep == ' '));
}

__global__ void __launch_bounds__(kRowsPerCta * 32)
k_rec_csv_measure(const int64_t* __restrict__ users, const int64_t* __restrict__ items, const float* __restrict__ scores,
                  int64_t N, int k, int style, char sep, int64_t* __restrict__ lens, uint8_t* __restrict__ quotes) {
    const int lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0) lens[N] = 0;        // the scan's extra element: row_offsets[N] = total
    for (int64_t r = (int64_t)blockIdx.x * kRowsPerCta + (threadIdx.x >> 5); r < N;
         r += (int64_t)gridDim.x * kRowsPerCta) {
        char t[recfmt::kMaxText];
        const int un = recfmt::format_i64(users[r], B2R_REC_STYLE_BARE, t);
        const bool uq = contains(t, un, sep);
        int il, sl;
        bool iq, sq;
        measure_cell<false>(items + r * k, k, style, sep, lane, il, iq);
        measure_cell<true>(scores + r * k, k, style, sep, lane, sl, sq);
        iq |= cell_fixed_has(sep, k);
        sq |= cell_fixed_has(sep, k);
        const int64_t seps = k > 0 ? 2 * (int64_t)(k - 1) : 0;
        if (lane == 0) {
            lens[r] = (un + (uq ? 2 : 0)) + 1 + (2 + seps + il + (iq ? 2 : 0)) + 1 + (2 + seps + sl + (sq ? 2 : 0)) + 1;
            quotes[r] = (uint8_t)((uq ? 1 : 0) | (iq ? 2 : 0) | (sq ? 4 : 0));
        }
    }
}

__global__ void __launch_bounds__(kRowsPerCta * 32)
k_rec_csv_write(const int64_t* __restrict__ users, const int64_t* __restrict__ items, const float* __restrict__ scores,
                int64_t N, int k, int style, char sep, const int64_t* __restrict__ offsets,
                const uint8_t* __restrict__ quotes, char* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kRowsPerCta + (threadIdx.x >> 5); r < N;
         r += (int64_t)gridDim.x * kRowsPerCta) {
        char* o = out + offsets[r];
        const int q = quotes[r];
        int64_t p;
        {
            char t[recfmt::kMaxText];
            const int un = recfmt::format_i64(users[r], B2R_REC_STYLE_BARE, t);
            const bool uq = q & 1;
            if (lane == 0) {
                int i = 0;
                if (uq) o[i++] = '"';
                for (int c = 0; c < un; ++c) o[i++] = t[c];
                if (uq) o[i++] = '"';
                o[i] = sep;
            }
            p = un + (uq ? 2 : 0) + 1;
        }
        p += write_cell<false>(o + p, items + r * k, k, style, q & 2, lane);
        if (lane == 0) o[p] = sep;
        ++p;
        p += write_cell<true>(o + p, scores + r * k, k, style, q & 4, lane);
        if (lane == 0) o[p] = '\n';
    }
}

struct CsvLayout {
    size_t lens, quotes, cub_tmp, cub_bytes, total;
};

static int csv_layout(int64_t N, CsvLayout* L) {
    size_t scan_bytes = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                                  (int)(N + 1), (cudaStream_t)0);
    if (e != cudaSuccess) return set_error((int)e, "cub scan size query failed: %s", cudaGetErrorString(e));
    L->lens = 0;
    L->quotes = align_up((size_t)(N + 1) * sizeof(int64_t), 256);
    L->cub_tmp = L->quotes + align_up((size_t)N + 1, 256);
    L->cub_bytes = scan_bytes;
    L->total = L->cub_tmp + align_up(scan_bytes, 256);
    return 0;
}

static bool csv_shape_ok(int64_t N, int k, int style) {
    return N >= 0 && N < 0x7fffffff && k >= 0 && k <= kMaxK &&
           (style == B2R_REC_STYLE_NP || style == B2R_REC_STYLE_BARE);
}

}  // namespace b2r

using namespace b2r;

extern "C" size_t b2r_rec_csv_workspace_bytes(int64_t N) {
    if (N < 0 || N >= 0x7fffffff) return 0;
    CsvLayout L;
    if (csv_layout(N, &L) != 0) return 0;
    return L.total;
}

extern "C" size_t b2r_rec_csv_text_bytes_max(int64_t N, int k, int style) {
    if (!csv_shape_ok(N, k, style)) return 0;
    return (size_t)N * (size_t)recfmt::row_bytes_max(k, style);
}

extern "C" int b2r_rec_csv(const int64_t* users, const int64_t* items, const float* scores, int64_t N, int k, int style,
                           int sep, char* out, size_t out_capacity, int64_t* row_offsets, void* ws, size_t ws_bytes,
                           b2r_stream_t stream) {
    B2R_REQUIRE(csv_shape_ok(N, k, style), B2R_E_BADARG,
                "b2r_rec_csv: need 0 <= N < 2^31 - 1, 0 <= k <= %d and style 0 or 1 (N=%lld, k=%d, style=%d)", kMaxK,
                (long long)N, k, style);
    B2R_REQUIRE(sep > 0 && sep < 128 && sep != '"' && sep != '\r' && sep != '\n', B2R_E_BADARG,
                "b2r_rec_csv: sep must be one ASCII byte other than NUL, '\"', CR and LF (sep=%d)", sep);
    B2R_REQUIRE(row_offsets && ws, B2R_E_BADARG, "b2r_rec_csv: null pointer");
    B2R_REQUIRE(N == 0 || (users && items && scores && out), B2R_E_BADARG, "b2r_rec_csv: null pointer");
    B2R_REQUIRE(out_capacity >= b2r_rec_csv_text_bytes_max(N, k, style), B2R_E_WORKSPACE,
                "b2r_rec_csv: out holds %zu bytes, the rows may need %zu", out_capacity,
                b2r_rec_csv_text_bytes_max(N, k, style));
    CsvLayout L;
    int rc = csv_layout(N, &L);
    if (rc != 0) return rc;
    B2R_REQUIRE(ws_bytes >= L.total, B2R_E_WORKSPACE, "b2r_rec_csv: workspace %zu < required %zu", ws_bytes, L.total);
    B2R_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, B2R_E_BADARG,
                "b2r_rec_csv: workspace must be 256-byte aligned");
    cudaStream_t s = as_stream(stream);
    char* base = static_cast<char*>(ws);
    int64_t* lens = reinterpret_cast<int64_t*>(base + L.lens);
    uint8_t* quotes = reinterpret_cast<uint8_t*>(base + L.quotes);
    int64_t cap = (N + kRowsPerCta - 1) / kRowsPerCta;
    const int64_t max_grid = (int64_t)sm_count() * 16;
    const int grid = (int)(cap < 1 ? 1 : (cap > max_grid ? max_grid : cap));
    k_rec_csv_measure<<<grid, kRowsPerCta * 32, 0, s>>>(users, items, scores, N, k, style, (char)sep, lens, quotes);
    B2R_LAUNCH_OK("k_rec_csv_measure");
    size_t tmp_bytes = L.cub_bytes;
    B2R_CUDA_OK(cub::DeviceScan::ExclusiveSum(base + L.cub_tmp, tmp_bytes, (const int64_t*)lens, row_offsets,
                                              (int)(N + 1), s));
    count_launch();
    if (N > 0) {
        k_rec_csv_write<<<grid, kRowsPerCta * 32, 0, s>>>(users, items, scores, N, k, style, (char)sep, row_offsets,
                                                          quotes, out);
        B2R_LAUNCH_OK("k_rec_csv_write");
    }
    return 0;
}
