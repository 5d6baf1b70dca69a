// neumf_all.cu -- NeuMF's scores against the whole catalogue (the test_all protocol, BaseModel.py:194-198) for a window
// of rows of one evaluation batch, without the forward's [Bn * n_items, 2d] concat input or its per-layer activations.
//
// Bit-identity with NeuMF.forward (plugin.py) is the contract: for candidate row m = b * n_items + c of the batch the
// forward computes
//   GMF  q = mf_u[b] * w_out[:d] (k_colscale), then <q, mf_i[item]> as k_rowdot_fwd<LPR = d / 4> does: dot4 per lane and
//        group_sum<LPR>'s xor butterfly;
//   MLP  per hidden layer k_linear_tc<KS, NW> on 64-row tiles anchored at row 0 of the batch: hi/lo split operands, the
//        3-product wgmma loop, then acc + bias and ReLU (rows past the batch enter the next layer as zeros);
//   out  k_gemm<0, 0> for N = 1: s = fmaf(h_k, w_out[d + k], s) for k ascending from s = 0;
//   and the final gmf + mlp.
// This kernel does exactly those operations on exactly those tiles (linear_tc.cuh holds the split and the MMA loop both
// kernels run), so a window's block equals the forward's bit for bit.  The envelope (b2r_neumf_score_rows_check) admits
// only shapes on which the forward itself takes the tensor-core kernel for every hidden layer.
//
// One warpgroup per CTA, persistent over 64-row tiles.  Every layer's W stays resident in shared memory as hi/lo tiles;
// a tile's input rows [mlp_u[b]; mlp_i[item]] are gathered straight into the first layer's swizzled hi/lo operand (the
// next tile's gather is in flight during this tile's first MMAs, as is the GMF dot), and each layer's epilogue writes
// the next layer's operand in shared memory, the last one an fp32 copy for the output layer's fmaf chain.  Tiles are
// visited column block by column block across the window's users, so the item rows of one block are read from HBM once
// and reused from L2 by every user of the window.
#include <algorithm>

#include "linear_tc.cuh"

namespace b2r {

constexpr int kNmMaxLayers = B2R_NEUMF_MAX_LAYERS;
constexpr size_t kNmWindowBytes = 32u << 20;      // one window's score block: topk.cu's kChunkBytes budget
constexpr size_t kNmSmemMax = 227 * 1024;         // dynamic shared memory of one CTA on sm_90

// widest hidden layer per embedding width: the accumulator (N / 2 registers) and the next tile's prefetched input rows
// (d floats) share one thread's 255 registers, and at d = 64 a 128-wide layer makes ptxas spill
constexpr int nm_max_width(int d) { return d == 32 ? 128 : 64; }

// The layer shapes (K / 32 slabs, wgmma width) the kernel is built for: every K the forward's tensor-core Linear takes
// (32, 64, 96, 128) at every width it uses up to 128.  The dispatch switch and the envelope check both expand this one
// list, so a layer the check admits is a layer the kernel runs.
#define B2R_NM_LAYER_SHAPES(X)                                                   \
    X(1, 16) X(1, 32) X(1, 64) X(1, 128) X(2, 16) X(2, 32) X(2, 64) X(2, 128)    \
    X(3, 16) X(3, 32) X(3, 64) X(3, 128) X(4, 16) X(4, 32) X(4, 64) X(4, 128)

// whether k_neumf_score_rows<d> has a case for a layer of KS slabs at wgmma width NW
static bool nm_layer_built(int d, int KS, int NW) {
    bool listed = false;
#define B2R_NM_LISTED(ks, nw) listed = listed || (KS == ks && NW == nw);
    B2R_NM_LAYER_SHAPES(B2R_NM_LISTED)
#undef B2R_NM_LISTED
    return listed && NW <= nm_max_width(d);
}

struct NmLayer {
    const float* W;
    const float* bias;
    int K, N, NW, KS;
    uint32_t w_off;          // W hi tile; lo at w_off + KS * NW * 128
    uint32_t a_off;          // this layer's A operand (hi); lo at a_off + KS * 64 * 128
};

struct NmParams {
    const float *mf_u, *mf_i, *mlp_u, *mlp_i, *w_out;
    const int64_t *users, *targets;
    int64_t n_users, n_items;
    NmLayer layer[kNmMaxLayers];
    int L, h_ld;
    uint32_t h_off, g_off;   // fp32 copy of the last hidden layer [64][h_ld], GMF dots [64]
    int64_t M;               // Bn * n_items rows of the batch
    int64_t r0, r1;          // the window's rows [b0 * n_items, b1 * n_items)
    int64_t t0, t1;          // tiles that meet the window
    int ub0, nu, jmax;       // tile owners (user of a tile's first row) and tiles per owner
    int b0;
    FastDiv div_n;
    float* out;
    int64_t ld_out;
    int32_t* err;
};

// a tile's first row belongs to its owner; owner u's tiles are [ceil(u n / 64), ceil((u + 1) n / 64))
__device__ __forceinline__ int64_t nm_first_tile(const NmParams& p, int64_t u) { return (u * p.n_items + TC_M - 1) / TC_M; }

// work item w -> tile, owners fastest (-1: no tile): consecutive work items take the same column block of successive users
__device__ __forceinline__ int64_t nm_tile_of(const NmParams& p, int64_t w) {
    const int64_t u = p.ub0 + w % p.nu, j = w / p.nu;
    const int64_t t = nm_first_tile(p, u) + j;
    return (t < nm_first_tile(p, u + 1) && t >= p.t0 && t < p.t1) ? t : -1;
}

__device__ __forceinline__ int64_t nm_next_work(const NmParams& p, int64_t w) {
    const int64_t total = (int64_t)p.nu * p.jmax;
    while (w < total && nm_tile_of(p, w) < 0) w += gridDim.x;
    return w < total ? w : -1;
}

// (user row, item row) of batch row m < M: column 0 is the target, column c >= 1 item c
__device__ __forceinline__ void nm_row_ids(const NmParams& p, int64_t m, int64_t& user, int64_t& item, int32_t* err) {
    const uint32_t b = fastdiv((uint32_t)m, p.div_n);
    const int64_t c = m - (int64_t)b * p.n_items;
    user = checked_id(p.users[b], p.n_users, err);
    item = c == 0 ? checked_id(p.targets[b], p.n_items, err) : c;
}

// the first layer's input rows of a tile, in k_linear_tc's load order: element e = i * 128 + tid is (row e / (8 KS),
// slab (e / 8) % KS, chunk e % 8); rows past the batch are zeros
template <int D>
__device__ __forceinline__ void nm_gather(const NmParams& p, int64_t tile, float4 (&v)[D / 4]) {
    constexpr int KS = 2 * D / 32;
    const int64_t m0 = tile * TC_M;
#pragma unroll
    for (int i = 0; i < D / 4; ++i) {
        const int e = i * TC_THREADS + threadIdx.x;
        const int c = e % 8, s = (e / 8) % KS, r = e / (8 * KS);
        const int col = s * 32 + c * 4;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m0 + r < p.M) {
            int64_t user, item;
            nm_row_ids(p, m0 + r, user, item, col == 0 ? p.err : nullptr);
            v[i] = col < D ? ld4(p.mlp_u + user * D + col) : ld_row4(p.mlp_i + item * D + (col - D));
        }
    }
}

// GMF dots of a tile's 64 rows in k_rowdot_fwd's lane-group layout (LPR = D / 4 lanes per row) -> g[64]
template <int D>
__device__ __forceinline__ void nm_gmf(const NmParams& p, int64_t m0, float* g) {
    constexpr int LPR = D / 4, G = TC_THREADS / LPR, PASSES = TC_M / G, BATCH = 4;
    const int sub = threadIdx.x % LPR, grp = threadIdx.x / LPR;
    const float4 w = ld4(p.w_out + sub * 4);
#pragma unroll
    for (int p0 = 0; p0 < PASSES; p0 += BATCH) {
        float4 q[BATCH], r[BATCH];
#pragma unroll
        for (int k = 0; k < BATCH; ++k) {
            const int64_t m = m0 + (p0 + k) * G + grp;
            q[k] = r[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < p.M) {
                int64_t user, item;
                nm_row_ids(p, m, user, item, nullptr);
                const float4 u = ld4(p.mf_u + user * D + sub * 4);
                q[k] = make_float4(u.x * w.x, u.y * w.y, u.z * w.z, u.w * w.w);       // k_colscale
                r[k] = ld_row4(p.mf_i + item * D + sub * 4);
            }
        }
#pragma unroll
        for (int k = 0; k < BATCH; ++k) {
            const float s = group_sum<LPR>(dot4(q[k], r[k]));
            if (sub == 0) g[(p0 + k) * G + grp] = s;
        }
    }
}

// one hidden layer of one tile: MMAs on the resident operands, then bias + ReLU into the next layer's operand (or the
// fp32 copy after the last layer).  Layer 0 also prefetches the next tile's input and computes the GMF dots meanwhile.
template <int D, int KS, int NW>
__device__ __forceinline__ void nm_layer(const NmParams& p, char* sm, int l, int64_t m0, int64_t next_tile,
                                         float4 (&v)[D / 4]) {
    const NmLayer& ly = p.layer[l];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    char* A_hi = sm + ly.a_off;
    char* B_hi = sm + ly.w_off;
    wg_fence();
    tc_mma_3x<KS, NW>(acc, A_hi, A_hi + KS * TC_M * 128, B_hi, B_hi + KS * NW * 128);
    wg_commit();
    if (l == 0) {
        if (next_tile >= 0) nm_gather<D>(p, next_tile, v);
        nm_gmf<D>(p, m0, reinterpret_cast<float*>(sm + p.g_off));
    }
    wg_wait_all();
    wg_fence_regs(acc);
    const bool last = l == p.L - 1;
    char* N_hi = last ? nullptr : sm + p.layer[l + 1].a_off;
    char* N_lo = last ? nullptr : N_hi + p.layer[l + 1].KS * TC_M * 128;
    float* h = reinterpret_cast<float*>(sm + p.h_off);
    const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < NW / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        if (col >= ly.N) continue;
        const float b0 = ly.bias != nullptr ? __ldg(ly.bias + col) : 0.f;
        const float b1 = ly.bias != nullptr ? __ldg(ly.bias + col + 1) : 0.f;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int row = r0 + 8 * hh;
            float y0 = fmaxf(acc[4 * j + 2 * hh] + b0, 0.f), y1 = fmaxf(acc[4 * j + 2 * hh + 1] + b1, 0.f);
            if (last) {
                h[row * p.h_ld + col] = y0;
                h[row * p.h_ld + col + 1] = y1;
                continue;
            }
            if (m0 + row >= p.M) y0 = y1 = 0.f;           // the forward's next layer reads zeros past the batch
            float2 hi, lo;
            tc_split(y0, hi.x, lo.x);
            tc_split(y1, hi.y, lo.y);
            const uint32_t off = (uint32_t)(col >> 5) * (TC_M * 128) + tc_swz(row, (col & 31) >> 2) + (col & 3) * 4;
            *reinterpret_cast<float2*>(N_hi + off) = hi;
            *reinterpret_cast<float2*>(N_lo + off) = lo;
        }
    }
}

template <int D>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_neumf_score_rows(const __grid_constant__ NmParams p) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr int KS0 = 2 * D / 32;
    char* sm = reinterpret_cast<char*>(smem_raw) + ((1024u - (wg_smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x;

    // every layer's W -> hi/lo tiles (once per CTA), in k_linear_tc's layout; rows N..NW-1 are zero
    for (int l = 0; l < p.L; ++l) {
        const NmLayer& ly = p.layer[l];
        char* B_hi = sm + ly.w_off;
        char* B_lo = B_hi + ly.KS * ly.NW * 128;
        for (int e = tid; e < ly.NW * ly.KS * 8; e += TC_THREADS) {
            const int c = e % 8, s = (e / 8) % ly.KS, n = e / (8 * ly.KS);
            const float4 v = n < ly.N ? *reinterpret_cast<const float4*>(ly.W + (size_t)n * ly.K + s * 32 + c * 4)
                                      : make_float4(0.f, 0.f, 0.f, 0.f);
            tc_store_split(B_hi + s * ly.NW * 128, B_lo + s * ly.NW * 128, n, c, v);
        }
    }

    float4 v[D / 4];
    int64_t w = nm_next_work(p, blockIdx.x);
    if (w >= 0) nm_gather<D>(p, nm_tile_of(p, w), v);
    char* A_hi = sm + p.layer[0].a_off;
    char* A_lo = A_hi + KS0 * TC_M * 128;
    const float* h = reinterpret_cast<const float*>(sm + p.h_off);
    const float* g = reinterpret_cast<const float*>(sm + p.g_off);
    while (w >= 0) {
        const int64_t m0 = nm_tile_of(p, w) * TC_M;
        const int64_t wn = nm_next_work(p, w + gridDim.x);
        __syncthreads();                  // the previous tile's MMAs and output chain are done with A, h and g
#pragma unroll
        for (int i = 0; i < D / 4; ++i) {
            const int e = i * TC_THREADS + tid;
            tc_store_split(A_hi + ((e / 8) % KS0) * TC_M * 128, A_lo + ((e / 8) % KS0) * TC_M * 128, e / (8 * KS0), e % 8,
                           v[i]);
        }
        for (int l = 0; l < p.L; ++l) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> async proxy
            __syncthreads();
            const int64_t nt = (l == 0 && wn >= 0) ? nm_tile_of(p, wn) : -1;
            const NmLayer& ly = p.layer[l];
            switch (ly.KS * 1024 + ly.NW) {
#define B2R_NM_CASE(KS, NW) \
                case KS * 1024 + NW: if constexpr (NW <= nm_max_width(D)) nm_layer<D, KS, NW>(p, sm, l, m0, nt, v); break;
                B2R_NM_LAYER_SHAPES(B2R_NM_CASE)
#undef B2R_NM_CASE
                default: break;           // not reached: b2r_neumf_score_rows_check admits listed shapes only
            }
        }
        __syncthreads();
        // output layer (k_gemm<0, 0>, N = 1) + GMF, one row per thread
        if (tid < TC_M) {
            const int64_t m = m0 + tid;
            if (m >= p.r0 && m < p.r1) {
                const float* wm = p.w_out + D;
                const int N = p.layer[p.L - 1].N;
                float s = 0.f;
                for (int k = 0; k < N; ++k) s = fmaf(h[tid * p.h_ld + k], __ldg(wm + k), s);
                const uint32_t b = fastdiv((uint32_t)m, p.div_n);
                const int64_t c = m - (int64_t)b * p.n_items;
                p.out[(int64_t)(b - p.b0) * p.ld_out + c] = __fadd_rn(g[tid], s);
            }
        }
        w = wn;
    }
}

struct NmPlan {
    int KS[kNmMaxLayers], NW[kNmMaxLayers];
    uint32_t w_off[kNmMaxLayers], a_off[kNmMaxLayers], h_off, g_off;
    int h_ld;
    size_t bytes;            // dynamic shared memory, 1 KB of alignment slack included
};

// shared memory: W tiles of every layer, two A operand buffers (layer l reads buffer l % 2, writes the other), the fp32
// copy of the last hidden layer and the GMF dots
static NmPlan nm_plan(int d, int L, const int32_t* widths) {
    NmPlan pl{};
    size_t off = 0, abuf[2] = {0, 0};
    for (int l = 0; l < L; ++l) {
        const int K = l == 0 ? 2 * d : widths[l - 1];
        pl.KS[l] = K / 32;
        pl.NW[l] = tc_width(widths[l]);
        pl.w_off[l] = (uint32_t)off;
        off += (size_t)2 * pl.KS[l] * pl.NW[l] * 128;
        abuf[l % 2] = std::max(abuf[l % 2], (size_t)2 * pl.KS[l] * TC_M * 128);
    }
    for (int l = 0; l < L; ++l) pl.a_off[l] = (uint32_t)(off + (l % 2 ? abuf[0] : 0));
    off += abuf[0] + abuf[1];
    pl.h_ld = widths[L - 1] + 1;                       // odd stride: the output chain reads one row per thread
    pl.h_off = (uint32_t)off;
    off += (size_t)TC_M * pl.h_ld * 4;
    pl.g_off = (uint32_t)off;
    off += (size_t)TC_M * 4;
    pl.bytes = off + 1024;
    return pl;
}

static int neumf_check(int d, int L, const int32_t* widths, int64_t Bn, int64_t n_items) {
    B2R_REQUIRE(d == 32 || d == 64, B2R_E_UNSUPPORTED, "b2r_neumf_score_rows: d=%d, the fused scorer is built for d in {32, 64}", d);
    B2R_REQUIRE(L >= 1 && L <= kNmMaxLayers && widths != nullptr, B2R_E_UNSUPPORTED,
                "b2r_neumf_score_rows: %d hidden layers, the fused scorer takes 1..%d", L, kNmMaxLayers);
    B2R_REQUIRE(Bn >= 1 && n_items >= 1, B2R_E_UNSUPPORTED, "b2r_neumf_score_rows: empty batch");
    const int64_t M = Bn * n_items;
    B2R_REQUIRE(M >= kTcMinRows && M <= 0x7fffffff, B2R_E_UNSUPPORTED,
                "b2r_neumf_score_rows: %lld candidate rows, the forward's tensor-core Linear starts at %lld and stops at 2^31 - 1",
                (long long)M, (long long)kTcMinRows);
    for (int l = 0; l < L; ++l) {
        const int K = l == 0 ? 2 * d : widths[l - 1], N = widths[l];
        B2R_REQUIRE(linear_tc_shape(M, N, K), B2R_E_UNSUPPORTED,
                    "b2r_neumf_score_rows: layer %d (K=%d, N=%d) is not on the forward's tensor-core Linear", l, K, N);
        B2R_REQUIRE(N <= nm_max_width(d), B2R_E_UNSUPPORTED,
                    "b2r_neumf_score_rows: layer %d has N=%d, above %d at d=%d (registers)", l, N, nm_max_width(d), d);
        B2R_REQUIRE(nm_layer_built(d, K / 32, tc_width(N)), B2R_E_UNSUPPORTED,
                    "b2r_neumf_score_rows: layer %d (K=%d, N=%d) has no case in the fused kernel", l, K, N);
    }
    const NmPlan pl = nm_plan(d, L, widths);
    B2R_REQUIRE(pl.bytes <= kNmSmemMax, B2R_E_UNSUPPORTED,
                "b2r_neumf_score_rows: the resident weights and operands need %zu bytes of shared memory, above %zu",
                pl.bytes, kNmSmemMax);
    return 0;
}

template <int D>
static int launch_neumf(const NmParams& p, size_t smem, int64_t work, cudaStream_t s) {
    B2R_CUDA_OK(cudaFuncSetAttribute(k_neumf_score_rows<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2R_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_neumf_score_rows<D>, TC_THREADS, smem));
    int64_t grid = (int64_t)sm_count() * (per_sm < 1 ? 1 : per_sm);
    if (grid > work) grid = work;
    k_neumf_score_rows<D><<<(int)grid, TC_THREADS, smem, s>>>(p);
    B2R_LAUNCH_OK("k_neumf_score_rows");
    return 0;
}

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_neumf_score_rows_check(int d, int n_layers, const int32_t* widths, int64_t Bn, int64_t n_items) {
    return neumf_check(d, n_layers, widths, Bn, n_items);
}

extern "C" int b2r_neumf_window_rows(int64_t Bn, int64_t n_items) {
    int64_t rows = n_items > 0 ? (int64_t)(kNmWindowBytes / (4 * (size_t)n_items)) : Bn;
    if (rows > Bn) rows = Bn;
    return (int)(rows < 1 ? 1 : rows);
}

extern "C" int b2r_neumf_score_rows(const b2r_neumf_rows* a, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(a != nullptr && a->mf_u && a->mf_i && a->mlp_u && a->mlp_i && a->w_out && a->users && a->targets && a->out,
                B2R_E_BADARG, "b2r_neumf_score_rows: null pointer");
    const int rc = neumf_check(a->d, a->n_layers, a->widths, a->Bn, a->n_items);
    if (rc != 0) return rc;
    B2R_REQUIRE(a->n_users >= 1 && a->b0 >= 0 && a->b0 < a->b1 && a->b1 <= a->Bn && a->ld_out >= a->n_items, B2R_E_BADARG,
                "b2r_neumf_score_rows: window [%d, %d) of %d rows, ld_out=%lld, n_items=%lld", a->b0, a->b1, a->Bn,
                (long long)a->ld_out, (long long)a->n_items);
    B2R_REQUIRE(aligned16(a->mf_u) && aligned16(a->mf_i) && aligned16(a->mlp_u) && aligned16(a->mlp_i) &&
                aligned16(a->w_out), B2R_E_BADARG, "b2r_neumf_score_rows: tables and w_out must be 16-byte aligned");
    const int d = a->d, L = a->n_layers;
    const NmPlan pl = nm_plan(d, L, a->widths);
    NmParams p{};
    p.mf_u = a->mf_u; p.mf_i = a->mf_i; p.mlp_u = a->mlp_u; p.mlp_i = a->mlp_i; p.w_out = a->w_out;
    p.users = a->users; p.targets = a->targets;
    p.n_users = a->n_users; p.n_items = a->n_items;
    p.L = L;
    for (int l = 0; l < L; ++l) {
        B2R_REQUIRE(a->W[l] != nullptr && aligned16(a->W[l]), B2R_E_BADARG,
                    "b2r_neumf_score_rows: W[%d] must be non-null and 16-byte aligned", l);
        p.layer[l] = NmLayer{a->W[l], a->bias[l], l == 0 ? 2 * d : a->widths[l - 1], a->widths[l], pl.NW[l], pl.KS[l],
                             pl.w_off[l], pl.a_off[l]};
    }
    p.h_ld = pl.h_ld; p.h_off = pl.h_off; p.g_off = pl.g_off;
    const int64_t n = a->n_items;
    p.M = (int64_t)a->Bn * n;
    p.r0 = (int64_t)a->b0 * n;
    p.r1 = (int64_t)a->b1 * n;
    p.t0 = p.r0 / TC_M;
    p.t1 = (p.r1 + TC_M - 1) / TC_M;
    p.ub0 = (int)(p.t0 * TC_M / n);
    p.nu = (int)((p.t1 - 1) * TC_M / n) + 1 - p.ub0;
    p.jmax = (int)((n + TC_M - 1) / TC_M);
    p.b0 = a->b0;
    p.div_n = make_fastdiv((uint32_t)n);
    p.out = a->out; p.ld_out = a->ld_out;
    p.err = err_flag;
    const int64_t work = (int64_t)p.nu * p.jmax;
    cudaStream_t s = as_stream(stream);
    return d == 32 ? launch_neumf<32>(p, pl.bytes, work, s) : launch_neumf<64>(p, pl.bytes, work, s);
}
