// segment.cu -- row-sparse embedding backward over an index plan, optionally fused with the optimizer step
// (the other half of K2), plus the dense optimizer.
//
// One lane group (LPR = d/4 lanes, one float4 each) owns one unique table row.  It walks the row's
// contributions in ascending batch position, accumulates in registers, and then either writes the
// gradient row once (mode 0), adds it to a dense gradient (mode 1), or applies SGD/Adam/Adagrad in place
// (mode 2: the weight/moment rows are requested before the walk so their HBM latency overlaps it).
// HBM-bound: per unique row 1 write (mode 0) or 3 reads + 3 writes of 4d bytes (Adam); contribution
// operands (user rows, grad_pred) are a few MB and stay in L2.
#include <stdlib.h>

#include "common.cuh"

namespace b2r {

struct Src {
    const float* src;
    const float* coef;
    const int64_t* src_id;
    int64_t n;
    int32_t div;
    int32_t ld;
};

__device__ __forceinline__ void contribution(const Src& s0, const Src& s1, uint32_t p, int64_t& row, float& c) {
    const bool first = (int64_t)p < s0.n;
    const Src& s = first ? s0 : s1;   // (references to kernel params: resolved by predication)
    const int64_t pp = first ? (int64_t)p : (int64_t)p - s0.n;
    int64_t r = (s.div == 1) ? pp : (int64_t)((uint32_t)pp / (uint32_t)s.div);
    if (s.src_id != nullptr) r = s.src_id[r];
    row = r;
    c = (s.coef != nullptr) ? s.coef[pp] : 1.f;
}

__device__ __forceinline__ void optim_update(const b2r_optim& o, float4& w, float4& m, float4& v, const float4& gin) {
    float* wp = &w.x;
    float* mp = &m.x;
    float* vp = &v.x;
    const float* gp = &gin.x;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float g = fmaf(o.weight_decay, wp[i], gp[i]);          // coupled L2 as torch.optim
        if (o.kind == 0) {                                           // SGD
            wp[i] = fmaf(-o.lr, g, wp[i]);
        } else if (o.kind == 1) {                                    // Adam (torch.optim.Adam, amsgrad off)
            mp[i] = fmaf(o.beta1, mp[i], (1.f - o.beta1) * g);
            vp[i] = fmaf(o.beta2, vp[i], (1.f - o.beta2) * g * g);
            const float denom = sqrtf(vp[i]) / sqrtf(o.bc2) + o.eps;
            wp[i] = wp[i] - (o.lr / o.bc1) * (mp[i] / denom);
        } else {                                                     // Adagrad (state sum in v)
            vp[i] = fmaf(g, g, vp[i]);
            wp[i] = wp[i] - o.lr * g / (sqrtf(vp[i]) + o.eps);
        }
    }
}

template <int LPR, int MODE>
__global__ void __launch_bounds__(256)
k_segment_apply(const uint32_t* __restrict__ sorted_key, const uint32_t* __restrict__ sorted_pos,
                const int32_t* __restrict__ seg_start, const int32_t* __restrict__ n_uniq, int n, int64_t n_rows,
                Src s0, Src s1, int64_t* __restrict__ uniq_rows, float* __restrict__ grad_rows,
                float* __restrict__ dense, float* __restrict__ W, float* __restrict__ M, float* __restrict__ V,
                OptK opt) {
    optk_use_clock(opt);
    constexpr int D = LPR * 4;
    constexpr int GPC = 256 / LPR;
    const int sub = threadIdx.x % LPR;
    const int grp = threadIdx.x / LPR;
    const int nu = *n_uniq;
    for (int u = blockIdx.x * GPC + grp; u < nu; u += gridDim.x * GPC) {
        const int beg = seg_start[u];
        const int end = (u + 1 < nu) ? seg_start[u + 1] : n;
        const int64_t row = sorted_key[beg];
        if (row >= n_rows) {                      // sentinel segment of ignored positions (always the last one)
            if (MODE == 0 && sub == 0) uniq_rows[u] = row;
            continue;
        }
        float4 w, m, v;
        if (MODE == 2) {
            w = ld4(W + row * D + sub * 4);
            if (opt.kind == 1) m = ld4(M + row * (opt.state_ld ? opt.state_ld : D) + sub * 4);
            if (opt.kind != 0) v = ld4(V + row * (opt.state_ld ? opt.state_ld : D) + sub * 4);
        } else if (MODE == 1) {
            w = ld4(dense + row * D + sub * 4);
        }
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = beg; j < end; ++j) {
            int64_t r;
            float c;
            contribution(s0, s1, sorted_pos[j], r, c);
            const Src& s = ((int64_t)sorted_pos[j] < s0.n) ? s0 : s1;
            fma4(acc, c, ld4(s.src + r * s.ld + sub * 4));
        }
        if (MODE == 0) {
            if (sub == 0) uniq_rows[u] = row;
            st4(grad_rows + (int64_t)u * D + sub * 4, acc);
        } else if (MODE == 1) {
            w.x += acc.x; w.y += acc.y; w.z += acc.z; w.w += acc.w;
            st4(dense + row * D + sub * 4, w);
        } else {
            optk_update4(opt, w, m, v, acc);
            st4(W + row * D + sub * 4, w);
            if (opt.kind == 1) st4(M + row * (opt.state_ld ? opt.state_ld : D) + sub * 4, m);
            if (opt.kind != 0) st4(V + row * (opt.state_ld ? opt.state_ld : D) + sub * 4, v);
        }
    }
}

// Fused backward+optimizer (mode 2) with RPI unique rows per lane group in flight: the dependent-load chain
// (segment bounds -> row id -> weight/moment rows, and position -> coefficient/source row) is walked for RPI
// rows at once, so RPI x (3 row loads + 1 source row load) are outstanding per lane instead of 4.  Consecutive
// unique rows are adjacent in the sorted order, i.e. ascending addresses a few rows apart in W/m/v.
template <int LPR, int RPI>
__global__ void __launch_bounds__(256)
k_segment_optim(const uint32_t* __restrict__ sorted_key, const uint32_t* __restrict__ sorted_pos,
                const int32_t* __restrict__ seg_start, const int32_t* __restrict__ n_uniq, int n, int64_t n_rows,
                Src s0, Src s1, float* __restrict__ W, float* __restrict__ M, float* __restrict__ V, OptK opt) {
    optk_use_clock(opt);
    static_assert(RPI < LPR, "segment bounds are loaded one per lane");
    constexpr int D = LPR * 4;
    constexpr int GPC = 256 / LPR;
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x % LPR;
    const int grp = threadIdx.x / LPR;
    // shuffles below run inside loops whose trip count differs between the lane groups of a warp
    const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (lane - sub));
    const int nu = *n_uniq;
    for (int u0 = (blockIdx.x * GPC + grp) * RPI; u0 < nu; u0 += gridDim.x * GPC * RPI) {
        // lane k <= RPI holds seg_start[u0 + k] (n past the end); lane k < RPI then its row id and length
        int sv = n;
        if (sub <= RPI && u0 + sub < nu) sv = seg_start[u0 + sub];
        const int nxt = __shfl_sync(gmask, sv, (sub + 1) % LPR, LPR);
        int64_t myrow = n_rows;            // sentinel = skip
        int mylen = 0;
        if (sub < RPI && u0 + sub < nu) {
            myrow = sorted_key[sv];
            mylen = nxt - sv;
            if (myrow >= n_rows) mylen = 0;
        }
        int64_t row[RPI];
        float4 w[RPI], m[RPI], v[RPI], acc[RPI];
        int maxlen = 0;
#pragma unroll
        for (int k = 0; k < RPI; ++k) {
            row[k] = __shfl_sync(gmask, myrow, k, LPR);
            maxlen = max(maxlen, __shfl_sync(gmask, mylen, k, LPR));
            acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row[k] < n_rows) {
                w[k] = ld4(W + row[k] * D + sub * 4);
                if (opt.kind == 1) m[k] = ld4(M + row[k] * (opt.state_ld ? opt.state_ld : D) + sub * 4);
                if (opt.kind != 0) v[k] = ld4(V + row[k] * (opt.state_ld ? opt.state_ld : D) + sub * 4);
            }
        }
        // contributions, t-th of every row in parallel (ascending position within a row -> deterministic)
        for (int t = 0; t < maxlen; ++t) {
            int64_t r = 0;
            float c = 0.f;
            int which = 0;
            if (sub < RPI && t < mylen) {
                const uint32_t p = sorted_pos[sv + t];
                contribution(s0, s1, p, r, c);
                which = ((int64_t)p < s0.n) ? 0 : 1;
            }
#pragma unroll
            for (int k = 0; k < RPI; ++k) {
                const int64_t rk = __shfl_sync(gmask, r, k, LPR);
                const float ck = __shfl_sync(gmask, c, k, LPR);
                const int wk = __shfl_sync(gmask, which, k, LPR);
                const int lk = __shfl_sync(gmask, mylen, k, LPR);
                if (t < lk) {
                    const float* base = wk ? s1.src : s0.src;
                    const int ld = wk ? s1.ld : s0.ld;
                    fma4(acc[k], ck, ld4(base + rk * ld + sub * 4));
                }
            }
        }
#pragma unroll
        for (int k = 0; k < RPI; ++k) {
            if (row[k] < n_rows) {
                optk_update4(opt, w[k], m[k], v[k], acc[k]);
                st4(W + row[k] * D + sub * 4, w[k]);
                if (opt.kind == 1) st4(M + row[k] * (opt.state_ld ? opt.state_ld : D) + sub * 4, m[k]);
                if (opt.kind != 0) st4(V + row[k] * (opt.state_ld ? opt.state_ld : D) + sub * 4, v[k]);
            }
        }
    }
}

// any d % 4 == 0: one warp per unique row, lanes stride over the row's float4 chunks
template <int MODE>
__global__ void __launch_bounds__(256)
k_segment_apply_generic(const uint32_t* __restrict__ sorted_key, const uint32_t* __restrict__ sorted_pos,
                        const int32_t* __restrict__ seg_start, const int32_t* __restrict__ n_uniq, int n,
                        int64_t n_rows, int d, Src s0, Src s1, int64_t* __restrict__ uniq_rows, float* __restrict__ grad_rows,
                        float* __restrict__ dense, float* __restrict__ W, float* __restrict__ M,
                        float* __restrict__ V, OptK opt) {
    optk_use_clock(opt);
    const int lane = threadIdx.x & 31;
    const int nu = *n_uniq;
    const int d4 = d >> 2;
    for (int u = blockIdx.x * 8 + (threadIdx.x >> 5); u < nu; u += gridDim.x * 8) {
        const int beg = seg_start[u];
        const int end = (u + 1 < nu) ? seg_start[u + 1] : n;
        const int64_t row = sorted_key[beg];
        if (MODE == 0 && lane == 0) uniq_rows[u] = row;
        if (row >= n_rows) continue;
        for (int k = lane; k < d4; k += 32) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int j = beg; j < end; ++j) {
                int64_t r;
                float c;
                contribution(s0, s1, sorted_pos[j], r, c);
                const Src& s = ((int64_t)sorted_pos[j] < s0.n) ? s0 : s1;
                fma4(acc, c, ld4(s.src + r * s.ld + k * 4));
            }
            if (MODE == 0) {
                st4(grad_rows + (int64_t)u * d + k * 4, acc);
            } else if (MODE == 1) {
                float4 w = ld4(dense + row * d + k * 4);
                w.x += acc.x; w.y += acc.y; w.z += acc.z; w.w += acc.w;
                st4(dense + row * d + k * 4, w);
            } else {
                float4 w = ld4(W + row * d + k * 4), m, v;
                if (opt.kind == 1) m = ld4(M + row * (opt.state_ld ? opt.state_ld : d) + k * 4);
                if (opt.kind != 0) v = ld4(V + row * (opt.state_ld ? opt.state_ld : d) + k * 4);
                optk_update4(opt, w, m, v, acc);
                st4(W + row * d + k * 4, w);
                if (opt.kind == 1) st4(M + row * (opt.state_ld ? opt.state_ld : d) + k * 4, m);
                if (opt.kind != 0) st4(V + row * (opt.state_ld ? opt.state_ld : d) + k * 4, v);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
k_dense_optim(float* __restrict__ W, const float* __restrict__ G, float* __restrict__ M, float* __restrict__ V,
              int64_t numel, OptK opt) {
    optk_use_clock(opt);
    const int64_t n4 = numel >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 w = ld4(W + i * 4), m, v;
        const float4 g = ld4(G + i * 4);
        if (opt.kind == 1) m = ld4(M + i * 4);
        if (opt.kind != 0) v = ld4(V + i * 4);
        optk_update4(opt, w, m, v, g);
        st4(W + i * 4, w);
        if (opt.kind == 1) st4(M + i * 4, m);
        if (opt.kind != 0) st4(V + i * 4, v);
    }
    // tail (numel % 4) handled by the first threads of block 0
    if (blockIdx.x == 0 && threadIdx.x < (numel & 3)) {
        const int64_t i = (n4 << 2) + threadIdx.x;
        float4 w = make_float4(W[i], 0, 0, 0), m = make_float4(0, 0, 0, 0), v = make_float4(0, 0, 0, 0);
        if (opt.kind == 1) m.x = M[i];
        if (opt.kind != 0) v.x = V[i];
        optk_update4(opt, w, m, v, make_float4(G[i], 0, 0, 0));
        W[i] = w.x;
        if (opt.kind == 1) M[i] = m.x;
        if (opt.kind != 0) V[i] = v.x;
    }
}

static Src to_src(const b2r_grad_source* s, int d) {
    Src r{nullptr, nullptr, nullptr, 0, 1, d};
    if (s) {
        r.src = s->src;
        r.coef = s->coef;
        r.src_id = s->src_id;
        r.n = s->n;
        r.div = s->div < 1 ? 1 : s->div;
        r.ld = s->ld > 0 ? s->ld : d;
    }
    return r;
}

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_segment_apply(const uint32_t* sorted_key, const uint32_t* sorted_pos, const int32_t* seg_start,
                                 const int32_t* n_uniq, int64_t n, int64_t n_rows, int d,
                                 const b2r_grad_source* s0,
                                 const b2r_grad_source* s1, int mode, int64_t* uniq_rows, float* grad_rows,
                                 float* dense, float* W, float* m, float* v, const b2r_optim* opt,
                                 b2r_stream_t stream) {
    B2R_REQUIRE(sorted_key && sorted_pos && seg_start && n_uniq && s0 && s0->src, B2R_E_BADARG,
                "b2r_segment_apply: null pointer");
    B2R_REQUIRE(n > 0 && n <= 0x7fffffff && d > 0 && d % 4 == 0, B2R_E_BADARG,
                "b2r_segment_apply: bad n=%lld or d=%d", (long long)n, d);
    B2R_REQUIRE(s0->n + (s1 ? s1->n : 0) == n, B2R_E_BADARG,
                "b2r_segment_apply: sources cover %lld positions, plan has %lld",
                (long long)(s0->n + (s1 ? s1->n : 0)), (long long)n);
    B2R_REQUIRE(!s1 || s1->src, B2R_E_BADARG, "b2r_segment_apply: second source has null src");
    b2r_optim o{};
    if (mode == 0) {
        B2R_REQUIRE(uniq_rows && grad_rows, B2R_E_BADARG, "b2r_segment_apply: mode 0 needs uniq_rows, grad_rows");
    } else if (mode == 1) {
        B2R_REQUIRE(dense, B2R_E_BADARG, "b2r_segment_apply: mode 1 needs dense");
    } else if (mode == 2) {
        B2R_REQUIRE(W && opt, B2R_E_BADARG, "b2r_segment_apply: mode 2 needs W and opt");
        o = *opt;
        B2R_REQUIRE(o.kind >= 0 && o.kind <= 2, B2R_E_BADARG, "b2r_segment_apply: optimizer kind %d", o.kind);
        B2R_REQUIRE(o.kind != 1 || (m && v), B2R_E_BADARG, "b2r_segment_apply: Adam needs m and v");
        B2R_REQUIRE(o.kind != 2 || v, B2R_E_BADARG, "b2r_segment_apply: Adagrad needs v (state sum)");
    } else {
        return set_error(B2R_E_BADARG, "b2r_segment_apply: mode %d", mode);
    }
    cudaStream_t s = as_stream(stream);
    const Src a = to_src(s0, d), b = to_src(s1, d);
    const int nn = (int)n;
    // n_uniq lives on the device: size the grid for the worst case (n unique rows), capped persistent
#define B2R_SEG(LPR, MODE)                                                                             \
    do {                                                                                               \
        constexpr int GPC = 256 / LPR;                                                                 \
        int64_t need = (n + GPC - 1) / GPC;                                                            \
        const int64_t cap = (int64_t)sm_count() * 16;                                                  \
        const int grid = (int)(need < cap ? need : cap);                                               \
        k_segment_apply<LPR, MODE><<<grid, 256, 0, s>>>(sorted_key, sorted_pos, seg_start, n_uniq, nn, n_rows, a, b, \
                                                        uniq_rows, grad_rows, dense, W, m, v, make_optk(o)); \
    } while (0)
#define B2R_SEG_D(MODE)                                                                                \
    do {                                                                                               \
        if (d == 32) B2R_SEG(8, MODE);                                                                 \
        else if (d == 64) B2R_SEG(16, MODE);                                                           \
        else if (d == 128) B2R_SEG(32, MODE);                                                          \
        else {                                                                                         \
            int64_t need = (n + 7) / 8;                                                                \
            const int64_t cap = (int64_t)sm_count() * 16;                                              \
            const int grid = (int)(need < cap ? need : cap);                                           \
            k_segment_apply_generic<MODE><<<grid, 256, 0, s>>>(sorted_key, sorted_pos, seg_start, n_uniq, nn, n_rows, d, \
                                                               a, b, uniq_rows, grad_rows, dense, W, m, v, make_optk(o)); \
        }                                                                                              \
    } while (0)
    // rows per lane-group iteration of the optimizer kernel: 4 measured best at config 2 (1: +9 %, 2: +3 % step time)
#define B2R_OPT(LPR, RPI)                                                                              \
    do {                                                                                               \
        constexpr int GPC = 256 / LPR;                                                                 \
        int64_t need = (n + (int64_t)GPC * RPI - 1) / ((int64_t)GPC * RPI);                            \
        const int64_t cap = (int64_t)sm_count() * 16;                                                  \
        const int grid = (int)(need < cap ? need : cap);                                               \
        k_segment_optim<LPR, RPI><<<grid, 256, 0, s>>>(sorted_key, sorted_pos, seg_start, n_uniq, nn, n_rows, a, b, \
                                                       W, m, v, make_optk(o));                         \
    } while (0)
    if (mode == 0) B2R_SEG_D(0);
    else if (mode == 1) B2R_SEG_D(1);
    else if (d == 32) B2R_OPT(8, 4);
    else if (d == 64) B2R_OPT(16, 4);
    else if (d == 128) B2R_OPT(32, 4);
    else B2R_SEG_D(2);
#undef B2R_OPT
#undef B2R_SEG_D
#undef B2R_SEG
    B2R_LAUNCH_OK("k_segment_apply");
    return 0;
}

extern "C" int b2r_dense_optim(float* W, const float* grad, float* m, float* v, int64_t numel,
                               const b2r_optim* opt, b2r_stream_t stream) {
    B2R_REQUIRE(W && grad && opt, B2R_E_BADARG, "b2r_dense_optim: null pointer");
    B2R_REQUIRE(opt->kind >= 0 && opt->kind <= 2, B2R_E_BADARG, "b2r_dense_optim: optimizer kind %d", opt->kind);
    B2R_REQUIRE(opt->kind != 1 || (m && v), B2R_E_BADARG, "b2r_dense_optim: Adam needs m and v");
    B2R_REQUIRE(opt->kind != 2 || v, B2R_E_BADARG, "b2r_dense_optim: Adagrad needs v");
    B2R_REQUIRE(opt->state_ld == 0, B2R_E_BADARG, "b2r_dense_optim: interleaved optimizer state is row-sparse only");
    B2R_REQUIRE(aligned16(W) && aligned16(grad), B2R_E_BADARG, "b2r_dense_optim: 16-byte alignment");
    if (numel <= 0) return 0;
    int64_t need = ((numel >> 2) + 255) / 256;
    if (need < 1) need = 1;
    const int64_t cap = (int64_t)sm_count() * 16;
    k_dense_optim<<<(int)(need < cap ? need : cap), 256, 0, as_stream(stream)>>>(W, grad, m, v, numel, make_optk(*opt));
    B2R_LAUNCH_OK("k_dense_optim");
    return 0;
}

// ---- device-side optimizer clock (b2r_optim.clock) ---------------------------------------------------------------------
namespace b2r {
// the betas arrive as doubles and the bias corrections are rounded to float before use, exactly as the host route does
// (python computes 1 - beta ** t in double, b2r_optim carries it as float, make_optk divides in double): a replayed step
// uses the same step size as the eagerly launched one
__global__ void k_optim_tick(float* __restrict__ clock, float lr, double beta1, double beta2) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const double t = (double)clock[0] + 1.0;
        const float bc1 = (float)(1.0 - pow(beta1, t)), bc2 = (float)(1.0 - pow(beta2, t));
        clock[0] = (float)t;
        clock[1] = (float)((double)lr / (double)bc1);                          // lr / bias_correction1
        clock[2] = (float)(1.0 / sqrt((double)bc2));                           // 1 / sqrt(bias_correction2)
    }
}
}  // namespace b2r

extern "C" int b2r_optim_tick(float* clock, float lr, double beta1, double beta2, b2r_stream_t stream) {
    B2R_REQUIRE(clock, B2R_E_BADARG, "b2r_optim_tick: null pointer");
    b2r::k_optim_tick<<<1, 32, 0, as_stream(stream)>>>(clock, lr, beta1, beta2);
    B2R_LAUNCH_OK("k_optim_tick");
    return 0;
}
