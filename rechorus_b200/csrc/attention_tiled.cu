// attention_tiled.cu -- causal multi-head attention of SASRec (utils/layers.py:52-63) at batch widths the shared-memory
// kernels cannot hold: L up to kTiledMaxL, shared memory independent of L.
//
// Same arithmetic as attention_rt.cu (attention_lane.cuh): one lane owns one (row, head), fp32 FMA, base-2 online softmax
// with a saved log-sum-exp, and a warp covers the same 32-row block with the same key range as there.  What changes is
// the staging: instead of the whole sequence, key/value tiles (forward, dQ) or query/dO/(lse, delta) tiles (dK/dV) of
// kTK rows of ONE head stream through a two-slot cp.async ring, and a CTA owns one (sequence, head, 128-row tile), so
// long causal rows spread over many CTAs.  Launched longest tiles first.
//   k_attention_fwd_tiled      lane = query i : ctx_i, lse_i
//   k_attention_bwd_dq_tiled   lane = query i : delta_i = dO_i . O_i (to the workspace), dQ_i
//   k_attention_bwd_dkv_tiled  lane = key j   : dK_j, dV_j over queries i >= j's 32-row block
// For d/H in {8, 16, 32} every lane runs exactly attention_rt.cu's sequence of operations, so the results are the same
// bits wherever both accept a shape.  d/H = 64 would need 4 x 64 registers per lane in the dK/dV pass: there two lanes
// share a row, each holding 32 columns, and dot products are the two halves' sum (a 16-row warp block).
// `live`: rows t >= live[b] are dead -- skipped, outputs written as zeros (attention.cu's contract).
#include "common.cuh"
#include "seq_limits.cuh"
#include "attention_lane.cuh"

namespace b2r {

constexpr int kTW = 4;                       // warps per CTA
constexpr int kTK = 32;                      // rows per staged tile

template <int DK>
struct TiledCfg {
    static constexpr int SP = DK > 32 ? 2 : 1;           // lanes per (row, head)
    static constexpr int DL = DK / SP;                   // columns per lane
    static constexpr int HO = DL + (SP > 1 ? 4 : 0);     // shared offset of a row's second half (keeps halves off one bank)
    static constexpr int S = SP * HO;                    // shared row stride
    static constexpr int RPW = 32 / SP;                  // rows per warp
    static constexpr int TR = kTW * RPW;                 // rows per CTA tile
};

__device__ __forceinline__ void cp16(float* smem_dst, const float* gsrc) {
    const uint32_t sa = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// rows r0 .. r0+n-1 of one head's DK columns (src = sequence row 0, column h*DK; row stride ld) -> dst [n][S]
template <int DK>
__device__ __forceinline__ void stage_head(float* dst, const float* src, int64_t ld, int r0, int n) {
    using C = TiledCfg<DK>;
    for (int e = threadIdx.x; e < n * (DK / 4); e += kTW * 32) {
        const int r = e / (DK / 4), c = (e - r * (DK / 4)) * 4;
        cp16(dst + r * C::S + (c / C::DL) * C::HO + c % C::DL, src + (int64_t)(r0 + r) * ld + c);
    }
}

// the two halves of a split row's dot product (SP = 2: lanes 2r, 2r+1 get the same sum)
template <int SP>
__device__ __forceinline__ float row_sum(float s) {
    if (SP > 1) s += __shfl_xor_sync(B2R_FULL_MASK, s, 1);
    return s;
}

template <int DL>
__device__ __forceinline__ void store_or_zero(float* dst, const float (&src)[DL], bool live) {
#pragma unroll
    for (int c = 0; c < DL; c += 4)
        *reinterpret_cast<float4*>(dst + c) =
            live ? make_float4(src[c], src[c + 1], src[c + 2], src[c + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// CTA -> (sequence, head, row tile); tiles in the order given by `longest_last` (queries: last tile has most keys)
struct TileId { int b, h, tile; };
__device__ __forceinline__ TileId tile_id(int B, int H, int ntiles, bool longest_last) {
    const int64_t bh = (int64_t)B * H;
    const int t = (int)(blockIdx.x / bh), rem = (int)(blockIdx.x % bh);
    return {rem / H, rem % H, longest_last ? ntiles - 1 - t : t};
}

template <int DK>
__global__ void __launch_bounds__(kTW * 32)
k_attention_fwd_tiled(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                      const int64_t* __restrict__ live, float* __restrict__ ctx, float* __restrict__ lse, int B, int L,
                      int d, int H, int ntiles, float scale2) {
    using C = TiledCfg<DK>;
    __shared__ __align__(16) float ks[2][kTK * C::S];
    __shared__ __align__(16) float vs[2][kTK * C::S];
    const TileId id = tile_id(B, H, ntiles, true);
    const int b = id.b, h = id.h, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int part = lane % C::SP;
    const int64_t row0 = (int64_t)b * L;
    const int Lb = live_rows(live, b, L);
    const int r_t = id.tile * C::TR, r_w = r_t + warp * C::RPW;
    const int i = r_w + lane / C::SP;
    const bool active = i < Lb;
    const int ii = active ? i : Lb - 1;
    const int jend = min(Lb - 1, r_t + C::TR - 1);                // last key the CTA needs
    const int jmax = r_w < Lb ? min(Lb - 1, r_w + C::RPW - 1) : -1;  // last key this warp needs (-1: all rows dead)
    const int nkt = r_t < Lb ? jend / kTK + 1 : 0;
    const float* kh = k + row0 * ld + h * DK;
    const float* vh = v + row0 * ld + h * DK;
    float qi[C::DL], acc[C::DL];
    if (r_w < Lb) load_vec<C::DL>(qi, q + (row0 + ii) * ld + h * DK + part * C::DL);
#pragma unroll
    for (int c = 0; c < C::DL; ++c) acc[c] = 0.f;
    float m = -INFINITY, z = 0.f;
    if (nkt > 0) {
        stage_head<DK>(ks[0], kh, ld, 0, min(kTK, jend + 1));
        stage_head<DK>(vs[0], vh, ld, 0, min(kTK, jend + 1));
        cp_commit();
    }
    for (int t = 0; t < nkt; ++t) {
        const int j0 = t * kTK;
        if (t + 1 < nkt) {
            const int n = min(kTK, jend + 1 - (j0 + kTK));
            stage_head<DK>(ks[(t + 1) & 1], kh, ld, j0 + kTK, n);
            stage_head<DK>(vs[(t + 1) & 1], vh, ld, j0 + kTK, n);
            cp_commit();
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        const float* kt = ks[t & 1] + part * C::HO;
        const float* vt = vs[t & 1] + part * C::HO;
        const int jhi = min(j0 + kTK - 1, jmax);
        for (int j = j0; j <= jhi; ++j) {                           // warp-uniform bounds
            float s = row_sum<C::SP>(dot_sm<C::DL>(qi, kt + (j - j0) * C::S)) * scale2;
            if (j > ii) s = -INFINITY;
            if (__any_sync(B2R_FULL_MASK, s > m)) {
                const float mn = fmaxf(m, s);
                const float a = exp2f(m - mn);
                z *= a;
#pragma unroll
                for (int c = 0; c < C::DL; ++c) acc[c] *= a;
                m = mn;
            }
            const float p = exp2f(s - m);
            z += p;
            axpy_sm<C::DL>(acc, p, vt + (j - j0) * C::S);
        }
        __syncthreads();                                            // slot t & 1 is refilled at t + 1
    }
    if (i < L) {
        const float inv = 1.f / z;
#pragma unroll
        for (int c = 0; c < C::DL; ++c) acc[c] *= inv;
        store_or_zero<C::DL>(ctx + (row0 + i) * d + h * DK + part * C::DL, acc, active);
        if (active && part == 0) lse[(row0 + i) * H + h] = m + log2f(z);
    }
}

template <int DK>
__global__ void __launch_bounds__(kTW * 32)
k_attention_bwd_dq_tiled(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                         const int64_t* __restrict__ live, const float* __restrict__ out, const float* __restrict__ lse,
                         const float* __restrict__ dctx, float* __restrict__ dq, float* __restrict__ delta_ws, int ldg,
                         int B, int L, int d, int H, int ntiles, float scale2, float scale) {
    using C = TiledCfg<DK>;
    __shared__ __align__(16) float ks[2][kTK * C::S];
    __shared__ __align__(16) float vs[2][kTK * C::S];
    const TileId id = tile_id(B, H, ntiles, true);
    const int b = id.b, h = id.h, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int part = lane % C::SP;
    const int64_t row0 = (int64_t)b * L;
    const int Lq = live_rows(live, b, L);
    const int r_t = id.tile * C::TR, r_w = r_t + warp * C::RPW;
    const int i = r_w + lane / C::SP;
    const bool active = i < Lq;
    const int ii = active ? i : Lq - 1;
    const int jend = min(Lq - 1, r_t + C::TR - 1);
    const int jmax = r_w < Lq ? min(Lq - 1, r_w + C::RPW - 1) : -1;
    const int nkt = r_t < Lq ? jend / kTK + 1 : 0;
    const float* kh = k + row0 * ld + h * DK;
    const float* vh = v + row0 * ld + h * DK;
    float qi[C::DL], gi[C::DL], acc[C::DL];
    float delta = 0.f, l2 = 0.f;
    if (r_w < Lq) {
        const int64_t col = h * DK + part * C::DL;
        load_vec<C::DL>(qi, q + (row0 + ii) * ld + col);
        load_vec<C::DL>(gi, dctx + (row0 + ii) * d + col);
        const float* oi = out + (row0 + ii) * d + col;
#pragma unroll
        for (int c = 0; c < C::DL; c += 4) delta += dot4(make_float4(gi[c], gi[c + 1], gi[c + 2], gi[c + 3]), ld_row4(oi + c));
        delta = row_sum<C::SP>(delta);
        l2 = lse[(row0 + ii) * H + h];
        if (active && part == 0) delta_ws[(row0 + i) * H + h] = delta;
    }
#pragma unroll
    for (int c = 0; c < C::DL; ++c) acc[c] = 0.f;
    if (nkt > 0) {
        stage_head<DK>(ks[0], kh, ld, 0, min(kTK, jend + 1));
        stage_head<DK>(vs[0], vh, ld, 0, min(kTK, jend + 1));
        cp_commit();
    }
    for (int t = 0; t < nkt; ++t) {
        const int j0 = t * kTK;
        if (t + 1 < nkt) {
            const int n = min(kTK, jend + 1 - (j0 + kTK));
            stage_head<DK>(ks[(t + 1) & 1], kh, ld, j0 + kTK, n);
            stage_head<DK>(vs[(t + 1) & 1], vh, ld, j0 + kTK, n);
            cp_commit();
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        const float* kt = ks[t & 1] + part * C::HO;
        const float* vt = vs[t & 1] + part * C::HO;
        const int jhi = min(j0 + kTK - 1, jmax);
        for (int j = j0; j <= jhi; ++j) {
            const float* kj = kt + (j - j0) * C::S;
            const float s = row_sum<C::SP>(dot_sm<C::DL>(qi, kj)) * scale2;
            const float p = j <= ii ? exp2f(s - l2) : 0.f;
            const float dp = row_sum<C::SP>(dot_sm<C::DL>(gi, vt + (j - j0) * C::S));
            axpy_sm<C::DL>(acc, p * (dp - delta), kj);
        }
        __syncthreads();
    }
    if (i < L) {
#pragma unroll
        for (int c = 0; c < C::DL; ++c) acc[c] *= scale;
        store_or_zero<C::DL>(dq + (row0 + i) * ldg + h * DK + part * C::DL, acc, active);
    }
}

template <int DK>
__global__ void __launch_bounds__(kTW * 32)
k_attention_bwd_dkv_tiled(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                          const int64_t* __restrict__ live, const float* __restrict__ lse,
                          const float* __restrict__ delta_ws, const float* __restrict__ dctx, float* __restrict__ dk_,
                          float* __restrict__ dv, int ldg, int B, int L, int d, int H, int ntiles, float scale2,
                          float scale) {
    using C = TiledCfg<DK>;
    __shared__ __align__(16) float qs[2][kTK * C::S];
    __shared__ __align__(16) float gs[2][kTK * C::S];
    __shared__ float2 ls[2][kTK];                                   // (lse_i, delta_i)
    const TileId id = tile_id(B, H, ntiles, false);                 // key tile 0 meets every query
    const int b = id.b, h = id.h, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int part = lane % C::SP;
    const int64_t row0 = (int64_t)b * L;
    const int Lq = live_rows(live, b, L);
    const int r_t = id.tile * C::TR, r_w = r_t + warp * C::RPW;
    const int j = r_w + lane / C::SP;
    const bool active = j < Lq;
    const int jj = active ? j : Lq - 1;
    const int nqt = r_t < Lq ? (Lq - r_t + kTK - 1) / kTK : 0;
    const float* qh = q + row0 * ld + h * DK;
    const float* gh = dctx + row0 * d + h * DK;
    float kj[C::DL], vj[C::DL], dka[C::DL], dva[C::DL];
    if (r_w < Lq) {
        const int64_t col = h * DK + part * C::DL;
        load_vec<C::DL>(kj, k + (row0 + jj) * ld + col);
        load_vec<C::DL>(vj, v + (row0 + jj) * ld + col);
    }
#pragma unroll
    for (int c = 0; c < C::DL; ++c) { dka[c] = 0.f; dva[c] = 0.f; }
    auto stage = [&](int slot, int i0) {
        const int n = min(kTK, Lq - i0);
        stage_head<DK>(qs[slot], qh, ld, i0, n);
        stage_head<DK>(gs[slot], gh, d, i0, n);
        for (int r = threadIdx.x; r < n; r += kTW * 32) {
            const int64_t e = (row0 + i0 + r) * H + h;
            ls[slot][r] = make_float2(lse[e], delta_ws[e]);
        }
        cp_commit();
    };
    if (nqt > 0) stage(0, r_t);
    for (int t = 0; t < nqt; ++t) {
        const int i0 = r_t + t * kTK;
        if (t + 1 < nqt) {
            stage((t + 1) & 1, i0 + kTK);
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        const float* qt = qs[t & 1] + part * C::HO;
        const float* gt = gs[t & 1] + part * C::HO;
        const int ilo = max(i0, r_w), ihi = min(i0 + kTK, Lq);
        for (int i = ilo; i < ihi; ++i) {                           // warp-uniform bounds
            const float* qi = qt + (i - i0) * C::S;
            const float* gi = gt + (i - i0) * C::S;
            const float2 ldi = ls[t & 1][i - i0];
            const float s = row_sum<C::SP>(dot_sm<C::DL>(kj, qi)) * scale2;
            const float p = jj <= i ? exp2f(s - ldi.x) : 0.f;
            const float dp = row_sum<C::SP>(dot_sm<C::DL>(vj, gi));
            axpy_sm<C::DL>(dva, p, gi);
            axpy_sm<C::DL>(dka, p * (dp - ldi.y), qi);
        }
        __syncthreads();
    }
    if (j < L) {
#pragma unroll
        for (int c = 0; c < C::DL; ++c) dka[c] *= scale;
        const int64_t col = h * DK + part * C::DL;
        store_or_zero<C::DL>(dk_ + (row0 + j) * ldg + col, dka, active);
        store_or_zero<C::DL>(dv + (row0 + j) * ldg + col, dva, active);
    }
}

}  // namespace b2r

using namespace b2r;

#define TILED_DISPATCH(dk, ...)                                  \
    switch (dk) {                                                \
        case 8:  { constexpr int DK = 8;  __VA_ARGS__; } break;  \
        case 16: { constexpr int DK = 16; __VA_ARGS__; } break;  \
        case 32: { constexpr int DK = 32; __VA_ARGS__; } break;  \
        default: { constexpr int DK = 64; __VA_ARGS__; } break;  \
    }

static int tiled_rows(int dk) { return dk > 32 ? kTW * 16 : kTW * 32; }

extern "C" size_t b2r_attention_bwd_tiled_workspace_bytes(int B, int L, int H) {
    if (B <= 0 || L <= 0 || H <= 0) return 0;
    return align_up((size_t)B * L * H * sizeof(float), 256);
}

extern "C" int b2r_attention_fwd_tiled(const float* q, const float* k, const float* v, int ld, const int64_t* live,
                                       float* ctx, float* lse, int B, int L, int d, int H, b2r_stream_t stream) {
    B2R_REQUIRE(q && k && v && ctx && lse, B2R_E_BADARG, "b2r_attention_fwd_tiled: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && d > 0 && ld >= d, B2R_E_BADARG, "b2r_attention_fwd_tiled: bad shape B=%d L=%d d=%d ld=%d",
                B, L, d, ld);
    if (!tiled_shape_ok(L, d, H, ld) || !aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(ctx))
        return b2r::set_error(B2R_E_UNSUPPORTED,
                              "b2r_attention_fwd_tiled: L=%d d=%d H=%d ld=%d not covered (d/H in {8, 16, 32, 64}, d <= %d, "
                              "L <= %d, d and ld multiples of 4, 16-byte aligned)", L, d, H, ld, kLNMaxD, kTiledMaxL);
    if (B == 0) return 0;
    const int dk = d / H, ntiles = (L + tiled_rows(dk) - 1) / tiled_rows(dk);
    B2R_REQUIRE((int64_t)ntiles * B * H <= INT32_MAX, B2R_E_UNSUPPORTED, "b2r_attention_fwd_tiled: B=%d L=%d H=%d: grid too large",
                B, L, H);
    const float scale2 = kLog2e / sqrtf((float)dk);
    TILED_DISPATCH(dk, {
        k_attention_fwd_tiled<DK><<<ntiles * B * H, kTW * 32, 0, as_stream(stream)>>>(q, k, v, ld, live, ctx, lse, B, L, d,
                                                                                      H, ntiles, scale2);
    });
    B2R_LAUNCH_OK("k_attention_fwd_tiled");
    return 0;
}

extern "C" int b2r_attention_bwd_tiled(const float* q, const float* k, const float* v, int ld, const int64_t* live,
                                       const float* ctx, const float* lse, const float* dctx, float* dq, float* dk,
                                       float* dv, int ldg, int B, int L, int d, int H, void* ws, size_t ws_bytes,
                                       b2r_stream_t stream) {
    B2R_REQUIRE(q && k && v && ctx && lse && dctx && dq && dk && dv && (ws || B == 0), B2R_E_BADARG,
                "b2r_attention_bwd_tiled: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && d > 0 && ld >= d && ldg >= d, B2R_E_BADARG,
                "b2r_attention_bwd_tiled: bad shape B=%d L=%d d=%d", B, L, d);
    if (!tiled_shape_ok(L, d, H, ld) || ldg % 4 != 0 || !aligned16(q) || !aligned16(k) || !aligned16(v) ||
        !aligned16(ctx) || !aligned16(dctx) || !aligned16(dq) || !aligned16(dk) || !aligned16(dv))
        return b2r::set_error(B2R_E_UNSUPPORTED,
                              "b2r_attention_bwd_tiled: L=%d d=%d H=%d not covered (d/H in {8, 16, 32, 64}, d <= %d, "
                              "L <= %d, d, ld and ldg multiples of 4, 16-byte aligned)", L, d, H, kLNMaxD, kTiledMaxL);
    B2R_REQUIRE(ws_bytes >= b2r_attention_bwd_tiled_workspace_bytes(B, L, H), B2R_E_WORKSPACE,
                "b2r_attention_bwd_tiled: workspace too small");
    if (B == 0) return 0;
    const int dk_ = d / H, ntiles = (L + tiled_rows(dk_) - 1) / tiled_rows(dk_);
    B2R_REQUIRE((int64_t)ntiles * B * H <= INT32_MAX, B2R_E_UNSUPPORTED, "b2r_attention_bwd_tiled: B=%d L=%d H=%d: grid too large",
                B, L, H);
    const float scale = 1.f / sqrtf((float)dk_);
    float* delta = static_cast<float*>(ws);
    cudaStream_t s = as_stream(stream);
    TILED_DISPATCH(dk_, {
        k_attention_bwd_dq_tiled<DK><<<ntiles * B * H, kTW * 32, 0, s>>>(q, k, v, ld, live, ctx, lse, dctx, dq, delta, ldg,
                                                                         B, L, d, H, ntiles, kLog2e * scale, scale);
    });
    B2R_LAUNCH_OK("k_attention_bwd_dq_tiled");
    TILED_DISPATCH(dk_, {
        k_attention_bwd_dkv_tiled<DK><<<ntiles * B * H, kTW * 32, 0, s>>>(q, k, v, ld, live, lse, delta, dctx, dk, dv, ldg,
                                                                          B, L, d, H, ntiles, kLog2e * scale, scale);
    });
    B2R_LAUNCH_OK("k_attention_bwd_dkv_tiled");
    return 0;
}
