// attention_rt.cu -- causal multi-head attention of SASRec (utils/layers.py:52-63, models/sequential/SASRec.py:68-72),
// forward and backward, with the per-(row, head) state held in REGISTERS.
//
// attention.cu's first kernels keep q, k, v in shared memory and read two shared operands per FMA: they are bound by the
// shared-memory pipe at ~10x (forward) and ~17x (backward) their HBM time.  Here one lane owns one (row, head):
//   forward           lane = query i : q_i[dk] and the output accumulator in registers, k_j / v_j arrive as broadcast
//                     128-bit shared loads (one wavefront per load, 8 loads per 2*dk FMAs), online softmax per lane,
//                     no cross-lane traffic at all; the row's log-sum-exp (base 2) is kept for the backward;
//   backward pass 2   lane = query i : dQ_i = scale * sum_j dS_ij k_j with dS_ij = p_ij (dO_i.v_j - delta_i),
//                     p_ij = 2^(s_ij - lse_i) recomputed from the saved lse, delta_i = dO_i.O_i (the softmax-Jacobian row
//                     term, from the saved output) -- again lane-local;
//   backward pass 1   lane = key j   : dK_j += dS_ij q_i, dV_j += p_ij dO_i accumulated in registers while q_i / dO_i /
//                     (lse_i, delta_i) are broadcast.
// One CTA per sequence, 8 warps = (head, 32-row block) work items; q/k/v/dO rows of the sequence are staged in shared
// memory with coalesced 128-bit loads and results leave through shared memory the same way.  `live` (optional): rows
// t >= live[b] are dead (nothing downstream reads them; their upstream gradient is zero): skipped, outputs written as
// zeros -- same contract as attention.cu.
#include "common.cuh"
#include "seq_limits.cuh"
#include "attention_lane.cuh"

namespace b2r {

// rows [0, n) of one [L, d] operand of sequence b: global (row stride ld) -> shared (row stride S)
__device__ __forceinline__ void stage_in(float* dst, int S, const float* src, int64_t row0, int ld, int n, int d4) {
    for (int e = threadIdx.x; e < n * d4; e += 256) {
        const int t = e / d4, c = (e - t * d4) * 4;
        st4(dst + t * S + c, ld_row4(src + (row0 + t) * ld + c));
    }
}

// rows [0, n) shared -> global, then rows [n, L) = 0
__device__ __forceinline__ void stage_out(float* dst, int64_t row0, int ld, const float* src, int S, int n, int L, int d4) {
    for (int e = threadIdx.x; e < L * d4; e += 256) {
        const int t = e / d4, c = (e - t * d4) * 4;
        st4(dst + (row0 + t) * ld + c, t < n ? ld4(src + t * S + c) : make_float4(0.f, 0.f, 0.f, 0.f));
    }
}

template <int DK>
__global__ void __launch_bounds__(256)
k_attention_fwd_rt(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                   const int64_t* __restrict__ live, float* __restrict__ ctx, float* __restrict__ lse, int L, int d, int H,
                   float scale2) {
    extern __shared__ __align__(16) float sm[];
    const int S = d + 4;                       // 16-byte aligned rows; lane-strided 128-bit accesses stay conflict-free
    float* qs = sm;                            // [L][S]  (q rows; the (i, h) slot is reused for that lane's output)
    float* ks = qs + L * S;
    float* vs = ks + L * S;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, d4 = d >> 2;
    const int64_t row0 = (int64_t)b * L;
    const int Lb = live_rows(live, b, L);
    stage_in(qs, S, q, row0, ld, Lb, d4);
    stage_in(ks, S, k, row0, ld, Lb, d4);
    stage_in(vs, S, v, row0, ld, Lb, d4);
    __syncthreads();
    const int NB = (Lb + 31) >> 5;
    for (int item = warp; item < H * NB; item += 8) {
        const int h = item % H, blk = item / H;
        const int i = blk * 32 + lane;
        const bool active = i < Lb;
        const int ii = active ? i : Lb - 1;
        float qi[DK], acc[DK];
        load_vec<DK>(qi, qs + ii * S + h * DK);
#pragma unroll
        for (int c = 0; c < DK; ++c) acc[c] = 0.f;
        float m = -INFINITY, z = 0.f;
        const int jmax = min(Lb - 1, blk * 32 + 31);
        for (int j = 0; j <= jmax; ++j) {
            float s = dot_sm<DK>(qi, ks + j * S + h * DK) * scale2;
            if (j > ii) s = -INFINITY;
            if (__any_sync(B2R_FULL_MASK, s > m)) {          // some lane's running max moves: rescale (rare after a few keys)
                const float mn = fmaxf(m, s);
                const float a = exp2f(m - mn);               // j = 0: m = -inf, mn finite (key 0 is visible to every row)
                z *= a;
#pragma unroll
                for (int c = 0; c < DK; ++c) acc[c] *= a;
                m = mn;
            }
            const float p = exp2f(s - m);
            z += p;
            axpy_sm<DK>(acc, p, vs + j * S + h * DK);
        }
        const float inv = 1.f / z;
#pragma unroll
        for (int c = 0; c < DK; ++c) acc[c] *= inv;
        if (active) {
            store_vec<DK>(qs + i * S + h * DK, acc);         // only this lane ever reads or writes slot (i, h)
            lse[(row0 + i) * H + h] = m + log2f(z);
        }
    }
    __syncthreads();
    stage_out(ctx, row0, d, qs, S, Lb, L, d4);
}

template <int DK>
__global__ void __launch_bounds__(256)
k_attention_bwd_rt(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                   const int64_t* __restrict__ live, const float* __restrict__ out, const float* __restrict__ lse,
                   const float* __restrict__ dctx, float* __restrict__ dq, float* __restrict__ dk_, float* __restrict__ dv,
                   int ldg, int L, int d, int H, float scale2, float scale) {
    extern __shared__ __align__(16) float sm[];
    const int S = d + 4;
    float* qs = sm;
    float* ks = qs + L * S;                    // k rows, then dK
    float* vs = ks + L * S;                    // v rows, then dV
    float* gs = vs + L * S;                    // dO rows
    float* os = gs + L * S;                    // dQ
    float2* ld2 = reinterpret_cast<float2*>(os + L * S);     // [L][H] (lse_i, delta_i)
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, d4 = d >> 2;
    const int64_t row0 = (int64_t)b * L;
    const int Lq = live_rows(live, b, L);
    stage_in(qs, S, q, row0, ld, Lq, d4);
    stage_in(ks, S, k, row0, ld, Lq, d4);
    stage_in(vs, S, v, row0, ld, Lq, d4);
    stage_in(gs, S, dctx, row0, d, Lq, d4);
    __syncthreads();
    const int NB = (Lq + 31) >> 5;
    // pass 2: lane = query row
    for (int item = warp; item < H * NB; item += 8) {
        const int h = item % H, blk = item / H;
        const int i = blk * 32 + lane;
        const bool active = i < Lq;
        const int ii = active ? i : Lq - 1;
        float qi[DK], gi[DK], acc[DK];
        load_vec<DK>(qi, qs + ii * S + h * DK);
        load_vec<DK>(gi, gs + ii * S + h * DK);
        float delta = 0.f;
        {
            const float* oi = out + (row0 + ii) * d + h * DK;
#pragma unroll
            for (int c = 0; c < DK; c += 4) delta += dot4(make_float4(gi[c], gi[c + 1], gi[c + 2], gi[c + 3]), ld_row4(oi + c));
        }
        const float l2 = lse[(row0 + ii) * H + h];
        if (active) ld2[i * H + h] = make_float2(l2, delta);
#pragma unroll
        for (int c = 0; c < DK; ++c) acc[c] = 0.f;
        const int jmax = min(Lq - 1, blk * 32 + 31);
        for (int j = 0; j <= jmax; ++j) {
            const float* kj = ks + j * S + h * DK;
            const float s = dot_sm<DK>(qi, kj) * scale2;
            const float p = j <= ii ? exp2f(s - l2) : 0.f;
            const float dp = dot_sm<DK>(gi, vs + j * S + h * DK);
            axpy_sm<DK>(acc, p * (dp - delta), kj);
        }
#pragma unroll
        for (int c = 0; c < DK; ++c) acc[c] *= scale;
        if (active) store_vec<DK>(os + i * S + h * DK, acc);
    }
    __syncthreads();
    // pass 1: lane = key row; queries i >= the block's first key
    for (int item = warp; item < H * NB; item += 8) {
        const int h = item % H, blk = item / H;
        const int j = blk * 32 + lane;
        const bool active = j < Lq;
        const int jj = active ? j : Lq - 1;
        float kj[DK], vj[DK], dka[DK], dva[DK];
        load_vec<DK>(kj, ks + jj * S + h * DK);
        load_vec<DK>(vj, vs + jj * S + h * DK);
#pragma unroll
        for (int c = 0; c < DK; ++c) { dka[c] = 0.f; dva[c] = 0.f; }
        for (int i = blk * 32; i < Lq; ++i) {
            const float* qi = qs + i * S + h * DK;
            const float* gi = gs + i * S + h * DK;
            const float2 ldi = ld2[i * H + h];
            const float s = dot_sm<DK>(kj, qi) * scale2;
            const float p = jj <= i ? exp2f(s - ldi.x) : 0.f;
            const float dp = dot_sm<DK>(vj, gi);
            axpy_sm<DK>(dva, p, gi);
            axpy_sm<DK>(dka, p * (dp - ldi.y), qi);
        }
#pragma unroll
        for (int c = 0; c < DK; ++c) dka[c] *= scale;
        if (active) {
            store_vec<DK>(ks + j * S + h * DK, dka);          // slot (j, h) belongs to this lane alone in this pass
            store_vec<DK>(vs + j * S + h * DK, dva);
        }
    }
    __syncthreads();
    stage_out(dq, row0, ldg, os, S, Lq, L, d4);
    stage_out(dk_, row0, ldg, ks, S, Lq, L, d4);
    stage_out(dv, row0, ldg, vs, S, Lq, L, d4);
}

}  // namespace b2r

using namespace b2r;

#define RT_DISPATCH(dk, ...)                                     \
    switch (dk) {                                                \
        case 8:  { constexpr int DK = 8;  __VA_ARGS__; } break;  \
        case 16: { constexpr int DK = 16; __VA_ARGS__; } break;  \
        default: { constexpr int DK = 32; __VA_ARGS__; } break;  \
    }

extern "C" int b2r_attention_fwd_rt(const float* q, const float* k, const float* v, int ld, const int64_t* live, float* ctx,
                                    float* lse, int B, int L, int d, int H, b2r_stream_t stream) {
    B2R_REQUIRE(q && k && v && ctx && lse, B2R_E_BADARG, "b2r_attention_fwd_rt: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && d > 0 && ld >= d, B2R_E_BADARG, "b2r_attention_fwd_rt: bad shape B=%d L=%d d=%d ld=%d", B, L, d, ld);
    const size_t smem = rt_fwd_smem(L, d);
    if (!rt_shape_ok(L, d, H, ld) || smem > kAttnSmemMax || !aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(ctx))
        return b2r::set_error(B2R_E_UNSUPPORTED, "b2r_attention_fwd_rt: L=%d d=%d H=%d ld=%d not covered (use b2r_attention_fwd_live)", L, d, H, ld);
    if (B == 0) return 0;
    const float scale2 = kLog2e / sqrtf((float)(d / H));
    RT_DISPATCH(d / H, {
        B2R_CUDA_OK(cudaFuncSetAttribute(k_attention_fwd_rt<DK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_attention_fwd_rt<DK><<<B, 256, smem, as_stream(stream)>>>(q, k, v, ld, live, ctx, lse, L, d, H, scale2);
    });
    B2R_LAUNCH_OK("k_attention_fwd_rt");
    return 0;
}

extern "C" int b2r_attention_bwd_rt(const float* q, const float* k, const float* v, int ld, const int64_t* live,
                                    const float* ctx, const float* lse, const float* dctx, float* dq, float* dk, float* dv,
                                    int ldg, int B, int L, int d, int H, b2r_stream_t stream) {
    B2R_REQUIRE(q && k && v && ctx && lse && dctx && dq && dk && dv, B2R_E_BADARG, "b2r_attention_bwd_rt: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && d > 0 && ld >= d && ldg >= d, B2R_E_BADARG, "b2r_attention_bwd_rt: bad shape B=%d L=%d d=%d", B, L, d);
    const size_t smem = rt_bwd_smem(L, d, H);
    if (!rt_shape_ok(L, d, H, ld) || ldg % 4 != 0 || smem > kAttnSmemMax || !aligned16(q) || !aligned16(k) || !aligned16(v) ||
        !aligned16(ctx) || !aligned16(dctx) || !aligned16(dq) || !aligned16(dk) || !aligned16(dv))
        return b2r::set_error(B2R_E_UNSUPPORTED, "b2r_attention_bwd_rt: L=%d d=%d H=%d not covered (use b2r_attention_bwd_live)", L, d, H);
    if (B == 0) return 0;
    const float scale = 1.f / sqrtf((float)(d / H));
    RT_DISPATCH(d / H, {
        B2R_CUDA_OK(cudaFuncSetAttribute(k_attention_bwd_rt<DK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_attention_bwd_rt<DK><<<B, 256, smem, as_stream(stream)>>>(q, k, v, ld, live, ctx, lse, dctx, dq, dk, dv, ldg, L, d, H,
                                                                    kLog2e * scale, scale);
    });
    B2R_LAUNCH_OK("k_attention_bwd_rt");
    return 0;
}
