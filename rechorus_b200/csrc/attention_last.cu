// attention_last.cu -- SASRec's last block for one query per sequence.  Batch widths up to kALMaxL = 256 (seq_limits.cuh)
// with the score row in shared memory; the _tiled entry points keep it in global memory instead (the prob output in the
// forward, a workspace row in the backward) and take widths up to kTiledMaxL with the same per-lane arithmetic.
//
// SASRec scores candidates against ONE vector per sequence: the encoder state at position len-1 of the LAST block
// (models/sequential/SASRec.py:74-81).  Every other position of the last block's output is dead, so for that block
// only one query per sequence has to go through attention, the residual LayerNorms and the FFN -- keys and values
// still come from all positions.  The result is identical to the full computation (nothing is approximated); the
// last block's cost drops from five [B*L, d] GEMMs + full attention to two (K and V) plus work on [B, d].
//
//   k_attention_last_fwd  one warp per (sequence, head): scores of the query at t* = clamp(len-1) against keys 0..t*
//                         (the causal row of utils/layers.py:52-63), softmax, context; the probabilities are kept
//   k_attention_last_bwd  same decomposition: dV = p (x) dctx, dS = p * (dP - <p, dP>), dq = scale * dS K,
//                         dK = scale * dS (x) q; rows beyond t* get exact zeros.  Every element has one writer.
#include "common.cuh"
#include "seq_limits.cuh"

namespace b2r {

constexpr int kALWarps = 8;

// One warp per (sequence, head).  kRowInProb: the score row lives in prob (global, the tiled form); otherwise in `ps`.
template <bool kRowInProb>
__device__ __forceinline__ void attention_last_fwd_body(const float* __restrict__ q, const float* __restrict__ k,
                                                        const float* __restrict__ v, int ld, const int64_t* __restrict__ lengths,
                                                        float* __restrict__ ctx, float* prob, int B, int L, int d, int H,
                                                        float scale, float* ps_warp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dk = d / H;
    const int64_t total = (int64_t)B * H;
    for (int64_t w = (int64_t)blockIdx.x * kALWarps + warp; w < total; w += (int64_t)gridDim.x * kALWarps) {
        const int b = (int)(w / H), h = (int)(w % H);
        int64_t tl = lengths[b] - 1;
        tl = tl < 0 ? 0 : (tl >= L ? L - 1 : tl);
        const int n = (int)tl + 1;                                   // keys 0 .. t*
        const float* qh = q + (int64_t)b * d + h * dk;
        float* pout = prob + ((int64_t)b * H + h) * L;
        float* row = kRowInProb ? pout : ps_warp;
        float mx = -INFINITY;
        for (int j = lane; j < n; j += 32) {
            const float* kj = k + ((int64_t)b * L + j) * ld + h * dk;
            float s = 0.f;
            for (int c = 0; c < dk; ++c) s = fmaf(qh[c], kj[c], s);
            s *= scale;
            row[j] = s;
            mx = fmaxf(mx, s);
        }
        mx = warp_max(mx);
        float z = 0.f;
        for (int j = lane; j < n; j += 32) {
            const float e = expf(row[j] - mx);
            row[j] = e;
            z += e;
        }
        z = warp_sum(z);
        const float inv = 1.f / z;
        for (int j = lane; j < L; j += 32) {
            const float p = j < n ? row[j] * inv : 0.f;
            if (!kRowInProb && j < n) row[j] = p;
            pout[j] = p;
        }
        __syncwarp();
        for (int c = lane; c < dk; c += 32) {
            float a = 0.f;
            for (int j = 0; j < n; ++j) a = fmaf(row[j], v[((int64_t)b * L + j) * ld + h * dk + c], a);
            ctx[(int64_t)b * d + h * dk + c] = a;
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(kALWarps * 32)
k_attention_last_fwd(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                     const int64_t* __restrict__ lengths, float* __restrict__ ctx, float* __restrict__ prob, int B, int L,
                     int d, int H, float scale) {
    __shared__ float ps[kALWarps][kALMaxL];
    attention_last_fwd_body<false>(q, k, v, ld, lengths, ctx, prob, B, L, d, H, scale, ps[threadIdx.x >> 5]);
}

__global__ void __launch_bounds__(kALWarps * 32)
k_attention_last_fwd_tiled(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                           const int64_t* __restrict__ lengths, float* __restrict__ ctx, float* prob, int B, int L, int d,
                           int H, float scale) {
    attention_last_fwd_body<true>(q, k, v, ld, lengths, ctx, prob, B, L, d, H, scale, nullptr);
}

// gs_rows: one [L] row per (sequence, head) in global memory (the tiled form), else nullptr and the row is `gs_warp`
__device__ __forceinline__ void attention_last_bwd_body(const float* __restrict__ q, const float* __restrict__ k,
                                                        const float* __restrict__ v, int ld, const int64_t* __restrict__ lengths,
                                                        const float* __restrict__ prob, const float* __restrict__ dctx,
                                                        float* __restrict__ dq, float* __restrict__ dk_, float* __restrict__ dv,
                                                        int ldg, int B, int L, int d, int H, float scale, float* gs_warp,
                                                        float* gs_rows) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dk = d / H;
    const int64_t total = (int64_t)B * H;
    for (int64_t w = (int64_t)blockIdx.x * kALWarps + warp; w < total; w += (int64_t)gridDim.x * kALWarps) {
        const int b = (int)(w / H), h = (int)(w % H);
        int64_t tl = lengths[b] - 1;
        tl = tl < 0 ? 0 : (tl >= L ? L - 1 : tl);
        const int n = (int)tl + 1;
        const float* qh = q + (int64_t)b * d + h * dk;
        const float* gh = dctx + (int64_t)b * d + h * dk;
        const float* ph = prob + ((int64_t)b * H + h) * L;
        float* row = gs_rows != nullptr ? gs_rows + ((int64_t)b * H + h) * L : gs_warp;
        // dP_j = <dctx, v_j>;  acc = sum_j p_j dP_j
        float acc = 0.f;
        for (int j = lane; j < n; j += 32) {
            const float* vj = v + ((int64_t)b * L + j) * ld + h * dk;
            float dp = 0.f;
            for (int c = 0; c < dk; ++c) dp = fmaf(gh[c], vj[c], dp);
            row[j] = dp;
            acc = fmaf(ph[j], dp, acc);
        }
        acc = warp_sum(acc);
        // dS_j = p_j (dP_j - acc); rows of dK, dV (zeros beyond t*)
        for (int j = lane; j < L; j += 32) {
            float* dkj = dk_ + ((int64_t)b * L + j) * ldg + h * dk;
            float* dvj = dv + ((int64_t)b * L + j) * ldg + h * dk;
            if (j < n) {
                const float p = ph[j];
                const float g = p * (row[j] - acc) * scale;          // d loss / d (q . k_j)
                row[j] = g;
                for (int c = 0; c < dk; ++c) {
                    dkj[c] = g * qh[c];
                    dvj[c] = p * gh[c];
                }
            } else {
                for (int c = 0; c < dk; ++c) {
                    dkj[c] = 0.f;
                    dvj[c] = 0.f;
                }
            }
        }
        __syncwarp();
        for (int c = lane; c < dk; c += 32) {
            float a = 0.f;
            for (int j = 0; j < n; ++j) a = fmaf(row[j], k[((int64_t)b * L + j) * ld + h * dk + c], a);
            dq[(int64_t)b * d + h * dk + c] = a;
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(kALWarps * 32)
k_attention_last_bwd(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                     const int64_t* __restrict__ lengths, const float* __restrict__ prob, const float* __restrict__ dctx,
                     float* __restrict__ dq, float* __restrict__ dk_, float* __restrict__ dv, int ldg, int B, int L, int d,
                     int H, float scale) {
    __shared__ float gs[kALWarps][kALMaxL];
    attention_last_bwd_body(q, k, v, ld, lengths, prob, dctx, dq, dk_, dv, ldg, B, L, d, H, scale, gs[threadIdx.x >> 5],
                            nullptr);
}

__global__ void __launch_bounds__(kALWarps * 32)
k_attention_last_bwd_tiled(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                           const int64_t* __restrict__ lengths, const float* __restrict__ prob,
                           const float* __restrict__ dctx, float* __restrict__ dq, float* __restrict__ dk_,
                           float* __restrict__ dv, int ldg, int B, int L, int d, int H, float scale, float* rows) {
    attention_last_bwd_body(q, k, v, ld, lengths, prob, dctx, dq, dk_, dv, ldg, B, L, d, H, scale, nullptr, rows);
}

}  // namespace b2r

using namespace b2r;

static int al_grid(int64_t warps) {
    int64_t need = (warps + kALWarps - 1) / kALWarps;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (int)(need < cap ? need : cap);
}

extern "C" int b2r_attention_last_fwd(const float* q_last, const float* k, const float* v, int ld,
                                      const int64_t* lengths, float* ctx_last, float* prob, int B, int L, int d, int H,
                                      b2r_stream_t stream) {
    B2R_REQUIRE(q_last && k && v && lengths && ctx_last && prob, B2R_E_BADARG, "b2r_attention_last_fwd: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && L <= kALMaxL && d > 0 && H > 0 && d % H == 0 && ld >= d, B2R_E_BADARG,
                "b2r_attention_last_fwd: bad shape B=%d L=%d d=%d H=%d ld=%d", B, L, d, H, ld);
    if (B == 0) return 0;
    k_attention_last_fwd<<<al_grid((int64_t)B * H), kALWarps * 32, 0, as_stream(stream)>>>(
        q_last, k, v, ld, lengths, ctx_last, prob, B, L, d, H, 1.f / sqrtf((float)(d / H)));
    B2R_LAUNCH_OK("k_attention_last_fwd");
    return 0;
}

extern "C" int b2r_attention_last_bwd(const float* q_last, const float* k, const float* v, int ld,
                                      const int64_t* lengths, const float* prob, const float* dctx_last, float* dq_last,
                                      float* dk, float* dv, int ldg, int B, int L, int d, int H, b2r_stream_t stream) {
    B2R_REQUIRE(q_last && k && v && lengths && prob && dctx_last && dq_last && dk && dv, B2R_E_BADARG,
                "b2r_attention_last_bwd: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && L <= kALMaxL && d > 0 && H > 0 && d % H == 0 && ld >= d && ldg >= d, B2R_E_BADARG,
                "b2r_attention_last_bwd: bad shape B=%d L=%d d=%d H=%d", B, L, d, H);
    if (B == 0) return 0;
    k_attention_last_bwd<<<al_grid((int64_t)B * H), kALWarps * 32, 0, as_stream(stream)>>>(
        q_last, k, v, ld, lengths, prob, dctx_last, dq_last, dk, dv, ldg, B, L, d, H, 1.f / sqrtf((float)(d / H)));
    B2R_LAUNCH_OK("k_attention_last_bwd");
    return 0;
}

extern "C" int b2r_attention_last_fwd_tiled(const float* q_last, const float* k, const float* v, int ld,
                                            const int64_t* lengths, float* ctx_last, float* prob, int B, int L, int d, int H,
                                            b2r_stream_t stream) {
    B2R_REQUIRE(q_last && k && v && lengths && ctx_last && prob, B2R_E_BADARG, "b2r_attention_last_fwd_tiled: null pointer");
    B2R_REQUIRE(B >= 0 && tiled_last_shape_ok(L, d, H) && d > 0 && ld >= d, B2R_E_BADARG,
                "b2r_attention_last_fwd_tiled: bad shape B=%d L=%d d=%d H=%d ld=%d (1 <= L <= %d)", B, L, d, H, ld, kTiledMaxL);
    if (B == 0) return 0;
    k_attention_last_fwd_tiled<<<al_grid((int64_t)B * H), kALWarps * 32, 0, as_stream(stream)>>>(
        q_last, k, v, ld, lengths, ctx_last, prob, B, L, d, H, 1.f / sqrtf((float)(d / H)));
    B2R_LAUNCH_OK("k_attention_last_fwd_tiled");
    return 0;
}

extern "C" int b2r_attention_last_bwd_tiled(const float* q_last, const float* k, const float* v, int ld,
                                            const int64_t* lengths, const float* prob, const float* dctx_last,
                                            float* dq_last, float* dk, float* dv, int ldg, int B, int L, int d, int H,
                                            void* ws, size_t ws_bytes, b2r_stream_t stream) {
    B2R_REQUIRE(q_last && k && v && lengths && prob && dctx_last && dq_last && dk && dv && (ws || B == 0), B2R_E_BADARG,
                "b2r_attention_last_bwd_tiled: null pointer");
    B2R_REQUIRE(B >= 0 && tiled_last_shape_ok(L, d, H) && d > 0 && ld >= d && ldg >= d, B2R_E_BADARG,
                "b2r_attention_last_bwd_tiled: bad shape B=%d L=%d d=%d H=%d (1 <= L <= %d)", B, L, d, H, kTiledMaxL);
    B2R_REQUIRE(ws_bytes >= b2r_attention_bwd_tiled_workspace_bytes(B, L, H), B2R_E_WORKSPACE,
                "b2r_attention_last_bwd_tiled: workspace too small");
    if (B == 0) return 0;
    k_attention_last_bwd_tiled<<<al_grid((int64_t)B * H), kALWarps * 32, 0, as_stream(stream)>>>(
        q_last, k, v, ld, lengths, prob, dctx_last, dq_last, dk, dv, ldg, B, L, d, H, 1.f / sqrtf((float)(d / H)),
        static_cast<float*>(ws));
    B2R_LAUNCH_OK("k_attention_last_bwd_tiled");
    return 0;
}
