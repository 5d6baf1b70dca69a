// attention.cu -- SASRec sequence kernels (models/sequential/SASRec.py:58-76, utils/layers.py:52-63):
//   * history embedding + reversed-position embedding,
//   * causal multi-head attention forward and backward (no output projection, probabilities recomputed in
//     the backward instead of being stashed),
//   * last-valid-state select and its backward,
//   * gradient of a small, heavily shared table (the position table: ~B*L contributions into <= L+1 rows).
// One CTA owns one sequence: the whole per-sequence problem (q,k,v: 3 x L x d fp32 = 38 KB at L=50,d=64)
// lives in shared memory, the batch is the parallel dimension (SURVEY.md section 5: no sequence parallelism).
//
// Softmax note: the reference subtracts the max over the ENTIRE score tensor before the softmax
// (layers.py:60), a scalar shift that cancels; the kernels subtract the row max (same function, no
// cross-row underflow).  Fully masked rows cannot occur under the causal mask (key j = query i is allowed).
#include "common.cuh"
#include "seq_limits.cuh"

namespace b2r {

// x[r,:] = I[hist[r],:] + P[pos(r),:],  pos = (len[b] - t) * (hist[r] > 0)   (SASRec.py:58-66)
__global__ void __launch_bounds__(256)
k_embed_hist(const float* __restrict__ I, int64_t n_items, const float* __restrict__ P, int64_t n_pos,
             const int64_t* __restrict__ hist, const int64_t* __restrict__ lengths, float* __restrict__ x,
             int64_t* __restrict__ pos_out, int B, int L, int d, int32_t* err_flag) {
    const int lane = threadIdx.x & 31;
    const int d4 = d >> 2;
    const int64_t rows = (int64_t)B * L;
    for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * 8) {
        const int b = (int)(r / L), t = (int)(r % L);
        const int64_t id = checked_id(hist[r], n_items, lane == 0 ? err_flag : nullptr);
        const int64_t pos = checked_id((lengths[b] - t) * (id > 0 ? 1 : 0), n_pos, lane == 0 ? err_flag : nullptr);
        if (lane == 0 && pos_out != nullptr) pos_out[r] = pos;
        for (int k = lane; k < d4; k += 32) {
            const float4 a = ld_row4(I + id * d + k * 4);
            const float4 p = ld4(P + pos * d + k * 4);
            st4(x + r * d + k * 4, make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w));
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// attention forward: CTA per sequence.  q,k,v rows of the sequence at q/k/v + (b*L + t)*ld
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_attention_fwd(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                float* __restrict__ ctx, int L, int d, int H, float scale, const int64_t* __restrict__ live) {
    extern __shared__ float sm[];
    const int S = d + 1;                       // padded row stride: lanes index rows -> distinct banks
    float* qs = sm;                            // [L][S]
    float* ks = qs + L * S;
    float* vs = ks + L * S;
    float* ps = vs + L * S;                    // [8 warps][H][L]
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dk = d / H;
    for (int e = threadIdx.x; e < L * d; e += 256) {
        const int t = e / d, c = e % d;
        const int64_t g = ((int64_t)b * L + t) * ld + c;
        qs[t * S + c] = q[g];
        ks[t * S + c] = k[g];
        vs[t * S + c] = v[g];
    }
    __syncthreads();
    // live[b] (optional): rows t >= live[b] of this sequence are dead -- nothing downstream reads them (causal attention:
    // SASRec uses position len-1 only, SASRec.py:74-81); their context is written as zeros and their work is skipped
    int Lb = L;
    if (live != nullptr) {
        const int64_t lv = live[b];
        Lb = lv < 0 ? 0 : (lv > L ? L : (int)lv);
        for (int e = threadIdx.x; e < (L - Lb) * d; e += 256) ctx[((int64_t)b * L + Lb) * d + e] = 0.f;
    }
    float* pw = ps + warp * H * L;
    for (int i = warp; i < Lb; i += 8) {
        for (int h = 0; h < H; ++h) {
            const float* qi = qs + i * S + h * dk;
            float mx = -INFINITY;
            for (int j = lane; j <= i; j += 32) {
                const float* kj = ks + j * S + h * dk;
                float s = 0.f;
                for (int c = 0; c < dk; ++c) s = fmaf(qi[c], kj[c], s);
                s *= scale;
                pw[h * L + j] = s;
                mx = fmaxf(mx, s);
            }
            mx = warp_max(mx);
            float z = 0.f;
            for (int j = lane; j <= i; j += 32) {
                const float e = expf(pw[h * L + j] - mx);
                pw[h * L + j] = e;
                z += e;
            }
            z = warp_sum(z);
            const float inv = 1.f / z;
            for (int j = lane; j <= i; j += 32) pw[h * L + j] *= inv;
        }
        __syncwarp();
        for (int c = lane; c < d; c += 32) {
            const float* ph = pw + (c / dk) * L;
            float a = 0.f;
            for (int j = 0; j <= i; ++j) a = fmaf(ph[j], vs[j * S + c], a);
            ctx[((int64_t)b * L + i) * d + c] = a;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------
// attention backward: CTA per sequence; recomputes P, then dV, dS (in place of P), dQ, dK
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_attention_bwd(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, int ld,
                const float* __restrict__ dctx, float* __restrict__ dq, float* __restrict__ dk_, float* __restrict__ dv,
                int ldg, int L, int d, int H, float scale, const int64_t* __restrict__ live) {
    extern __shared__ float sm[];
    const int S = d + 1;
    const int LP = L + 1;
    float* qs = sm;
    float* ks = qs + L * S;
    float* vs = ks + L * S;
    float* gs = vs + L * S;                    // dctx
    float* P = gs + L * S;                     // [H][L][LP]
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dk = d / H;
    for (int e = threadIdx.x; e < L * d; e += 256) {
        const int t = e / d, c = e % d;
        const int64_t g = ((int64_t)b * L + t) * ld + c;
        qs[t * S + c] = q[g];
        ks[t * S + c] = k[g];
        vs[t * S + c] = v[g];
        gs[t * S + c] = dctx[((int64_t)b * L + t) * d + c];
    }
    __syncthreads();
    // dead rows (t >= live[b], see k_attention_fwd): their upstream gradient is zero by construction and so are the
    // gradients they would receive; every phase below runs over the live rows only (Lq = live length)
    int Lq = L;
    if (live != nullptr) {
        const int64_t lv = live[b];
        Lq = lv < 0 ? 0 : (lv > L ? L : (int)lv);
        for (int e = threadIdx.x; e < (L - Lq) * d; e += 256) {
            const int t = Lq + e / d, c = e % d;
            const int64_t g = ((int64_t)b * L + t) * ldg + c;
            dq[g] = 0.f;
            dk_[g] = 0.f;
            dv[g] = 0.f;
        }
    }
    // phase A: probabilities (zero above the diagonal)
    for (int i = warp; i < Lq; i += 8) {
        for (int h = 0; h < H; ++h) {
            float* pr = P + ((int64_t)h * L + i) * LP;
            const float* qi = qs + i * S + h * dk;
            float mx = -INFINITY;
            for (int j = lane; j < Lq; j += 32) {
                float s = -INFINITY;
                if (j <= i) {
                    const float* kj = ks + j * S + h * dk;
                    s = 0.f;
                    for (int c = 0; c < dk; ++c) s = fmaf(qi[c], kj[c], s);
                    s *= scale;
                }
                pr[j] = s;
                mx = fmaxf(mx, s);
            }
            mx = warp_max(mx);
            float z = 0.f;
            for (int j = lane; j < Lq; j += 32) {
                const float e = (j <= i) ? expf(pr[j] - mx) : 0.f;
                pr[j] = e;
                z += e;
            }
            z = warp_sum(z);
            const float inv = 1.f / z;
            for (int j = lane; j < Lq; j += 32) pr[j] *= inv;
        }
    }
    __syncthreads();
    // phase B: dV[j,c] = sum_{i>=j} P[h(c)][i][j] * dctx[i,c]
    for (int e = threadIdx.x; e < Lq * d; e += 256) {
        const int j = e / d, c = e % d;
        const float* ph = P + (int64_t)(c / dk) * L * LP;
        float a = 0.f;
        for (int i = j; i < Lq; ++i) a = fmaf(ph[i * LP + j], gs[i * S + c], a);
        dv[((int64_t)b * L + j) * ldg + c] = a;
    }
    __syncthreads();
    // phase C: dS = P * (dP - sum_j P dP) * scale, in place
    for (int i = warp; i < Lq; i += 8) {
        for (int h = 0; h < H; ++h) {
            float* pr = P + ((int64_t)h * L + i) * LP;
            const float* gi = gs + i * S + h * dk;
            float rs = 0.f;
            float dp_loc[4];                    // L <= 128 -> at most 4 keys per lane
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int j = lane + 32 * u;
                float dp = 0.f;
                if (j <= i) {
                    const float* vj = vs + j * S + h * dk;
                    for (int c = 0; c < dk; ++c) dp = fmaf(gi[c], vj[c], dp);
                    rs = fmaf(pr[j], dp, rs);
                }
                dp_loc[u] = dp;
            }
            rs = warp_sum(rs);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int j = lane + 32 * u;
                if (j <= i) pr[j] = pr[j] * (dp_loc[u] - rs) * scale;
            }
        }
    }
    __syncthreads();
    // phase D: dQ[i,c] = sum_{j<=i} dS[h][i][j] k[j,c];  dK[j,c] = sum_{i>=j} dS[h][i][j] q[i,c]
    for (int e = threadIdx.x; e < Lq * d; e += 256) {
        const int t = e / d, c = e % d;
        const float* ph = P + (int64_t)(c / dk) * L * LP;
        float aq = 0.f, ak = 0.f;
        for (int j = 0; j <= t; ++j) aq = fmaf(ph[t * LP + j], ks[j * S + c], aq);
        for (int i = t; i < Lq; ++i) ak = fmaf(ph[i * LP + t], qs[i * S + c], ak);
        dq[((int64_t)b * L + t) * ldg + c] = aq;
        dk_[((int64_t)b * L + t) * ldg + c] = ak;
    }
}

// h[b,:] = y[b, len[b]-1, :] * (hist[b, len[b]-1] > 0)     (SASRec.py:74-76)
__global__ void __launch_bounds__(256)
k_select_last(const float* __restrict__ y, const int64_t* __restrict__ hist, const int64_t* __restrict__ lengths,
              float* __restrict__ h, int B, int L, int d) {
    const int64_t total = (int64_t)B * d;
    for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256) {
        const int b = (int)(e / d), c = (int)(e % d);
        int64_t t = lengths[b] - 1;
        t = t < 0 ? 0 : (t >= L ? L - 1 : t);
        const float valid = hist[(int64_t)b * L + t] > 0 ? 1.f : 0.f;
        h[e] = y[((int64_t)b * L + t) * d + c] * valid;
    }
}

// dy = 0 except row (b, len[b]-1) = dh[b] * valid
__global__ void __launch_bounds__(256)
k_select_last_bwd(const float* __restrict__ dh, const int64_t* __restrict__ hist, const int64_t* __restrict__ lengths,
                  float* __restrict__ dy, int B, int L, int d) {
    const int64_t total = (int64_t)B * L * d;
    for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256) {
        const int c = (int)(e % d);
        const int64_t r = e / d;
        const int b = (int)(r / L), t = (int)(r % L);
        int64_t tl = lengths[b] - 1;
        tl = tl < 0 ? 0 : (tl >= L ? L - 1 : tl);
        float v = 0.f;
        if (t == tl && hist[r] > 0) v = dh[(int64_t)b * d + c];
        dy[e] = v;
    }
}

// gradient of a small table with massive sharing: CTA c walks rows [c*R, (c+1)*R) in order, thread = column,
// accumulating into its private column of a shared-memory copy of the table; partial tables are then summed
// in CTA order by k_reduce_chunks (dense.cu) -> deterministic, no atomics.
__global__ void __launch_bounds__(256)
k_small_table_partial(const float* __restrict__ src, int ld, const int64_t* __restrict__ ids, int64_t n, int n_rows,
                      int d, int rows_per_cta, float* __restrict__ part) {
    // G = 256 / d row groups (d <= 256, a divisor of 256: otherwise G = 1 and the spare threads idle): group g walks rows
    // beg + g, beg + g + G, ... of the CTA's range in order, thread = column, into the group's private copy of the table
    // (no two threads ever touch the same shared-memory word); eight rows' loads are in flight before the first add.
    // The G copies are then added in group order -> deterministic, no atomics.
    extern __shared__ float tab[];             // [G][n_rows][d]
    const int G = (d <= 256 && 256 % d == 0) ? 256 / d : 1;
    for (int e = threadIdx.x; e < G * n_rows * d; e += 256) tab[e] = 0.f;
    __syncthreads();
    const int64_t beg = (int64_t)blockIdx.x * rows_per_cta;
    const int64_t end = min(n, beg + rows_per_cta);
    const int g = threadIdx.x / d, c0 = threadIdx.x % d;
    if (g < G) {
        float* mine = tab + (size_t)g * n_rows * d;
        for (int c = c0; c < d; c += (G == 1 ? 256 : d)) {
            int64_t r = beg + g;
            for (; r + 7 * G < end; r += 8 * G) {
                int64_t id[8];
                float v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    id[u] = ids[r + u * G];
                    v[u] = src[(r + u * G) * ld + c];
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int64_t k = (id[u] < 0 || id[u] >= n_rows) ? 0 : id[u];
                    mine[k * d + c] += v[u];
                }
            }
            for (; r < end; r += G) {
                int64_t k = ids[r];
                k = (k < 0 || k >= n_rows) ? 0 : k;
                mine[k * d + c] += src[r * ld + c];
            }
        }
    }
    __syncthreads();
    float* out = part + (int64_t)blockIdx.x * n_rows * d;
    for (int e = threadIdx.x; e < n_rows * d; e += 256) {
        float a = tab[e];
        for (int g2 = 1; g2 < G; ++g2) a += tab[(size_t)g2 * n_rows * d + e];
        out[e] = a;
    }
}

// fixed-order sum over the partial tables: 8 lanes per element (chunks c, c+8, ...), then a fixed shuffle tree
__global__ void __launch_bounds__(256)
k_reduce_chunks_fwd(const float* __restrict__ part, int64_t size, int chunks, float* __restrict__ out) {
    const int cl = threadIdx.x & 7;
    for (int64_t i = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3); i < ((size + 31) / 32) * 32; i += (int64_t)gridDim.x * 32) {
        float a = 0.f;
        if (i < size)
            for (int c = cl; c < chunks; c += 8) a += part[(int64_t)c * size + i];
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 1);
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 2);
        a += __shfl_xor_sync(B2R_FULL_MASK, a, 4);
        if (cl == 0 && i < size) out[i] = a;
    }
}

// out[r,k] = a[r,k] * w[k]
__global__ void __launch_bounds__(256)
k_colscale(const float* __restrict__ a, const float* __restrict__ w, float* __restrict__ out, int64_t rows, int d) {
    const int64_t total = rows * d;
    for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256)
        out[e] = a[e] * w[e % d];
}

// out[k] = sum_r a[r,k] * b[r,k]   (single CTA, thread t owns rows t/d-strided ... fixed order)
__global__ void __launch_bounds__(1024)
k_colsum_prod(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int64_t rows, int d) {
    // thread (rg, k): rg = row group; partial over rows rg, rg+G, ... ; then groups combined in order
    extern __shared__ float part[];            // [G][d]
    const int G = 1024 / d > 0 ? 1024 / d : 1;
    const int k = threadIdx.x % d, rg = threadIdx.x / d;
    if (rg < G) {
        float s = 0.f;
        for (int64_t r = rg; r < rows; r += G) s = fmaf(a[r * d + k], b[r * d + k], s);
        part[rg * d + k] = s;
    }
    __syncthreads();
    if (threadIdx.x < d) {
        float s = 0.f;
        for (int g = 0; g < G; ++g) s += part[g * d + threadIdx.x];
        out[threadIdx.x] = s;
    }
}

static int capped_grid(int64_t need, int per_sm) {
    const int64_t cap = (int64_t)sm_count() * per_sm;
    int64_t g = need < cap ? need : cap;
    return (int)(g < 1 ? 1 : g);
}

constexpr int kSmallTableRows = 1024;

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_embed_history(const float* I, int64_t n_items, const float* P, int64_t n_pos, const int64_t* hist,
                                 const int64_t* lengths, float* x, int64_t* pos_out, int B, int L, int d,
                                 int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(I && P && hist && lengths && x, B2R_E_BADARG, "b2r_embed_history: null pointer");
    B2R_REQUIRE(B >= 0 && L >= 0 && d > 0 && d % 4 == 0, B2R_E_BADARG, "b2r_embed_history: bad shape");
    if (B == 0 || L == 0) return 0;
    k_embed_hist<<<capped_grid(((int64_t)B * L + 7) / 8, 16), 256, 0, as_stream(stream)>>>(
        I, n_items, P, n_pos, hist, lengths, x, pos_out, B, L, d, err_flag);
    B2R_LAUNCH_OK("k_embed_hist");
    return 0;
}

extern "C" int b2r_attention_fwd_live(const float* q, const float* k, const float* v, int ld, const int64_t* live, float* ctx,
                                      int B, int L, int d, int H, b2r_stream_t stream) {
    B2R_REQUIRE(q && k && v && ctx, B2R_E_BADARG, "b2r_attention_fwd_live: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && d > 0 && H > 0 && d % H == 0 && ld >= d, B2R_E_BADARG,
                "b2r_attention_fwd_live: bad shape B=%d L=%d d=%d H=%d ld=%d", B, L, d, H, ld);
    if (B == 0) return 0;
    const size_t smem = attn_fwd_smem(L, d, H);
    B2R_REQUIRE(smem <= kAttnSmemMax, B2R_E_UNSUPPORTED, "b2r_attention_fwd_live: L=%d d=%d needs %zu B of shared memory", L, d,
                smem);
    B2R_CUDA_OK(cudaFuncSetAttribute(k_attention_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_attention_fwd<<<B, 256, smem, as_stream(stream)>>>(q, k, v, ld, ctx, L, d, H, 1.f / sqrtf((float)(d / H)), live);
    B2R_LAUNCH_OK("k_attention_fwd");
    return 0;
}

extern "C" int b2r_attention_bwd_live(const float* q, const float* k, const float* v, int ld, const int64_t* live,
                                      const float* dctx, float* dq, float* dk, float* dv, int ldg, int B, int L, int d, int H,
                                      b2r_stream_t stream) {
    B2R_REQUIRE(q && k && v && dctx && dq && dk && dv, B2R_E_BADARG, "b2r_attention_bwd_live: null pointer");
    B2R_REQUIRE(B >= 0 && L > 0 && L <= kAttnBwdMaxL && d > 0 && H > 0 && d % H == 0 && ld >= d && ldg >= d, B2R_E_BADARG,
                "b2r_attention_bwd_live: bad shape B=%d L=%d d=%d H=%d", B, L, d, H);
    if (B == 0) return 0;
    const size_t smem = attn_bwd_smem(L, d, H);
    B2R_REQUIRE(smem <= kAttnSmemMax, B2R_E_UNSUPPORTED, "b2r_attention_bwd_live: L=%d d=%d H=%d needs %zu B of shared memory",
                L, d, H, smem);
    B2R_CUDA_OK(cudaFuncSetAttribute(k_attention_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_attention_bwd<<<B, 256, smem, as_stream(stream)>>>(q, k, v, ld, dctx, dq, dk, dv, ldg, L, d, H,
                                                        1.f / sqrtf((float)(d / H)), live);
    B2R_LAUNCH_OK("k_attention_bwd");
    return 0;
}

extern "C" int b2r_select_last(const float* y, const int64_t* hist, const int64_t* lengths, float* h, int B, int L,
                               int d, b2r_stream_t stream) {
    B2R_REQUIRE(y && hist && lengths && h, B2R_E_BADARG, "b2r_select_last: null pointer");
    if (B <= 0) return 0;
    k_select_last<<<capped_grid(((int64_t)B * d + 255) / 256, 8), 256, 0, as_stream(stream)>>>(y, hist, lengths, h, B, L, d);
    B2R_LAUNCH_OK("k_select_last");
    return 0;
}

extern "C" int b2r_select_last_bwd(const float* dh, const int64_t* hist, const int64_t* lengths, float* dy, int B,
                                   int L, int d, b2r_stream_t stream) {
    B2R_REQUIRE(dh && hist && lengths && dy, B2R_E_BADARG, "b2r_select_last_bwd: null pointer");
    if (B <= 0) return 0;
    k_select_last_bwd<<<capped_grid(((int64_t)B * L * d + 255) / 256, 16), 256, 0, as_stream(stream)>>>(dh, hist, lengths,
                                                                                                       dy, B, L, d);
    B2R_LAUNCH_OK("k_select_last_bwd");
    return 0;
}

extern "C" size_t b2r_small_table_grad_workspace_bytes(int64_t n, int n_rows, int d) {
    if (n <= 0 || n_rows <= 0 || d <= 0) return 0;
    const int64_t ctas = (n + kSmallTableRows - 1) / kSmallTableRows;
    return (size_t)ctas * n_rows * d * sizeof(float);
}

extern "C" int b2r_small_table_grad(const float* src, int ld, const int64_t* ids, int64_t n, int n_rows, int d,
                                    float* dense_out, void* ws, size_t ws_bytes, b2r_stream_t stream) {
    B2R_REQUIRE(src && ids && dense_out && ws, B2R_E_BADARG, "b2r_small_table_grad: null pointer");
    B2R_REQUIRE(n > 0 && n_rows > 0 && d > 0 && ld >= d, B2R_E_BADARG, "b2r_small_table_grad: bad shape");
    const int G = (d <= 256 && 256 % d == 0) ? 256 / d : 1;
    const size_t smem = (size_t)G * n_rows * d * sizeof(float);
    B2R_REQUIRE(smem <= 200 * 1024, B2R_E_UNSUPPORTED, "b2r_small_table_grad: table %d x %d does not fit shared memory",
                n_rows, d);
    B2R_REQUIRE(ws_bytes >= b2r_small_table_grad_workspace_bytes(n, n_rows, d), B2R_E_WORKSPACE,
                "b2r_small_table_grad: workspace too small");
    cudaStream_t s = as_stream(stream);
    const int ctas = (int)((n + kSmallTableRows - 1) / kSmallTableRows);
    B2R_CUDA_OK(cudaFuncSetAttribute(k_small_table_partial, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_small_table_partial<<<ctas, 256, smem, s>>>(src, ld, ids, n, n_rows, d, kSmallTableRows, static_cast<float*>(ws));
    B2R_LAUNCH_OK("k_small_table_partial");
    const int64_t size = (int64_t)n_rows * d;
    k_reduce_chunks_fwd<<<(int)((size + 31) / 32), 256, 0, s>>>(static_cast<float*>(ws), size, ctas, dense_out);
    B2R_LAUNCH_OK("k_reduce_chunks");
    return 0;
}

extern "C" int b2r_colscale(const float* a, const float* w, float* out, int64_t rows, int d, b2r_stream_t stream) {
    B2R_REQUIRE(a && w && out && rows >= 0 && d > 0, B2R_E_BADARG, "b2r_colscale: bad argument");
    if (rows == 0) return 0;
    k_colscale<<<capped_grid((rows * d + 255) / 256, 8), 256, 0, as_stream(stream)>>>(a, w, out, rows, d);
    B2R_LAUNCH_OK("k_colscale");
    return 0;
}

extern "C" int b2r_colsum_prod(const float* a, const float* b, float* out, int64_t rows, int d, b2r_stream_t stream) {
    B2R_REQUIRE(a && b && out && rows >= 0 && d > 0 && d <= 1024, B2R_E_BADARG, "b2r_colsum_prod: bad argument");
    const int G = 1024 / d > 0 ? 1024 / d : 1;
    k_colsum_prod<<<1, 1024, (size_t)G * d * sizeof(float), as_stream(stream)>>>(a, b, out, rows, d);
    B2R_LAUNCH_OK("k_colsum_prod");
    return 0;
}
