// adam_exact.cu -- the exact dense-Adam mode of the row-sparse optimizer (--exact_adam 1; reference semantics:
// torch.optim.Adam built by helpers/BaseRunner.py:110-114, applied to the whole table at :206).
//
// Dense Adam keeps moving a row it has no gradient for: m <- b1 m, v <- b2 v (plus the g = wd * w terms under weight
// decay) and w <- w - lr * m_hat / (sqrt(v_hat) + eps) at every step.  A row-sparse table reproduces that if every
// row carries the step it is up to date with (`last`) and is advanced through the skipped steps before it is read or
// updated (oracle.LazyExactAdam proves the bookkeeping on CPU).  k_adam_exact_advance is that advance, in three forms:
//   b2r_adam_exact_advance, rows == NULL : every row of the table (the flush before evaluation / saving)
//   b2r_adam_exact_advance, rows != NULL : the n listed rows, which must be unique
//   b2r_adam_exact_catch_up               : the raw ids a forward reads or an update writes, with every repeat
// One lane group (d/4 lanes, one float4 each) per listed id; the skipped steps are a register loop, beta^t is tracked by
// repeated multiplication from exp2(t0 * log2 beta).  Rows whose moments are all zero and that see no weight decay do
// not move under dense Adam either and are only re-stamped.
//
// Raw ids are deduplicated on the device with no sort: the stamp word is the claim.  Lane 0 of a group raises
// last[row] to max(upto, stamp) with one atomicMax and takes the old value as t0; exactly one group sees t0 < upto and
// advances the row, every other group sees t0 >= upto and leaves it.  The winner's arithmetic depends on t0 and the
// row's state only, both fixed before the launch, so the result is the same bits whichever group wins.
#include "common.cuh"

namespace b2r {

struct ExactK {
    float lr, beta1, beta2, eps, wd, omb1, omb2, log2b1, log2b2;
    int state_ld;
};

// CLAIM: rows are raw ids (repeats allowed) and positions [0, ignore_n) holding ignore_id are skipped
template <int LPR, bool CLAIM>
__global__ void __launch_bounds__(256)
k_adam_exact_advance(const int64_t* __restrict__ rows, int64_t n, int64_t n_rows, float* __restrict__ W,
                     float* __restrict__ M, float* __restrict__ V, int32_t* __restrict__ last, int upto, int stamp,
                     int64_t ignore_id, int64_t ignore_n, ExactK k, int32_t* __restrict__ err_flag) {
    constexpr int D = LPR * 4;
    constexpr int GPC = 256 / LPR;
    const int sub = threadIdx.x % LPR, grp = threadIdx.x / LPR;
    const int sld = k.state_ld ? k.state_ld : D;
    for (int64_t i = (int64_t)blockIdx.x * GPC + grp; i < n; i += (int64_t)gridDim.x * GPC) {
        int64_t row = rows ? rows[i] : i;
        if (CLAIM && i < ignore_n && row == ignore_id) continue;
        if (row < 0 || row >= n_rows) {
            if (err_flag && sub == 0) atomicAdd(err_flag, 1);
            continue;
        }
        // lane 0 of the group reads (or claims) the stamp and broadcasts it: the same lane re-stamps the row, so no
        // other lane may read last[row] itself (a lagging lane could see the new stamp and skip)
        const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << ((threadIdx.x & 31) / LPR * LPR));
        const int target = stamp > upto ? stamp : upto;
        int t0 = 0;
        if (sub == 0) {
            if (CLAIM) {
                // stamps only grow: a row already at the target needs no atomic (the common case of a repeated id)
                t0 = __ldcg(last + row);
                if (t0 < target) t0 = atomicMax(last + row, target);
            } else {
                t0 = last[row];
            }
        }
        t0 = __shfl_sync(gmask, t0, 0, LPR);
        if (t0 >= upto) {                                  // already there, or another group owns it (group-uniform)
            if (!CLAIM && sub == 0 && stamp > t0) last[row] = stamp;
            continue;
        }
        float4 w = ld4(W + row * D + sub * 4);
        float4 m = ld4(M + row * sld + sub * 4);
        float4 v = ld4(V + row * sld + sub * 4);
        // per lane: a slice whose moments are all zero (and no weight decay) does not move under dense Adam either;
        // slices are elementwise independent, so lanes may decide this on their own
        const bool still = (k.wd == 0.f) && m.x == 0.f && m.y == 0.f && m.z == 0.f && m.w == 0.f && v.x == 0.f &&
                           v.y == 0.f && v.z == 0.f && v.w == 0.f;
        if (!still) {
            float p1 = exp2f(k.log2b1 * (float)t0), p2 = exp2f(k.log2b2 * (float)t0);
            float* wp = &w.x;
            float* mp = &m.x;
            float* vp = &v.x;
            for (int t = t0 + 1; t <= upto; ++t) {
                p1 *= k.beta1;
                p2 *= k.beta2;
                const float step = __fdividef(k.lr, 1.f - p1);          // lr / bias_correction1
                const float isb2 = rsqrtf(1.f - p2);                    // 1 / sqrt(bias_correction2)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float g = k.wd * wp[e];
                    mp[e] = fmaf(k.beta1, mp[e], k.omb1 * g);
                    vp[e] = fmaf(k.beta2, vp[e], k.omb2 * g * g);
                    const float denom = fmaf(sqrtf(vp[e]), isb2, k.eps);
                    wp[e] = fmaf(-step, __fdividef(mp[e], denom), wp[e]);
                }
            }
            st4(W + row * D + sub * 4, w);
            st4(M + row * sld + sub * 4, m);
            st4(V + row * sld + sub * 4, v);
        }
        if (!CLAIM) {
            __syncwarp(gmask);
            if (sub == 0) last[row] = target;
        }
    }
}

static int exact_launch(const char* what, const int64_t* rows, int64_t count, int64_t ignore_id, int64_t ignore_n,
                        int64_t n_rows, int d, float* W, float* m, float* v, int32_t* last, int upto, int stamp,
                        const b2r_optim* opt, int32_t* err_flag, b2r_stream_t stream, bool claim) {
    B2R_REQUIRE(W && m && v && last && opt, B2R_E_BADARG, "%s: null pointer", what);
    B2R_REQUIRE(opt->kind == 1, B2R_E_BADARG, "%s: Adam only (kind %d)", what, opt->kind);
    B2R_REQUIRE(d == 32 || d == 64 || d == 128, B2R_E_UNSUPPORTED, "%s: d=%d (have 32, 64, 128)", what, d);
    B2R_REQUIRE(n_rows > 0 && upto >= 0, B2R_E_BADARG, "%s: bad sizes", what);
    if (count <= 0) return 0;
    ExactK k;
    k.lr = opt->lr;
    k.beta1 = opt->beta1;
    k.beta2 = opt->beta2;
    k.eps = opt->eps;
    k.wd = opt->weight_decay;
    k.omb1 = (float)(1.0 - (double)opt->beta1);
    k.omb2 = (float)(1.0 - (double)opt->beta2);
    k.log2b1 = (float)log2((double)opt->beta1);
    k.log2b2 = (float)log2((double)opt->beta2);
    k.state_ld = opt->state_ld;
    const int gpc = 256 / (d / 4);
    int64_t grid = (count + gpc - 1) / gpc;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    cudaStream_t s = as_stream(stream);
#define B2R_EXACT_LAUNCH(LPR, CL)                                                                                      \
    k_adam_exact_advance<LPR, CL><<<(int)grid, 256, 0, s>>>(rows, count, n_rows, W, m, v, last, upto, stamp, ignore_id, \
                                                            ignore_n, k, err_flag)
    if (claim) {
        if (d == 32) B2R_EXACT_LAUNCH(8, true);
        else if (d == 64) B2R_EXACT_LAUNCH(16, true);
        else B2R_EXACT_LAUNCH(32, true);
    } else {
        if (d == 32) B2R_EXACT_LAUNCH(8, false);
        else if (d == 64) B2R_EXACT_LAUNCH(16, false);
        else B2R_EXACT_LAUNCH(32, false);
    }
#undef B2R_EXACT_LAUNCH
    B2R_LAUNCH_OK("k_adam_exact_advance");
    return 0;
}

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_adam_exact_advance(const int64_t* rows, int64_t n, int64_t n_rows, int d, float* W, float* m,
                                      float* v, int32_t* last, int upto, int stamp, const b2r_optim* opt,
                                      int32_t* err_flag, b2r_stream_t stream) {
    return exact_launch("b2r_adam_exact_advance", rows, rows ? n : n_rows, -1, 0, n_rows, d, W, m, v, last, upto, stamp,
                        opt, err_flag, stream, false);
}

extern "C" int b2r_adam_exact_catch_up(const int64_t* ids, int64_t n, int64_t ignore_id, int64_t ignore_n,
                                       int64_t n_rows, int d, float* W, float* m, float* v, int32_t* last, int upto,
                                       int stamp, const b2r_optim* opt, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(ids || n == 0, B2R_E_BADARG, "b2r_adam_exact_catch_up: null ids");
    B2R_REQUIRE(n >= 0 && ignore_n >= 0 && ignore_n <= n, B2R_E_BADARG, "b2r_adam_exact_catch_up: n=%lld ignore_n=%lld",
                (long long)n, (long long)ignore_n);
    return exact_launch("b2r_adam_exact_catch_up", ids, n, ignore_id, ignore_n, n_rows, d, W, m, v, last, upto, stamp,
                        opt, err_flag, stream, true);
}
