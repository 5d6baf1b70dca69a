// pairdot_p2p.cu -- the scoring hop of config 5's fused compute+exchange form (DESIGN.md §8; the default exchange,
// ShardedBPRMF exchange="p2p").  Same scoring as k_pairdot_fwd (pairdot.cu): out = <Q[qidx[e]], T[rows[e]]>
// for the (sample, local row) pairs an item-shard owner received -- but the score of pair e, which belongs to source
// rank s = e / seg, is stored straight into THAT rank's receive buffer through its peer-mapped pointer
// (out_tab[s] + e % seg; NVLink stores), so the scores need no all-to-all of their own: a signal-pad barrier after the
// kernel is all the home ranks wait for.  out_tab[s] already points at this owner's row of rank s's buffer.
#include "common.cuh"

namespace b2r {

template <int LPR, int RCH>
__global__ void __launch_bounds__(256)
k_pairdot_fwd_p2p(const float* __restrict__ Q, const int64_t* __restrict__ qidx, int64_t n_q, const float* __restrict__ T,
                  const int64_t* __restrict__ rows, int64_t n_t, float* const* __restrict__ out_tab, int64_t seg,
                  int64_t n, int32_t* err_flag) {
    static_assert(RCH <= LPR, "ids of a chunk are loaded one per lane");
    constexpr int D = LPR * 4;
    constexpr int GPC = 256 / LPR;
    constexpr int GPW = 32 / LPR;
    const int sub = threadIdx.x % LPR;
    const int grp = threadIdx.x / LPR;
    const int64_t nchunks = (n + RCH - 1) / RCH;
    const int64_t warp_first = (int64_t)blockIdx.x * GPC + (grp / GPW) * GPW;
    for (int64_t wbase = warp_first; wbase < nchunks; wbase += (int64_t)gridDim.x * GPC) {
        const int64_t ch = wbase + (grp % GPW);
        const int64_t e0 = ch * RCH;
        const int nr = (ch < nchunks) ? (int)min((int64_t)RCH, n - e0) : 0;
        int64_t my_row = -1, my_q = 0;
        if (sub < nr) {
            my_row = rows[e0 + sub];
            if (my_row >= 0) {
                my_row = checked_id(my_row, n_t, err_flag);
                my_q = checked_id(qidx[e0 + sub], n_q, err_flag);
            }
        }
        float4 r[RCH], q[RCH];
#pragma unroll
        for (int k = 0; k < RCH; ++k) {
            const int64_t rk = __shfl_sync(B2R_FULL_MASK, my_row, k, LPR);
            const int64_t qk = __shfl_sync(B2R_FULL_MASK, my_q, k, LPR);
            if (k < nr && rk >= 0) {
                r[k] = ld_row4(T + rk * D + sub * 4);
                q[k] = ld4(Q + qk * D + sub * 4);
            } else {
                r[k] = q[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        float mine = 0.f;
#pragma unroll
        for (int k = 0; k < RCH; ++k) {
            const float v = group_sum<LPR>(dot4(q[k], r[k]));
            if (sub == k) mine = v;
        }
        if (sub < nr) {
            const int64_t e = e0 + sub;
            out_tab[e / seg][e % seg] = mine;              // peer store: the requester's buffer, this owner's row
        }
    }
}

}  // namespace b2r

using namespace b2r;

extern "C" int b2r_pairdot_fwd_p2p(const float* Q, const int64_t* qidx, int64_t n_q, const float* T, const int64_t* rows,
                                   int64_t n_t, float* const* out_tab, int64_t seg, int64_t n, int d, int32_t* err_flag,
                                   b2r_stream_t stream) {
    B2R_REQUIRE(Q && qidx && T && rows && out_tab, B2R_E_BADARG, "b2r_pairdot_fwd_p2p: null pointer");
    B2R_REQUIRE(n >= 0 && seg > 0 && n % seg == 0 && n_q > 0 && n_t > 0, B2R_E_BADARG, "b2r_pairdot_fwd_p2p: bad sizes");
    B2R_REQUIRE(d == 32 || d == 64 || d == 128, B2R_E_UNSUPPORTED, "b2r_pairdot_fwd_p2p: d=%d (have 32, 64, 128)", d);
    if (n == 0) return 0;
    cudaStream_t s = as_stream(stream);
    const int64_t cap = (int64_t)sm_count() * 16;
#define B2R_PP(LPR, RCH)                                                                                   \
    do {                                                                                                   \
        constexpr int GPC = 256 / LPR;                                                                     \
        int64_t need = ((n + RCH - 1) / RCH + GPC - 1) / GPC;                                              \
        k_pairdot_fwd_p2p<LPR, RCH><<<(int)(need < cap ? need : cap), 256, 0, s>>>(Q, qidx, n_q, T, rows, n_t, out_tab, \
                                                                                  seg, n, err_flag);        \
    } while (0)
    if (d == 32) B2R_PP(8, 4); else if (d == 64) B2R_PP(16, 4); else B2R_PP(32, 4);
#undef B2R_PP
    B2R_LAUNCH_OK("k_pairdot_fwd_p2p");
    return 0;
}
