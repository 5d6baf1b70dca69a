// bprmf_step.cu -- one whole BPRMF training step enqueued from C (b2r_bprmf_train_step) on a step context.
//
// Stream plan (step t):
//   main :  [exact dense-Adam mode: catch-up(U), catch-up(I)] -> fused gather+score+loss+dQ (rows read once) -> mean(loss)
//           -> [wait plan(t)] -> opt(I) + opt(U) in one launch
//   side :  plan(t+1) for the NEXT batch's ids (or plan(t) itself when nothing was prefetched)
// The index plan (per-bucket sort of the ids) only depends on the ids, so the context builds it one step ahead on
// a library-owned non-blocking stream while the HBM-bound kernels of the current step run; joins are event
// waits, never host synchronisations.  The plan has a whole step of slack before the update that reads it, so its
// kernels run as small persistent grids (kPlanCtas): the forward and optimizer kernels each fill every SM's register
// file, and every resident plan CTA takes the slot of one of their CTAs.  Sized to the work instead (~1,600 CTAs at
// config 2, placed first at high priority), the plan pushed part of the forward kernel into a second wave and slowed
// the optimizer behind it (H100: 0.296 ms per step against 0.265 ms for the two kernels alone).  Plans (direct plans, plan_direct.cuh) are double-buffered in the caller-provided
// workspace.  d must be 32, 64 or 128 (the widths the plan's apply kernel is built for).  Shapes the streaming forward
// kernel does not take (C > 1024) run the unfused gather / rowdot / loss / query-backward kernels instead.
#include "common.cuh"
#include "plan_direct.cuh"

int b2r_bprmf_fused_fwd_bwd_loss(const float* U, const int64_t* uid, int64_t n_users, const float* I, const int64_t* iid,
                                 int64_t n_items, float* grad_pred, float* row_loss, float* dQ, float* qout, int B, int C,
                                 int d, int32_t* err_flag, float* loss_out, unsigned int* done_counter,
                                 b2r_stream_t stream);
int b2r_adam_exact_catch_up(const int64_t* ids, int64_t n, int64_t ignore_id, int64_t ignore_n, int64_t n_rows, int d,
                            float* W, float* m, float* v, int32_t* last, int upto, int stamp, const b2r_optim* opt,
                            int32_t* err_flag, b2r_stream_t stream);

namespace b2r {

struct StepLayout {
    size_t q, pred, g, rows, dQ, counter;
    size_t dir_i[2], dir_u[2], dir_i_bytes, dir_u_bytes; // direct plans (plan_direct.cuh), double-buffered
    size_t total;
};

static bool step_layout(int B, int C, int d, int64_t n_users, int64_t n_items, StepLayout* L) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        size_t o = off;
        off += align_up(bytes, 256);
        return o;
    };
    const size_t n = (size_t)B * C;
    L->q = take((size_t)B * d * 4);
    L->pred = take(n * 4);
    L->g = take(n * 4);
    L->rows = take((size_t)B * 4);
    L->dQ = take((size_t)B * d * 4);
    L->counter = take(256);
    L->dir_i_bytes = direct_workspace_bytes((int64_t)n, n_items);
    L->dir_u_bytes = direct_workspace_bytes(B, n_users);
    for (int sl = 0; sl < 2; ++sl) {
        L->dir_i[sl] = take(L->dir_i_bytes);
        L->dir_u[sl] = take(L->dir_u_bytes);
    }
    L->total = off;
    return L->dir_i_bytes != 0 && L->dir_u_bytes != 0;
}

// CTAs of each plan launch of the step (persistent grids; b2r_bprmf_ctx_plan_launch changes them) and the side
// stream's priority.  Measured on an H100 SXM (700 W) at config 2 with tools/c2_breakdown.py --sweep, ms per step:
//   CTAs            0 (sized to the work)   66      132     264     528
//   highest prio    0.284                   0.286   0.287   0.284   0.284
//   default prio    0.282                   0.356   0.307   0.278   0.282
// At the default priority the plan's CTAs no longer jump ahead of the forward and optimizer CTAs; 264 (two per SM)
// keep it fast enough to finish inside its step of slack, fewer starve it.
constexpr int kPlanCtas = 264;
constexpr bool kPlanHighPriority = false;

struct StepCtx {
    int B, C, d;
    int plan_ctas;                    // CTAs per plan launch (0: sized to the work)
    bool plan_high;                   // side stream at the highest priority
    int64_t n_users, n_items;
    StepLayout L;
    char* ws;
    cudaStream_t side;                // builds the plan of the next batch
    cudaEvent_t fork, join[2];
    int slot;                         // plan buffer the NEXT step will read if it was prefetched
    const void* pre_uid;
    const void* pre_iid;
    bool have_pre;
    int32_t* last_u;                  // exact dense-Adam stamps (b2r_bprmf_ctx_exact); NULL: lazy row-sparse Adam
    int32_t* last_i;
    int exact_step;                   // the optimizer step the next train_step applies
};

// the plan stream, at the highest or the default priority (kPlanHighPriority)
static cudaError_t create_side_stream(StepCtx* c) {
    int prio_lo = 0, prio_hi = 0;
    cudaError_t e = cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&c->side, cudaStreamNonBlocking, c->plan_high ? prio_hi : prio_lo);
    return e;
}

}  // namespace b2r

using namespace b2r;

extern "C" size_t b2r_bprmf_step_workspace_bytes(int B, int C, int d, int64_t n_users, int64_t n_items) {
    if (B <= 0 || C <= 0 || d <= 0) return 0;
    StepLayout L;
    if (!step_layout(B, C, d, n_users, n_items, &L)) return 0;
    return L.total;
}

extern "C" int b2r_bprmf_ctx_create(void** ctx_out, int B, int C, int d, int64_t n_users, int64_t n_items, void* ws,
                                    size_t ws_bytes) {
    B2R_REQUIRE(ctx_out && ws, B2R_E_BADARG, "b2r_bprmf_ctx_create: null pointer");
    B2R_REQUIRE(B > 0 && C > 0 && d > 0 && d % 4 == 0, B2R_E_BADARG, "b2r_bprmf_ctx_create: B=%d C=%d d=%d", B, C, d);
    B2R_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, B2R_E_BADARG, "workspace must be 256-byte aligned");
    StepCtx* c = new StepCtx();
    c->B = B; c->C = C; c->d = d; c->n_users = n_users; c->n_items = n_items;
    if (!step_layout(B, C, d, n_users, n_items, &c->L)) {
        delete c;
        return set_error(B2R_E_UNSUPPORTED, "b2r_bprmf_ctx_create: cannot size the index plans");
    }
    if (ws_bytes < c->L.total) {
        const size_t need = c->L.total;
        delete c;
        return set_error(B2R_E_WORKSPACE, "b2r_bprmf_ctx_create: workspace %zu < required %zu", ws_bytes, need);
    }
    c->ws = static_cast<char*>(ws);
    c->slot = 0;
    c->have_pre = false;
    c->pre_uid = c->pre_iid = nullptr;
    c->last_u = c->last_i = nullptr;
    c->exact_step = 0;
    c->plan_ctas = kPlanCtas;
    c->plan_high = kPlanHighPriority;
    cudaError_t e = create_side_stream(c);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->fork, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->join[0], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->join[1], cudaEventDisableTiming);
    if (e != cudaSuccess) {
        delete c;
        return set_error((int)e, "b2r_bprmf_ctx_create: %s", cudaGetErrorString(e));
    }
    e = cudaMemsetAsync(c->ws + c->L.counter, 0, 256, c->side);
    if (e != cudaSuccess) {
        delete c;
        return set_error((int)e, "b2r_bprmf_ctx_create: %s", cudaGetErrorString(e));
    }
    // Index plans: "direct" plans (plan_direct.cuh: one scatter launch into fixed-capacity bucket regions, one sort launch,
    // both tables per launch) built for the NEXT batch on the high-priority side stream underneath this step's kernels.
    for (int sl = 0; sl < 2; ++sl) {
        int rc = direct_workspace_init(c->ws + c->L.dir_i[sl], c->L.dir_i_bytes, (int64_t)B * C, n_items, c->side);
        if (rc == 0) rc = direct_workspace_init(c->ws + c->L.dir_u[sl], c->L.dir_u_bytes, B, n_users, c->side);
        if (rc != 0) {
            delete c;
            return rc;
        }
    }
    e = cudaStreamSynchronize(c->side);
    if (e != cudaSuccess) {
        delete c;
        return set_error((int)e, "b2r_bprmf_ctx_create: %s", cudaGetErrorString(e));
    }
    *ctx_out = c;
    return 0;
}

extern "C" int b2r_bprmf_ctx_destroy(void* ctx) {
    if (!ctx) return 0;
    StepCtx* c = static_cast<StepCtx*>(ctx);
    cudaStreamSynchronize(c->side);
    cudaStreamDestroy(c->side);
    cudaEventDestroy(c->fork);
    cudaEventDestroy(c->join[0]);
    cudaEventDestroy(c->join[1]);
    delete c;
    return 0;
}

extern "C" int b2r_bprmf_ctx_plan_launch(void* ctx, int ctas, int high_priority) {
    B2R_REQUIRE(ctx && ctas >= 0, B2R_E_BADARG, "b2r_bprmf_ctx_plan_launch: ctx=%p ctas=%d", ctx, ctas);
    StepCtx* c = static_cast<StepCtx*>(ctx);
    c->plan_ctas = ctas;
    if ((high_priority != 0) != c->plan_high) {
        // the old stream's work (a prefetched plan) must be complete: the next step joins it through join[], which
        // records on the new stream from then on
        B2R_CUDA_OK(cudaStreamSynchronize(c->side));
        B2R_CUDA_OK(cudaStreamDestroy(c->side));
        c->plan_high = high_priority != 0;
        B2R_CUDA_OK(create_side_stream(c));
    }
    return 0;
}

extern "C" int b2r_bprmf_ctx_reset(void* ctx) {
    if (!ctx) return 0;
    StepCtx* c = static_cast<StepCtx*>(ctx);
    c->have_pre = false;
    c->pre_uid = c->pre_iid = nullptr;
    return 0;
}

extern "C" int b2r_bprmf_ctx_exact(void* ctx, int32_t* last_u, int32_t* last_i, int step) {
    B2R_REQUIRE(ctx, B2R_E_BADARG, "b2r_bprmf_ctx_exact: null context");
    B2R_REQUIRE((last_u == nullptr) == (last_i == nullptr), B2R_E_BADARG, "b2r_bprmf_ctx_exact: pass both stamp arrays or neither");
    B2R_REQUIRE(!last_u || step >= 1, B2R_E_BADARG, "b2r_bprmf_ctx_exact: step %d < 1", step);
    StepCtx* c = static_cast<StepCtx*>(ctx);
    c->last_u = last_u;
    c->last_i = last_i;
    c->exact_step = last_u ? step : 0;
    return 0;
}

static int build_plans(StepCtx* c, int slot, const int64_t* uid, const int64_t* iid, int32_t* err_flag) {
    char* base = c->ws;
    const int64_t n = (int64_t)c->B * c->C;
    profile_begin(B2R_PROF_PLAN_I, c->side);
    int rc = direct_scatter_pair(iid, n, c->n_items, base + c->L.dir_i[slot], uid, c->B, c->n_users,
                                 base + c->L.dir_u[slot], err_flag, c->plan_ctas, c->side);
    if (rc == 0)
        rc = direct_sort_pair(base + c->L.dir_i[slot], n, c->n_items, base + c->L.dir_u[slot], c->B, c->n_users,
                              c->plan_ctas, c->side);
    if (rc != 0) return rc;
    profile_end(B2R_PROF_PLAN_I, c->side);
    B2R_CUDA_OK(cudaEventRecord(c->join[slot], c->side));
    return 0;
}

extern "C" int b2r_bprmf_train_step(void* ctx, const b2r_bprmf_tables* t, const int64_t* uid, const int64_t* iid,
                                    const int64_t* next_uid, const int64_t* next_iid, const b2r_optim* opt,
                                    float* loss_out, int32_t* err_flag, b2r_stream_t stream) {
    B2R_REQUIRE(ctx && t && uid && iid && opt && loss_out, B2R_E_BADARG, "b2r_bprmf_train_step: null pointer");
    StepCtx* c = static_cast<StepCtx*>(ctx);
    B2R_REQUIRE(t->d == c->d && t->n_users == c->n_users && t->n_items == c->n_items, B2R_E_BADARG,
                "b2r_bprmf_train_step: tables do not match the context");
    const int B = c->B, C = c->C, d = c->d;
    char* base = c->ws;
    float* pred = reinterpret_cast<float*>(base + c->L.pred);
    float* g = reinterpret_cast<float*>(base + c->L.g);
    float* rows = reinterpret_cast<float*>(base + c->L.rows);
    float* dQ = reinterpret_cast<float*>(base + c->L.dQ);
    cudaStream_t main_s = as_stream(stream);
    const int64_t n = (int64_t)B * C;
    int rc;

    // everything the side stream does from here on is ordered after what main has enqueued so far
    // (in particular after the previous step's readers of the plan buffer about to be overwritten)
    B2R_CUDA_OK(cudaEventRecord(c->fork, main_s));
    B2R_CUDA_OK(cudaStreamWaitEvent(c->side, c->fork, 0));

    const int cur = c->slot;
    if (!(c->have_pre && c->pre_uid == uid && c->pre_iid == iid)) {
        rc = build_plans(c, cur, uid, iid, err_flag);     // nothing prefetched for this batch: build it now
        if (rc != 0) return rc;
    }
    const bool prefetch = next_uid != nullptr && next_iid != nullptr;
    if (prefetch) {
        rc = build_plans(c, cur ^ 1, next_uid, next_iid, err_flag);
        if (rc != 0) return rc;
    }
    c->have_pre = prefetch;
    c->pre_uid = prefetch ? next_uid : nullptr;
    c->pre_iid = prefetch ? next_iid : nullptr;
    c->slot = cur ^ 1;

    // exact dense-Adam mode: every row the step reads and updates is advanced through the steps it skipped (to t - 1)
    // and stamped t before the forward reads it; the update below then applies step t to rows standing at t - 1
    if (c->last_u) {
        const int t_ = c->exact_step;
        rc = b2r_adam_exact_catch_up(uid, B, -1, 0, t->n_users, d, t->U, t->Um, t->Uv, c->last_u, t_ - 1, t_, opt,
                                     err_flag, main_s);
        if (rc == 0)
            rc = b2r_adam_exact_catch_up(iid, n, -1, 0, t->n_items, d, t->I, t->Im, t->Iv, c->last_i, t_ - 1, t_, opt,
                                         err_flag, main_s);
        if (rc != 0) return rc;
    }

    // main: forward + loss + query-side backward; the gathered user rows are kept in q (the item gradient's source)
    float* q = reinterpret_cast<float*>(base + c->L.q);
    profile_begin(B2R_PROF_SCORE_FWD, main_s);
    rc = b2r_bprmf_fused_fwd_bwd_loss(t->U, uid, t->n_users, t->I, iid, t->n_items, g, rows, dQ, q, B, C, d, err_flag,
                                      loss_out, reinterpret_cast<unsigned int*>(base + c->L.counter), main_s);
    const bool fused = (rc == 0);
    if (rc != 0 && rc != B2R_E_UNSUPPORTED) return rc;
    if (fused) profile_end(B2R_PROF_SCORE_FWD, main_s);
    if (!fused) {
        rc = b2r_gather_rows(t->U, uid, t->n_users, q, B, d, err_flag, main_s);
        if (rc != 0) return rc;
        rc = b2r_rowdot_fwd(q, nullptr, B, t->I, iid, t->n_items, pred, B, C, d, err_flag, main_s);
        if (rc != 0) return rc;
        profile_end(B2R_PROF_SCORE_FWD, main_s);
        profile_begin(B2R_PROF_LOSS, main_s);
        rc = b2r_bpr_loss(pred, loss_out, g, rows, B, C, main_s);
        if (rc != 0) return rc;
        profile_end(B2R_PROF_LOSS, main_s);
        profile_begin(B2R_PROF_SCORE_BWDQ, main_s);
        rc = b2r_rowdot_bwd_query(g, t->I, iid, t->n_items, dQ, B, C, d, main_s);
        if (rc != 0) return rc;
        profile_end(B2R_PROF_SCORE_BWDQ, main_s);
    }

    // join plan(t); then the fused backward+optimizer on both tables in one launch: dI = g * q reads the saved user
    // rows, so the two updates are independent and the small user-table job runs underneath the item-table job
    B2R_CUDA_OK(cudaStreamWaitEvent(main_s, c->join[cur], 0));
    const b2r_grad_source su{dQ, nullptr, nullptr, B, 1, 0};
    const b2r_grad_source si{q, g, nullptr, n, C, 0};
    const b2r_apply_job ji{base + c->L.dir_i[cur], n, t->n_items, &si, nullptr, nullptr, t->I, t->Im, t->Iv};
    const b2r_apply_job ju{base + c->L.dir_u[cur], B, t->n_users, &su, nullptr, nullptr, t->U, t->Um, t->Uv};
    profile_begin(B2R_PROF_SEGMENT_I, main_s);
    rc = direct_apply_pair(&ji, &ju, d, 2, opt, main_s);
    if (rc != 0) return rc;
    profile_end(B2R_PROF_SEGMENT_I, main_s);
    return 0;
}
