/* b200rec.h -- C ABI of libb200rec.so: the ReChorus training hot path as sm_90a (H100) CUDA kernels.
 *
 * The reference (THUwangcy/ReChorus) has no FFI: its hot path is Python calling ATen.  Each entry point below
 * names the reference code it replaces (paths relative to the reference's src/).  The Python plugin layer
 * (rechorus_b200/) binds these with ctypes; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (e.g. torch.Tensor.data_ptr()), row-major,
 *     contiguous; tables/activations float32, ids int64 exactly as the reference's collate emits them
 *     (models/BaseModel.py:135-152); row pointers must be 16-byte aligned and d % 4 == 0.
 *   - all work is enqueued on `stream` (a cudaStream_t); no entry point synchronises or allocates.
 *     Scratch memory is an explicit caller-provided workspace sized by the matching *_workspace_bytes().
 *   - return value: 0 = ok; >0 = cudaError_t; <0 = B2R_E_* below.  b2r_last_error() gives the message
 *     (thread-local).  Out-of-range ids never read out of bounds: they are clamped to row 0 and counted in
 *     the device-side int32 `err_flag` the caller passes (may be NULL); the reference raises an ATen index
 *     error in that case, the plugin raises IndexError when it polls the flag.
 */
#ifndef B200REC_H
#define B200REC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2R_VERSION 103          /* major*10000 + minor*100 + patch */

#define B2R_E_BADARG   (-1)      /* null pointer, d % 4 != 0, negative size ... */
#define B2R_E_WORKSPACE (-2)     /* workspace too small */
#define B2R_E_UNSUPPORTED (-3)   /* shape outside what the kernels were built for */

typedef void* b2r_stream_t;      /* cudaStream_t */

#if defined(__GNUC__)
#define B2R_API __attribute__((visibility("default")))
#else
#define B2R_API
#endif

B2R_API int         b2r_version(void);
B2R_API const char* b2r_last_error(void);

/* Measurement hooks for bench.py (no effect on results):
 *  - b2r_launch_count(): kernels launched by this library so far (a CUB device-wide call counts as one);
 *  - b2r_profile_arm(tag, ev_start, ev_stop): the next launch of the tagged kernel inside a whole-step entry
 *    point is bracketed by cudaEventRecord on its own stream (one-shot; pass NULLs to disarm). */
#define B2R_PROF_TAGS 8
#define B2R_PROF_SCORE_FWD   0
#define B2R_PROF_SCORE_BWDQ  1
#define B2R_PROF_SEGMENT_I   2
#define B2R_PROF_SEGMENT_U   3
#define B2R_PROF_PLAN_I      4
#define B2R_PROF_LOSS        5
B2R_API long long b2r_launch_count(void);
B2R_API int       b2r_profile_arm(int tag, void* ev_start, void* ev_stop);

/* ------------------------------------------------------------------------------------------------
 * Scoring: pred[b,c] = < Q[qid[b]], T[ids[b,c]] >
 * replaces  models/general/BPRMF.py:39-42  (embedding x2, mul, sum)  with Q=u_embeddings, qid=user_id
 * and       models/sequential/SASRec.py:80-81                        with Q=user state [B,d], qid=NULL
 * ids [B,C] int64, pred [B,C] float32.  n_q / n_t = number of rows in Q / T (for range checks).
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_rowdot_fwd(const float* Q, const int64_t* qid, int64_t n_q,
                   const float* T, const int64_t* ids, int64_t n_t,
                   float* pred, int B, int C, int d, int32_t* err_flag, b2r_stream_t stream);

/* Backward of the scoring w.r.t. the query side: dQ[b,:] = sum_c g[b,c] * T[ids[b,c],:]   (dense [B,d];
 * replaces the mul/sum backward half of loss.backward(), helpers/BaseRunner.py:205).  Fixed summation
 * order -> bit-reproducible. */
B2R_API int b2r_rowdot_bwd_query(const float* g, const float* T, const int64_t* ids, int64_t n_t,
                         float* dQ, int B, int C, int d, b2r_stream_t stream);

/* Plain row gather out[r,:] = T[ids[r],:]  (nn.Embedding forward, e.g. NeuMF.py:63-66, SASRec.py:59) */
B2R_API int b2r_gather_rows(const float* T, const int64_t* ids, int64_t n_t, float* out, int64_t n, int d,
                    int32_t* err_flag, b2r_stream_t stream);
/* out[r*out_ld + 0..d) = T[ids[r / ids_div]]: writes into a column block of a wider activation matrix and
 * repeats each id ids_div times (NeuMF.py:61 repeats user ids over the candidates; :69 concatenates) */
B2R_API int b2r_gather_rows_strided(const float* T, const int64_t* ids, int64_t n_t, float* out, int out_ld,
                            int64_t n, int d, int ids_div, int32_t* err_flag, b2r_stream_t stream);

/* Flat pair scoring out[e] = < Q[qidx[e]], T[rows[e]] >, rows[e] < 0 = unused slot (score 0).  The shard owner's
 * half of BPRMF.py:39-42 when the item table is row-range sharded across GPUs (BASELINE config 5): the pairs are
 * what the all-to-all delivered, Q is the all-gathered user-vector block. */
B2R_API int b2r_pairdot_fwd(const float* Q, const int64_t* qidx, int64_t n_q, const float* T, const int64_t* rows,
                    int64_t n_t, float* out, int64_t n, int d, int32_t* err_flag, b2r_stream_t stream);

/* The scoring hop of the default config-5 exchange (exchange="p2p"): b2r_pairdot_fwd whose result for pair e is stored at out_tab[e / seg][e % seg] -- out_tab is a DEVICE array of n / seg pointers, typically the
 * peer-mapped receive buffers of the ranks the pairs came from (torch.distributed._symmetric_memory), so the scores
 * reach their requesters by NVLink stores from inside the kernel instead of an all-to-all. */
B2R_API int b2r_pairdot_fwd_p2p(const float* Q, const int64_t* qidx, int64_t n_q, const float* T, const int64_t* rows,
                                int64_t n_t, float* const* out_tab, int64_t seg, int64_t n, int d, int32_t* err_flag,
                                b2r_stream_t stream);

/* out[key[e],:] = sum over each run of consecutive valid pairs sharing key[e] of coef[e] * T[rows[e],:]  (rows < 0 =
 * unused slot; every key occupies one contiguous run, as the stable owner-bucketing of the sharded exchange
 * guarantees; out rows without pairs are left untouched).  The shard owner's half of dQ = sum_c g * I[id]. */
B2R_API int b2r_pair_runs_sum(const int64_t* key, const int64_t* rows, const float* coef, const float* T, int64_t n_t,
                      float* out, int64_t n_out, int64_t n, int d, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * BPR loss + closed-form gradient (models/BaseModel.py:175-189; formula SURVEY.md A.4).
 * pred [B,C] (column 0 = positive).  loss_out: 1 float.  grad_pred [B,C] = d loss / d pred (may be NULL).
 * row_ws: B floats of scratch.  Deterministic (fixed-order reduction).
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_bpr_loss(const float* pred, float* loss_out, float* grad_pred, float* row_ws,
                 int B, int C, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Index plan: the sorted, de-duplicated view of the ids a batch touches in one table.  It replaces the
 * accumulation half of ATen's embedding_dense_backward (the autograd node behind nn.Embedding,
 * BPRMF.py:31-32) and is what makes the scatter deterministic: every unique row gets ONE owner that sums
 * its contributions in ascending position order.
 *   in : ids[n] int64 in [0, n_rows)
 *   out: sorted_key[n] uint32 (row ids ascending), sorted_pos[n] uint32 (original flat position, stable),
 *        seg_start[n] int32 (index into sorted_* where unique row u starts), n_uniq (device int32)
 * ---------------------------------------------------------------------------------------------- */
B2R_API size_t b2r_plan_workspace_bytes(int64_t n, int64_t n_rows);
/* positions p < ignore_n whose id equals ignore_id are dropped from the gradient (they get the sentinel key n_rows,
 * which b2r_segment_apply skips): the right-padding of SASRec histories, whose gradient is exactly zero in the
 * reference (SASRec.py:74 masks them).  ignore_n = 0 keeps every position. */
B2R_API int b2r_plan_build_ex(const int64_t* ids, int64_t n, int64_t n_rows, int64_t ignore_id, int64_t ignore_n,
                      uint32_t* sorted_key, uint32_t* sorted_pos, int32_t* seg_start, int32_t* n_uniq,
                      void* ws, size_t ws_bytes, int32_t* err_flag, b2r_stream_t stream);

/* One contribution stream into a table gradient: position p (0 <= p < n) contributes
 *      coef[p] * src[row(p), :]      with   row(p) = src_id ? src_id[p / div] : p / div
 * BPRMF item table : src = u_embeddings, coef = grad_pred, src_id = user_id, div = C     (dI = g * u)
 * BPRMF user table : src = dQ [B,d],     coef = NULL(=1),  src_id = NULL,    div = 1
 * NeuMF / SASRec   : src = dense gradient of the gathered activations, coef = NULL, div = 1            */
typedef struct {
    const float*   src;
    const float*   coef;
    const int64_t* src_id;
    int64_t        n;
    int32_t        div;
    int32_t        ld;             /* leading dimension of src in floats (0 = d) */
} b2r_grad_source;

/* Optimizer applied to the touched rows (helpers/BaseRunner.py:110-114 builds torch.optim.<name>;
 * here the update is row-sparse / lazy: untouched rows do not move).  kind: 0 SGD, 1 Adam, 2 Adagrad.
 * Coupled L2 (weight_decay) as torch.optim does: g += wd * w.  bc1/bc2 = 1 - beta^t for Adam. */
typedef struct {
    int32_t kind;
    float   lr, beta1, beta2, eps, weight_decay, bc1, bc2;
    int32_t state_ld;   /* row stride (floats) of the m / v arrays in the row-sparse kernels; 0 = d.  2*d lets a table
                           keep m and v interleaved per row ([n_rows][2][d]): one 2*4d-byte burst instead of two */
    const float* clock; /* NULL: bc1 / bc2 above are used.  Else a DEVICE array float[4] kept by b2r_optim_tick:
                           [0] = step count t, [1] = lr / (1 - beta1^t), [2] = 1 / sqrt(1 - beta2^t); the kernels read the
                           Adam step size and bias correction from there, so an enqueued / graph-captured optimizer
                           launch needs no per-step host parameters */
} b2r_optim;

/* advance a device-side optimizer clock by one step (see b2r_optim.clock); one thread, double precision.  The betas are
 * doubles (torch computes 1 - beta ** t from the python floats); the bias corrections are rounded to float before use,
 * as the host-parameter route (bc1 / bc2 above) does, so both routes take bit-identical step sizes */
B2R_API int b2r_optim_tick(float* clock, float lr, double beta1, double beta2, b2r_stream_t stream);

/* Segment reduce over a plan built on the concatenation of up to two sources' ids
 * (positions [0, s0.n) belong to s0, [s0.n, s0.n + s1.n) to s1; s1 may be NULL).
 *   mode 0: write row-sparse gradient: uniq_rows[u] (int64) and grad_rows[u,:]  (u < *n_uniq)
 *   mode 1: add into a dense gradient table dense[row,:] += (one writer per row, no atomics)
 *   mode 2: apply `opt` in place to W (and state m, v) for the touched rows -- fused backward+optimizer
 * replaces embedding_dense_backward + grad zero-fill + the embedding part of optimizer.step()
 * (helpers/BaseRunner.py:193,205,206). */
B2R_API int b2r_segment_apply(const uint32_t* sorted_key, const uint32_t* sorted_pos, const int32_t* seg_start,
                      const int32_t* n_uniq, int64_t n, int64_t n_rows, int d,
                      const b2r_grad_source* s0, const b2r_grad_source* s1,
                      int mode, int64_t* uniq_rows, float* grad_rows, float* dense,
                      float* W, float* m, float* v, const b2r_optim* opt, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Bucketed form of plan + segment for the hot path ("direct" plans; modes 1 and 2 only; d in {32, 64, 128}):
 *   b2r_direct_plan_build : every (row id, position) pair is dropped into the fixed-capacity region of its bucket of
 *                           2^shift consecutive table rows (~200 pairs each) with one L2 atomic (pairs beyond a
 *                           region's capacity go to a spill list), then one kernel sorts every bucket by (row, position)
 *                           in shared memory and lists the row heads;
 *   b2r_direct_plan_apply : mode 1 (dense[row] += gradient row) or mode 2 (optimizer in place), each row's
 *                           contributions summed in ascending position -> same bits on every run.
 * The workspace must be initialised once with b2r_direct_plan_init; build/apply may then alternate.
 * b2r_direct_plan_workspace_bytes returns 0 for shapes it cannot take (n > 2^30 - 1, n_rows >= 2^32 - 1).
 * ---------------------------------------------------------------------------------------------- */
B2R_API size_t b2r_direct_plan_workspace_bytes(int64_t n, int64_t n_rows);
B2R_API int b2r_direct_plan_init(void* ws, size_t ws_bytes, int64_t n, int64_t n_rows, b2r_stream_t stream);
B2R_API int b2r_direct_plan_build(const int64_t* ids, int64_t n, int64_t n_rows, int64_t ignore_id, int64_t ignore_n,
                                  void* ws, size_t ws_bytes, int32_t* err_flag, b2r_stream_t stream);
B2R_API int b2r_direct_plan_apply(const void* ws, int64_t n, int64_t n_rows, int d, const b2r_grad_source* s0,
                                  const b2r_grad_source* s1, int mode, float* dense, float* W, float* m, float* v,
                                  const b2r_optim* opt, b2r_stream_t stream);

/* Dense optimizer step over a whole parameter tensor (exact torch.optim semantics; used for the small dense
 * parameters of NeuMF/SASRec and for the exact-reference dense-Adam mode of the embedding tables). */
B2R_API int b2r_dense_optim(float* W, const float* grad, float* m, float* v, int64_t numel,
                    const b2r_optim* opt, b2r_stream_t stream);


/* ------------------------------------------------------------------------------------------------
 * Dense layers (fp32 CUDA-core SGEMM with fused epilogues) -- the MLP tower of models/general/NeuMF.py:69-75
 * and the q/k/v + feed-forward Linear layers of utils/layers.py:26-28,106-107.  W is a torch nn.Linear
 * weight [N, K] row-major (its leading dimension may exceed K only through the pointer/ld pairs of X, Y).
 *   fwd        : Y[M,N] = act(X[M,K] W^T + bias),  relu != 0 applies ReLU
 *   bwd_input  : dX[M,K] = (dY * [relu_out > 0]) W          (relu_out = the layer's saved output, or NULL)
 *   bwd_weight : dW[N,K] = (dY * [relu_out > 0])^T X ; dbias[N] = column sums (NULL to skip); split over M
 *                in fixed chunks whose partial sums are added in order -> bit-reproducible
 * relu_out, when given, must share dY's leading dimension.
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_linear_fwd(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy,
                   int64_t M, int N, int K, int relu, b2r_stream_t stream);
/* Same forward on the tensor cores: wgmma.mma_async with TF32 operands, the accumulator in registers and a 3-product
 * hi/lo operand split (error ~2^-21 relative, i.e. fp32 class).  K % 32 == 0 (<= 128), N % 16 == 0 (<= 256), contiguous W.  Returns
 * B2R_E_UNSUPPORTED outside that class. */
B2R_API int b2r_linear_fwd_tc(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy,
                      int64_t M, int N, int K, int relu, b2r_stream_t stream);
/* The route of the Linear forward for Y[M, N] = X[M, K] W^T: 1 when it runs on the tensor-core kernel above -- M >= 4096
 * and the kernel's class, which also excludes N > 128 with K > 64 (W's tiles would not fit in one CTA's shared memory) --
 * and 0 when it runs on the SGEMM (b2r_linear_fwd).  Alignment and leading dimensions aside.  Host only. */
B2R_API int b2r_linear_fwd_uses_tc(int64_t M, int N, int K);
/* general form: x_mask (same layout as X, may be NULL) zeroes X where x_mask <= 0 -- with X = dY, x_mask = the layer's
 * saved ReLU output and W = the transposed weight this is the input gradient dX = (dY * [y > 0]) W of a Linear layer */
B2R_API int b2r_linear_tc(const float* X, int ldx, const float* x_mask, const float* W, const float* bias, float* Y,
                  int ldy, int64_t M, int N, int K, int relu, b2r_stream_t stream);
B2R_API int b2r_linear_bwd_input(const float* dY, int lddy, const float* relu_out, const float* W, float* dX, int lddx,
                         int64_t M, int N, int K, b2r_stream_t stream);
B2R_API size_t b2r_linear_bwd_weight_workspace_bytes(int64_t M, int N, int K);
B2R_API int b2r_linear_bwd_weight(const float* dY, int lddy, const float* relu_out, const float* X, int ldx,
                          float* dW, float* dbias, int64_t M, int N, int K, void* ws, size_t ws_bytes,
                          b2r_stream_t stream);

/* The same weight gradient on the tensor cores (wgmma TF32 with a hi/lo operand split, accumulator in registers; the
 * batch-row index is the MMA's reduction dimension, activations are transposed on their way into shared memory).
 * Shape class: N % 4 == 0, N <= 128, K % 16 == 0, K <= 240; returns B2R_E_UNSUPPORTED otherwise. */
B2R_API size_t b2r_linear_bwd_weight_tc_workspace_bytes(int64_t M, int N, int K);
B2R_API int b2r_linear_bwd_weight_tc(const float* dY, int lddy, const float* relu_out, const float* X, int ldx,
                                     float* dW, float* dbias, int64_t M, int N, int K, void* ws, size_t ws_bytes,
                                     b2r_stream_t stream);

/* y = LayerNorm(x + res) * gamma + beta, eps inside the sqrt, biased variance (utils/layers.py:113,117 via
 * nn.LayerNorm); mean/rstd [rows] are saved for the backward.  Backward returns dz (gradient of x + res, to be
 * used for both addends) and dgamma/dbeta (fixed-order two-stage reduction).  d <= 256 in the backward. */
B2R_API int b2r_add_layernorm_fwd(const float* x, const float* res, const float* gamma, const float* beta, float* y,
                          float* mean, float* rstd, int64_t rows, int d, float eps, b2r_stream_t stream);
B2R_API size_t b2r_add_layernorm_bwd_workspace_bytes(int64_t rows, int d);
B2R_API int b2r_add_layernorm_bwd(const float* dy, const float* x, const float* res, const float* gamma,
                          const float* mean, const float* rstd, float* dz, float* dgamma, float* dbeta,
                          int64_t rows, int d, void* ws, size_t ws_bytes, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Dropout fused into the kernels around it (nn.Dropout of models/general/NeuMF.py:70-72 and the dropout1 / dropout2
 * of utils/layers.py:113,117).  The mask is a pure function of an element's logical coordinates -- (row r, position t,
 * column j) of dropout site `site` at training step `step` -- so the backward regenerates it instead of storing it:
 *   word = Philox4x32-10(counter = (r, (t << 16) | (j >> 2), 0x80000000 | site, lo32(step)),
 *                        key = (lo32(seed), hi32(seed)))[j & 3];
 *   kept iff word >= floor(p * 2^32) (nothing at p = 1); kept elements are scaled by float(1 / (1 - p)) (0 at p = 1).
 * Each element is kept independently with probability 1 - p, as torch's dropout does; torch's own mask bits are not
 * reproduced.  Bit 31 of counter word 2 separates this stream from b2r_sample_negatives'.
 * Activation row -> (r, t): L == 0: (row, 0) (NeuMF: r = b*C + c); L > 0 and lengths == NULL: (row / L, row % L)
 * (SASRec's [B, L, d] block); lengths != NULL: (row, clamp(lengths[row] - 1, 0, L - 1)) (SASRec's last-query block,
 * one row per sequence at the position select_last reads).  So both SASRec forms draw the same mask, and the mask does
 * not depend on how far a batch is right-padded beyond its sequences.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const uint64_t* state;     /* DEVICE {seed, step}: the snapshot b2r_dropout_tick wrote for this forward */
    const int64_t*  lengths;   /* row mapping (see above); NULL unless the rows are one per sequence */
    double          p;         /* drop probability, 0 <= p <= 1 */
    int32_t         site;      /* NeuMF: layer index l; SASRec block i: 2i (dropout1), 2i + 1 (dropout2) */
    int32_t         L;         /* row mapping (see above) */
} b2r_dropout;

/* snapshot[0..1] = state[0..1] (seed, step), then state[1] += 1.  One thread; enqueued once per training forward, so a
 * captured CUDA graph advances the step on every replay and a second forward cannot shift the first one's masks. */
B2R_API int b2r_dropout_tick(uint64_t* state, uint64_t* snapshot, b2r_stream_t stream);
/* Y = dropout(act(X W^T + bias)): NeuMF.py:70-71 (layer(...).relu() then self.dropout_layer) in one kernel; CUDA-core
 * (b2r_linear_fwd) and tensor-core (b2r_linear_fwd_tc, same shape class and B2R_E_UNSUPPORTED outside it) forms.  The
 * backward needs no mask: the saved Y is > 0 exactly where the ReLU passed and the element was kept, so
 * b2r_linear_bwd_input / b2r_linear_tc with relu_out = Y and the weight scaled by 1 / (1 - p) give dX. */
B2R_API int b2r_linear_fwd_dropout(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy,
                                   int64_t M, int N, int K, int relu, const b2r_dropout* drop, b2r_stream_t stream);
B2R_API int b2r_linear_fwd_tc_dropout(const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy,
                                      int64_t M, int N, int K, int relu, const b2r_dropout* drop, b2r_stream_t stream);
/* b2r_linear_bwd_weight / b2r_linear_bwd_weight_tc of a layer followed by dropout: dW and dbias scaled by 1 / (1 - p)
 * in the final fixed-order reduction (the autograd of NeuMF.py:71's dropout, helpers/BaseRunner.py:205) */
B2R_API int b2r_linear_bwd_weight_dropout(const float* dY, int lddy, const float* relu_out, const float* X, int ldx,
                                          float* dW, float* dbias, int64_t M, int N, int K, const b2r_dropout* drop,
                                          void* ws, size_t ws_bytes, b2r_stream_t stream);
B2R_API int b2r_linear_bwd_weight_tc_dropout(const float* dY, int lddy, const float* relu_out, const float* X, int ldx,
                                             float* dW, float* dbias, int64_t M, int N, int K, const b2r_dropout* drop,
                                             void* ws, size_t ws_bytes, b2r_stream_t stream);
/* y = LayerNorm(dropout(x) + res) * gamma + beta: utils/layers.py:113 (layer_norm1(dropout1(context) + seq)) and :117
 * (layer_norm2(dropout2(output) + context)).  The backward regenerates the mask and writes dres = dz and
 * dx = dz * mask / (1 - p); workspace as b2r_add_layernorm_bwd.  d <= 256 in both directions. */
B2R_API int b2r_add_layernorm_fwd_dropout(const float* x, const float* res, const float* gamma, const float* beta, float* y,
                                          float* mean, float* rstd, int64_t rows, int d, float eps, const b2r_dropout* drop,
                                          b2r_stream_t stream);
B2R_API int b2r_add_layernorm_bwd_dropout(const float* dy, const float* x, const float* res, const float* gamma,
                                          const float* mean, const float* rstd, float* dz, float* dx, float* dgamma,
                                          float* dbeta, int64_t rows, int d, const b2r_dropout* drop, void* ws,
                                          size_t ws_bytes, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * SASRec sequence kernels (models/sequential/SASRec.py:51-86, utils/layers.py:34-63).
 *   embed_history : x[b,t,:] = I[hist[b,t]] + P[(len[b]-t) * (hist[b,t] > 0)]; pos_out (optional) gets the
 *                   position index used per element                                    (SASRec.py:58-66)
 *   attention_fwd_live : causal multi-head attention, heads = contiguous d/H chunks, scores / sqrt(d/H),
 *                   softmax over keys j <= i, no output projection; q,k,v rows at ld stride (layers.py:52-63)
 *   attention_bwd_live : recomputes the probabilities; writes dq, dk, dv rows at ldg stride.  L <= 128.
 *   select_last   : h[b] = y[b, len[b]-1] * (hist[b, len[b]-1] > 0)                    (SASRec.py:74-76)
 *   small_table_grad : dense gradient of a small table shared by many positions (the position table):
 *                   dense_out[id] = sum_{r: ids[r]=id} src[r], fixed order, no atomics.
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_embed_history(const float* I, int64_t n_items, const float* P, int64_t n_pos, const int64_t* hist,
                      const int64_t* lengths, float* x, int64_t* pos_out, int B, int L, int d,
                      int32_t* err_flag, b2r_stream_t stream);
/* Attention with dead rows skipped: live[b] (int64, NULL = L) is the number of leading positions of sequence b whose
 * output anything downstream reads -- SASRec uses position len-1 only (SASRec.py:74-81) and attention is causal, so the
 * positions >= len are exact dead work (forward and backward).  Dead rows of ctx / dq / dk / dv are written as zeros. */
B2R_API int b2r_attention_fwd_live(const float* q, const float* k, const float* v, int ld, const int64_t* live, float* ctx,
                                   int B, int L, int d, int H, b2r_stream_t stream);
B2R_API int b2r_attention_bwd_live(const float* q, const float* k, const float* v, int ld, const int64_t* live,
                                   const float* dctx, float* dq, float* dk, float* dv, int ldg, int B, int L, int d, int H,
                                   b2r_stream_t stream);
/* The same function with the per-(row, head) state in registers (csrc/attention_rt.cu): one lane owns one query row (forward,
 * dQ) or one key row (dK, dV) of one head, the other operand arrives as broadcast shared-memory loads.  The forward also
 * writes lse [B, L, H]: log2 of the softmax denominator plus the running max (base-2 domain); the backward recomputes the
 * probabilities from it and takes the forward's output ctx for the softmax-Jacobian row term dO_i . O_i.
 * Covers d/H in {8, 16, 32}, L <= 128, d and ld multiples of 4, 16-byte aligned pointers; anything else returns
 * B2R_E_UNSUPPORTED (callers fall back to b2r_attention_*_live).  Same dead-row contract. */
B2R_API int b2r_attention_fwd_rt(const float* q, const float* k, const float* v, int ld, const int64_t* live, float* ctx,
                                 float* lse, int B, int L, int d, int H, b2r_stream_t stream);
B2R_API int b2r_attention_bwd_rt(const float* q, const float* k, const float* v, int ld, const int64_t* live,
                                 const float* ctx, const float* lse, const float* dctx, float* dq, float* dk, float* dv,
                                 int ldg, int B, int L, int d, int H, b2r_stream_t stream);
/* Attention for ONE query per
 * sequence -- the query at position t* = clamp(lengths[b]-1, 0, L-1), the only position of SASRec's last block whose
 * output is used (models/sequential/SASRec.py:74-81) -- against keys/values 0..t* (the causal row of
 * utils/layers.py:52-63).  q_last, ctx_last, dq_last are [B, d]; k, v, dk, dv are [B, L, d] rows with leading
 * dimension ld / ldg; prob [B, H, L] keeps the softmax row for the backward.  Identical results to
 * b2r_attention_fwd/bwd_live restricted to that query; rows of dk, dv beyond t* are written as zeros. */
B2R_API int b2r_attention_last_fwd(const float* q_last, const float* k, const float* v, int ld, const int64_t* lengths,
                                   float* ctx_last, float* prob, int B, int L, int d, int H, b2r_stream_t stream);
B2R_API int b2r_attention_last_bwd(const float* q_last, const float* k, const float* v, int ld, const int64_t* lengths,
                                   const float* prob, const float* dctx_last, float* dq_last, float* dk, float* dv,
                                   int ldg, int B, int L, int d, int H, b2r_stream_t stream);
B2R_API int b2r_select_last(const float* y, const int64_t* hist, const int64_t* lengths, float* h, int B, int L,
                    int d, b2r_stream_t stream);
B2R_API int b2r_select_last_bwd(const float* dh, const int64_t* hist, const int64_t* lengths, float* dy, int B, int L,
                        int d, b2r_stream_t stream);
/* small_table_grad keeps G = 256 / d copies of the table in shared memory (G = 1 when d does not divide 256) and
 * returns B2R_E_UNSUPPORTED when they exceed 200 KB, e.g. more than 200 rows at d in {32, 64, 128}; callers then use the
 * plan route (b2r_plan_* / b2r_direct_plan_*), which has no size limit. */
B2R_API size_t b2r_small_table_grad_workspace_bytes(int64_t n, int n_rows, int d);
B2R_API int b2r_small_table_grad(const float* src, int ld, const int64_t* ids, int64_t n, int n_rows, int d,
                         float* dense_out, void* ws, size_t ws_bytes, b2r_stream_t stream);

/* Training envelope of SASRec: 0 when every kernel of a training step (forward and backward) accepts batches of width
 * 1..L at embedding width d with H heads, else B2R_E_UNSUPPORTED with b2r_last_error() naming the refusing kernel and its
 * limit.  full_blocks = the blocks that run full causal attention (b2r_attention_*_rt where it applies, else
 * b2r_attention_*_live); flags: B2R_SEQ_LAST_QUERY when the last block runs for the one query per sequence
 * (b2r_attention_last_*); any other flag bit is B2R_E_BADARG.  Host only: no device call is made. */
#define B2R_SEQ_LAST_QUERY 1
B2R_API int b2r_seq_train_check(int L, int d, int H, int full_blocks, int flags);

/* out[r,k] = a[r,k] * w[k]   and   out[k] = sum_r a[r,k] * b[r,k]   (the GMF half of NeuMF's final Linear,
 * models/general/NeuMF.py:68,74-75, and its weight gradient) */
B2R_API int b2r_colscale(const float* a, const float* w, float* out, int64_t rows, int d, b2r_stream_t stream);
B2R_API int b2r_colsum_prod(const float* a, const float* b, float* out, int64_t rows, int d, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Row f3, batch production on the device (opt-in): the per-epoch negative sampling of
 * models/BaseModel.py:206-214.  out[i*K + j] is uniform over the items of [1, n_items) that are not in
 * the training clicks of user_ids[i] (CSR: clicked_ptr [n_users+1], clicked_items sorted ascending and unique per user,
 * all within [1, n_items)).  No rejection loop: with m clicks the user has A = n_items-1-m allowed items; r =
 * floor(x * A / 2^32), x = word 0 of Philox4x32-10(counter = (lo32(i*K+j), hi32(i*K+j), 0, epoch), key = seed), and
 * the (r+1)-th allowed item is found by one binary search over the click row.  Same distribution as the reference,
 * NOT the same stream (NumPy's global Mersenne Twister consumed by a data-dependent Python loop).
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_sample_negatives(const int64_t* user_ids, int64_t N, int K, const int64_t* clicked_ptr,
                                 const int64_t* clicked_items, int64_t n_users, int64_t n_items, uint64_t seed,
                                 uint32_t epoch, int64_t* out, int32_t* err_flag, b2r_stream_t stream);
/* One training batch of a GeneralModel assembled on the device (GeneralModel.Dataset._get_feed_dict + collate_batch,
 * models/BaseModel.py:192-203,135-152): batch row t is training row perm[start + t] (perm NULL: start + t);
 * out_uid[t] = users[row], out_iid[t, 0] = items[row], out_iid[t, 1 + k] = neg[row, k]. */
B2R_API int b2r_collate_general(const int64_t* users, const int64_t* items, const int64_t* neg, const int64_t* perm,
                                int64_t start, int Bn, int K, int64_t* out_uid, int64_t* out_iid, b2r_stream_t stream);
/* The history part of a SequentialModel training batch (SequentialModel.Dataset._get_feed_dict, models/BaseModel.py:236-245,
 * + the padding of collate_batch, :135-152), right-padded to the fixed width Lp: batch row t is training row
 * perm[start + t] (perm NULL: start + t); with u = users[row], p = positions[row] and len = H > 0 ? min(p, H) : p,
 * out_hist[t, j] = his_items[his_ptr[u] + p - len + j] for j < len, else 0, and out_len[t] = len.  out_hist int64
 * [Bn, Lp], out_len int64 [Bn]; his_ptr [n_users+1] / his_items is the CSR of corpus.user_his (items only).  Bad rows
 * (u out of range, p < 1, p beyond the user's history, len > Lp) are clamped inside the CSR and counted in err_flag. */
B2R_API int b2r_collate_history(const int64_t* users, const int64_t* positions, const int64_t* his_ptr,
                                const int64_t* his_items, int64_t n_users, const int64_t* perm, int64_t start, int Bn,
                                int H, int Lp, int64_t* out_hist, int64_t* out_len, int32_t* err_flag,
                                b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Groundwork for the exact dense-Adam mode (not used by the default paths of this round): advance rows of a table whose
 * Adam state is kept row-sparsely through the optimizer steps they skipped, exactly as torch.optim.Adam over the whole
 * table (helpers/BaseRunner.py:110-114,206) would have moved them with a zero data gradient (g = weight_decay * w).
 * last [n_rows] int32 holds the step each row is up to date with.  rows == NULL: all n_rows rows (flush); otherwise n
 * unique row ids.  Every processed row is brought to step `upto` and stamped max(upto, stamp) -- pass stamp = upto + 1
 * when the step-(upto+1) update with b2r_direct_plan_apply / b2r_segment_apply follows.  opt carries lr, betas, eps,
 * weight_decay, state_ld (kind must be Adam; bc1/bc2 are not used: every skipped step has its own).
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_adam_exact_advance(const int64_t* rows, int64_t n, int64_t n_rows, int d, float* W, float* m, float* v,
                                   int32_t* last, int upto, int stamp, const b2r_optim* opt, int32_t* err_flag,
                                   b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation (row f2): integer ranks of the ground-truth item on the device.
 *
 * b2r_gt_rank:        rank[r] = #{c : pred[r*ld + c] >= pred[r*ld]}  -- helpers/BaseRunner.py:63 (column 0 is the
 *                     ground truth, ties count against it, rank >= 1; NaN compares false as in NumPy).
 * b2r_rank_histogram: hist[k] = #{r : rank[r] == k} for k <= kmax, hist[kmax+1] = #{rank > kmax}; hist has kmax+2
 *                     int64 slots.  HR@k and NDCG@k (BaseRunner.py:66-74) are sums over hist[1..k].
 * b2r_rank_all_items: the test_all protocol (BaseModel.py:194-198: candidates = [target] + arange(1, n_items),
 *                     scored by a dot product with the query row -- BPRMF.py:42, SASRec.py:81 -- then
 *                     preds[row, clicked item] = -inf, BaseRunner.py:244-251) without materialising the
 *                     [B, n_items] score matrix: rank[b] = 1 + #{1 <= j < n_items, (b,j) not masked :
 *                     <Q[b], I[j]> >= <Q[b], I[target[b]]>}.  Q [B, ldq] are the query rows (user vectors or
 *                     sequence states), (mask_row[e], mask_item[e]) the n_mask unique (batch row, item id) pairs to
 *                     exclude, s0 [B] scratch that receives the targets' scores.  The unmasked target column counts
 *                     (it scores equal to column 0), exactly as in the reference.
 * b2r_rank_all_items_clicked: the same ranks with the masked pairs read from the clicked-item CSR of the top-k section
 *                     below (clicked_ptr [n_users + 1], clicked_items; sorted, no duplicates): row b excludes every
 *                     clicked item j of user users[b] with 1 <= j < n_items, i.e. the pairs BaseRunner.py:244-251 sets
 *                     to -inf.  Each clicked item is scored by one thread with the fmaf order of the GEMM tile, so the
 *                     ranks equal b2r_rank_all_items' with (mask_row, mask_item) listing the same pairs.  A user outside
 *                     [0, n_users) is counted in err_flag and its row left unmasked; a bad target is clamped to 0 and
 *                     counted.  s0 [B] is scratch as above.
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_gt_rank(const float* pred, int64_t N, int64_t C, int64_t ld, int64_t* rank, b2r_stream_t stream);
B2R_API int b2r_rank_histogram(const int64_t* rank, int64_t N, int kmax, int64_t* hist, b2r_stream_t stream);
B2R_API int b2r_rank_all_items(const float* Q, int ldq, const float* I, const int64_t* target, int B, int64_t n_items,
                               int d, const int64_t* mask_row, const int64_t* mask_item, int64_t n_mask, float* s0,
                               int64_t* rank, int32_t* err_flag, b2r_stream_t stream);
B2R_API int b2r_rank_all_items_clicked(const float* Q, int ldq, const float* I, int64_t n_items, int d,
                                       const int64_t* target, const int64_t* users, int B, const int64_t* clicked_ptr,
                                       const int64_t* clicked_items, int64_t n_users, float* s0, int64_t* rank,
                                       int32_t* err_flag, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Top-k recommendation lists (row a11): the TopK branch of save_rec_results (main.py:117-132) on the device.
 *
 * Ordering contract -- each row's list equals Python's stable sorted(zip(item_id, pred), key=score, reverse=True)[:k]:
 *   - score descending, ties by candidate column ascending.  Candidate (score s, column c) becomes the 64-bit key
 *     (~mono(s) << 32) | c, mono() the order-preserving map of the float bits to uint32; ascending key order is the
 *     output order.  It is a total order, so results do not depend on grid or scheduling;
 *   - -0.0 is canonicalised to +0.0 before the key is built (the two compare equal in Python);
 *   - -inf (masked entries) sorts after every finite score, in column order; NaN sorts last, after -inf (Python's
 *     result is undefined there);
 *   - each row returns k' = min(k, C) entries, C the candidate count (1 + K, or n_items under test_all, where the list
 *     [target] + arange(1, n_items) has n_items columns).  1 <= k <= 1024; larger k is B2R_E_UNSUPPORTED, as is
 *     C >= 2^31 - 1.
 *
 * Clicked sets are a CSR over users: clicked_ptr int64 [n_users + 1], clicked_items int64, user u's items at
 * clicked_items[clicked_ptr[u] .. clicked_ptr[u + 1]), sorted ascending without duplicates (b2r_topk_all_items
 * binary-searches them; b2r_mask_clicked does not need the order).  For save_rec_results that is
 * train_clicked_set[u] | residual_clicked_set[u] (BaseRunner.py:244-251).
 *
 * b2r_topk_rows:      top-k' of each row of pred [N, C] (row stride ld): out_idx int64 [N, k'] candidate columns,
 *                     out_score float32 [N, k'] the scores as pred holds them (bit for bit).  A row of C <= 4096
 *                     columns is one CTA (one warp when C <= 1024); a longer row is split into ranges of at least 4096 columns (at most
 *                     ceil(1024 / N) of them), each range's top-k goes to the workspace and a second pass merges them.
 *                     Workspace: b2r_topk_rows_workspace_bytes(N, C, k) (0 when rows are not split).
 * b2r_mask_clicked:   pred[b*ld + j] = -inf for every clicked item j of user users[b] with 1 <= j < C: the test_all
 *                     masking of BaseRunner.py:244-251 (column j is item j; column 0, the target, is never masked).
 *                     Users outside [0, n_users) are counted in err_flag and their rows left as they are.
 * b2r_topk_all_items: the test_all protocol fused -- candidates [target] + arange(1, n_items) scored <Q[b], I[j]>,
 *                     clicked items masked as b2r_mask_clicked does, top-k' by the contract above -- without the
 *                     [B, n_items] score matrix.  Q [B, ldq] query rows, I [n_items, d], target [B], users [B].
 *                     out_items int64 [B, k'] item ids (column 0 reports target[b]), out_scores float32 [B, k'].
 *                     Items are scored in chunks of W columns (W = 32 MB / (4 B), a multiple of 128 in [128, 8192])
 *                     into the workspace, and each chunk is merged into a running top-k list per row; workspace
 *                     b2r_topk_all_items_workspace_bytes(B, n_items, k) = B * (4 W + 8 k + 8) bytes rounded up,
 *                     independent of n_items once n_items exceeds W.  Scores are accumulated s = fmaf(q_k, i_k, s) for
 *                     k ascending, as b2r_rank_all_items does, so a row whose rank r <= k has no exact ties puts its
 *                     target at position r; they can differ in the last bit from b2r_rowdot_fwd's.  Scores are
 *                     returned from the keys: a -0.0 score comes back as +0.0 and every NaN as 0x7fc00000.  Bad target
 *                     or user ids are clamped to 0 and counted in err_flag.
 * ---------------------------------------------------------------------------------------------- */
B2R_API size_t b2r_topk_rows_workspace_bytes(int64_t N, int64_t C, int k);
B2R_API int b2r_topk_rows(const float* pred, int64_t N, int64_t C, int64_t ld, int k, int64_t* out_idx, float* out_score,
                          void* workspace, size_t workspace_bytes, b2r_stream_t stream);
B2R_API int b2r_mask_clicked(float* pred, int64_t N, int64_t C, int64_t ld, const int64_t* users,
                             const int64_t* clicked_ptr, const int64_t* clicked_items, int64_t n_users, int32_t* err_flag,
                             b2r_stream_t stream);
B2R_API size_t b2r_topk_all_items_workspace_bytes(int B, int64_t n_items, int k);
B2R_API int b2r_topk_all_items(const float* Q, int ldq, const float* I, int64_t n_items, int d, const int64_t* target,
                               const int64_t* users, int B, const int64_t* clicked_ptr, const int64_t* clicked_items,
                               int64_t n_users, int k, int64_t* out_items, float* out_scores, int32_t* err_flag,
                               void* workspace, size_t workspace_bytes, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Impression evaluation and training batches (row f4): ImpressionRunner.evaluate (helpers/ImpressionRunner.py:135-171)
 * for the non-test_all branch on the device, batch by batch, without feed dicts or a host copy of the predictions; and
 * the batches and labels of ImpressionRunner.fit (:173-197) in the DataLoader's shuffled order.
 *
 * b2r_collate_impression: rows [start, start + Bn) of an evaluation phase as ImpressionModel.Dataset builds them
 *                     (models/BaseImpressionModel.py:152-184): out_uid int64 [Bn] = users[start + t], out_iid int64
 *                     [Bn, mp + mn] = [pos[:mp] | 0 up to mp | neg[:mn] | 0 up to mn].  The lists are a CSR over the
 *                     phase's rows: row r's positives at pos_items[pos_ptr[r] .. pos_ptr[r + 1]), its negatives at
 *                     neg_items[neg_ptr[r] .. neg_ptr[r + 1]); only the first mp / mn entries are read.  A user outside
 *                     [0, n_users) is clamped to 0 and counted in err_flag.
 * b2r_collate_impression_train: the same for one training batch whose rows are perm[start + t] (perm int64, indices of
 *                     the phase's rows; NULL: start + t), plus the labels ImpressionRunner.fit builds (:186-189) in out_labels int64
 *                     [Bn, mp + mn].  With P = min(pos_num[row], mp) and Q = min(neg_num[row], mn) -- the raw data
 *                     columns clipped as _get_feed_dict clips them (models/BaseImpressionModel.py:178-179):
 *                       - column c < mp: 1 if c < P, else -1;
 *                       - column c >= mp: 0 if c - mp < Q, else -1.
 *                     b2r_collate_impression runs the same kernel without a permutation or labels.
 * b2r_impression_metrics: adds the per-row NDCG@k, MAP@k and HR@k of one batch's predictions pred [Bn, C] (row stride ld,
 *                     C = mp + mn) into acc float64 [3 * nk]: acc[i] += sum of NDCG@topk[i], acc[nk + i] += sum of MAP@..,
 *                     acc[2 nk + i] += sum of HR@..; the caller divides by the row count.  pos_num / neg_num int64 [Bn]
 *                     are the raw data columns of the batch's rows; topk is a HOST array of 1 <= nk <= 16 cut-offs.
 *                     The contract, per row, with P = min(pos_num, mp), Q = min(neg_num, C - mp), W = P + Q:
 *                       - columns [0, P) and [mp, mp + Q) are valid; every other column's prediction is -inf;
 *                       - key[c] = (double)pred[c] - 1e-6 for c < mp, (double)pred[c] otherwise;
 *                       - order: key descending, ties by column ascending, NaN after everything (NaNs by column);
 *                         +0.0 and -0.0 are equal.  That is NumPy's stable argsort of -key;
 *                       - r_j = the number of columns before valid positive j (j < P); only r_j < W count, and Pm is
 *                         how many do.  With m_j = 1 + #{j' : r_j' < r_j}:
 *                         DCG@k = sum_{r_j < k} 1 / log2(r_j + 2), IDCG@k = sum_{t < min(Pm, k)} 1 / log2(t + 2)
 *                         (1 when 0), NDCG@k = DCG / IDCG;  MAP@k = sum_{r_j < k} m_j / (r_j + 1) / min(max(Pm, 1), k);
 *                         HR@k = 1 if some r_j < k, else 0.
 *                     One warp per row ranks every valid positive by counting over the row's keys in shared memory.
 *                     Sums run in a fixed order: lanes, then the rows of a CTA (a CTA holds a number of rows fixed
 *                     by C), then the CTAs in index order in the last CTA to finish -- so the result does not depend
 *                     on scheduling and two calls give identical bits.  Workspace:
 *                     b2r_impression_metrics_workspace_bytes(Bn, C, nk); its first 16 bytes are a counter that must be
 *                     zero before the first call (every call leaves it zero).  C above what one warp's shared memory
 *                     holds (about 19,000) or nk > 16 is B2R_E_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
#define B2R_IMPRESSION_MAX_TOPK 16
B2R_API int b2r_collate_impression(const int64_t* users, const int64_t* pos_ptr, const int64_t* pos_items,
                                   const int64_t* neg_ptr, const int64_t* neg_items, int64_t n_users, int64_t start,
                                   int Bn, int mp, int mn, int64_t* out_uid, int64_t* out_iid, int32_t* err_flag,
                                   b2r_stream_t stream);
B2R_API int b2r_collate_impression_train(const int64_t* users, const int64_t* pos_ptr, const int64_t* pos_items,
                                         const int64_t* neg_ptr, const int64_t* neg_items, const int64_t* pos_num,
                                         const int64_t* neg_num, const int64_t* perm, int64_t n_users, int64_t start,
                                         int Bn, int mp, int mn, int64_t* out_uid, int64_t* out_iid, int64_t* out_labels,
                                         int32_t* err_flag, b2r_stream_t stream);
B2R_API size_t b2r_impression_metrics_workspace_bytes(int Bn, int C, int nk);
B2R_API int b2r_impression_metrics(const float* pred, int64_t ld, int Bn, int C, int mp, const int64_t* pos_num,
                                   const int64_t* neg_num, const int* topk, int nk, double* acc, void* workspace,
                                   size_t workspace_bytes, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * NeuMF (models/general/NeuMF.py) against the whole catalogue: for the rows [b0, b1) of one evaluation batch of Bn
 * users, out[(b - b0) * ld_out + c] = the score NeuMF's forward gives candidate column c of row b under test_all
 * (column 0 the target, column c >= 1 item c) -- bit for bit, because the kernel runs the forward's own operations on the
 * forward's own 64-row tiles of the flattened [Bn * n_items] candidate rows (the GMF dot of b2r_rowdot_fwd, the
 * tensor-core Linear of b2r_linear_fwd_tc for every hidden layer, then the output layer's sequential fmaf chain).  The
 * [Bn * n_items, 2d] concat input and the activations are never written.  Masking, ranking and top-k then run on the
 * block through b2r_mask_clicked, b2r_gt_rank and b2r_topk_rows.
 *
 * b2r_neumf_score_rows_check: 0 when the shape is in the envelope, else B2R_E_UNSUPPORTED with b2r_last_error() naming
 *   the refusing condition: d in {32, 64}, 1..B2R_NEUMF_MAX_LAYERS hidden layers, 4096 <= Bn * n_items < 2^31 (the
 *   forward's tensor-core threshold), every hidden layer on the tensor-core kernel (b2r_linear_fwd_uses_tc) with at most
 *   128 outputs at d = 32 and 64 at d = 64 (registers), and the resident weights plus operands within one CTA's shared memory.  Host only.
 * b2r_neumf_window_rows: rows per window so that a [rows, n_items] float block stays within 32 MB (at least 1, at most
 *   Bn).  Host only.
 * b2r_neumf_score_rows: out-of-range user or target ids are clamped to row 0 and counted in err_flag.
 * ---------------------------------------------------------------------------------------------- */
#define B2R_NEUMF_MAX_LAYERS 4
typedef struct {
    const float*   mf_u;       /* [n_users, d]  mf_u_embeddings */
    const float*   mf_i;       /* [n_items, d]  mf_i_embeddings */
    const float*   mlp_u;      /* [n_users, d]  mlp_u_embeddings */
    const float*   mlp_i;      /* [n_items, d]  mlp_i_embeddings */
    int64_t        n_users;
    int64_t        n_items;
    int32_t        d;
    int32_t        n_layers;
    int32_t        widths[B2R_NEUMF_MAX_LAYERS];   /* hidden layer l: [widths[l], K_l] weight, K_0 = 2 d, K_l = widths[l - 1] */
    const float*   W[B2R_NEUMF_MAX_LAYERS];        /* contiguous nn.Linear weights */
    const float*   bias[B2R_NEUMF_MAX_LAYERS];     /* NULL: no bias */
    const float*   w_out;      /* [d + widths[n_layers - 1]]  prediction.weight (GMF part first) */
    const int64_t* users;      /* [Bn] */
    const int64_t* targets;    /* [Bn]  column 0 of the candidate list */
    int32_t        Bn;
    int32_t        b0;
    int32_t        b1;
    int32_t        _pad;
    float*         out;        /* [b1 - b0, ld_out] */
    int64_t        ld_out;
} b2r_neumf_rows;

B2R_API int b2r_neumf_score_rows_check(int d, int n_layers, const int32_t* widths, int64_t Bn, int64_t n_items);
B2R_API int b2r_neumf_window_rows(int64_t Bn, int64_t n_items);
B2R_API int b2r_neumf_score_rows(const b2r_neumf_rows* rows, int32_t* err_flag, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused BPRMF forward + loss + query-side backward in one streaming pass: every candidate row is read from HBM once
 * and used once (online-softmax recurrence for the gradient).  Outputs: grad_pred [B,C] (= d loss / d pred, loss = mean
 * of the per-sample losses), row_loss [B] (per-sample -log S), dQ [B,d] (= sum_c g[b,c] I[iid[b,c]]), pred [B,C]
 * optional (NULL to skip).  Returns B2R_E_UNSUPPORTED outside the kernel's class -- d not in {32, 64, 128}, C > 1024,
 * n_users, n_items or B*C >= 2^32 - 1 -- callers then use b2r_rowdot_fwd / b2r_bpr_loss / b2r_rowdot_bwd_query.
 * Replaces BPRMF.py:39-42, BaseModel.py:182-185 and their autograd (BaseRunner.py:205) in one kernel.
 * ---------------------------------------------------------------------------------------------- */
B2R_API int b2r_bprmf_fused_fwd_bwd(const float* U, const int64_t* uid, int64_t n_users, const float* I,
                            const int64_t* iid, int64_t n_items, float* pred, float* grad_pred, float* row_loss,
                            float* dQ, int B, int C, int d, int32_t* err_flag, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * One whole BPRMF training step enqueued from C (no Python between kernels) on a step context:
 *   fused gather/score/loss/dQ -> row-sparse fused optimizer on I, then on U (lazy rule, see b2r_optim).
 * Replaces one iteration of the hot loop helpers/BaseRunner.py:193-206 for models/general/BPRMF.py (the
 * per-row candidate shuffle of :187-191 is a mathematical no-op for this model and is not performed).
 * The context owns a side stream on which the index plans (sorts) are built; passing the NEXT batch's ids
 * (next_uid/next_iid, device pointers that must stay unmodified until the next call) lets the sort of step
 * t+1 overlap the HBM-bound kernels of step t, like a data loader's prefetch.  Pass NULLs to disable.
 * The workspace (b2r_bprmf_step_workspace_bytes) is caller-owned and must outlive the context.  Shapes whose index
 * plans cannot be sized (b2r_direct_plan_workspace_bytes == 0 for the item or the user table) get 0 bytes and
 * B2R_E_UNSUPPORTED from b2r_bprmf_ctx_create.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    float*  U;  float* I;            /* [n_users, d], [n_items, d]                       */
    float*  Um; float* Uv;           /* optimizer state for U (Adam: m, v; Adagrad: v)   */
    float*  Im; float* Iv;           /* optimizer state for I                            */
    int64_t n_users, n_items;
    int32_t d, _pad;
} b2r_bprmf_tables;

B2R_API size_t b2r_bprmf_step_workspace_bytes(int B, int C, int d, int64_t n_users, int64_t n_items);
B2R_API int b2r_bprmf_ctx_create(void** ctx_out, int B, int C, int d, int64_t n_users, int64_t n_items, void* ws,
                         size_t ws_bytes);
B2R_API int b2r_bprmf_ctx_destroy(void* ctx);
/* forget the prefetched plan (call at the start of an epoch and after an aborted one): a prefetched plan is matched to
 * the next batch by its id pointers, which a caching allocator may hand out again for a different batch */
B2R_API int b2r_bprmf_ctx_reset(void* ctx);
/* how the context builds the next batch's index plan underneath a step: the plan kernels as persistent grids of at most
 * `ctas` CTAs (0: grids sized to the work) on a side stream of the highest (high_priority != 0) or the default priority.
 * The defaults were measured on an H100 at the BASELINE config 2 shape; this entry point is for measuring others. */
B2R_API int b2r_bprmf_ctx_plan_launch(void* ctx, int ctas, int high_priority);
B2R_API int b2r_bprmf_train_step(void* ctx, const b2r_bprmf_tables* t, const int64_t* uid, const int64_t* iid,
                         const int64_t* next_uid, const int64_t* next_iid, const b2r_optim* opt,
                         float* loss_out, int32_t* err_flag, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * List-wise ranking losses of the impression models: value and closed-form gradient of ImpressionModel.loss
 * (models/BaseImpressionModel.py:44-128).  pred [B, Cn] float32, target [B, Cn] int64 (1 clicked, 0 shown, -1 padding);
 * columns < max_pos are the positive slots (:55-58; the reference also reads column max_pos: max_pos < Cn).
 * kind: 0 'BPR' (reweight between sigmoid and log, :82-85), 1 'BPR..after' (:73-75), 2 'BPR..before' (:76-78), each
 * with hard = 0/1 ('hard' in the name, :63-68); 3 'listnet' (:88-97), 4 'softmaxCE' (:99-110), 5 'attention_rank'
 * (:112-128).  loss_out: 1 float; grad_pred [B, Cn] = d loss / d pred (may be NULL).  ws: b2r_listwise_workspace_bytes(B).
 * ---------------------------------------------------------------------------------------------- */
B2R_API size_t b2r_listwise_workspace_bytes(int B);
B2R_API int b2r_listwise_loss(const float* pred, const int64_t* target, int B, int Cn, int max_pos, int kind, int hard,
                              float* loss_out, float* grad_pred, void* ws, size_t ws_bytes, b2r_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Row-sharded tables (BASELINE config 5): the exchange done by kernels over peer-mapped memory (symmetric-memory
 * buffers of the ranks of one box; NVLink loads / stores) instead of collectives between kernels.  No reference
 * counterpart (the reference is single-device); contract: SURVEY.md 8(e).  Pointer tables are HOST arrays of W device
 * pointers (W <= 16).  Ordering between ranks is the caller's (signal-pad barriers between the phases).
 *
 * b2r_route_ids: stable partition of one table's ids [B, C] by owner (id / rows_per): pair (b, c) goes to slot
 *   s of its owner o, slots counted in (sample, candidate) order; written through peer_rows[o][s] = local row and
 *   peer_q[o][s] = q_base + b (the row of the replicated query block); the unused tail of each region gets row -1;
 *   slot_of[b*C + c] = o * cap + s; dest_total[o] = pairs sent to o; *overflow += 1 if some dest_total > cap.
 * b2r_serve_rows: for every request e with req_rows[e] >= 0: row req_rows[e] of T is stored into row req_q[e] of EVERY
 *   rank's block peer_dst[k] (gather + all-gather in one pass).
 * b2r_scatter_f32_to_peers / b2r_scatter_rows_to_peers: val[i] * scale (resp. row i of src) -> peer_dst[slot_of[i] / cap]
 *   at element (row) slot_of[i] % cap.
 * b2r_sum_rows_from_peers: out[i] = sum_k peer_src[k][offset + i], k ascending (fixed order -> deterministic).
 * ---------------------------------------------------------------------------------------------- */
B2R_API size_t b2r_route_workspace_bytes(int B, int W);
B2R_API int b2r_route_ids(const int64_t* ids, int B, int C, int W, int64_t rows_per, int64_t n_rows,
                          const void* const* peer_rows, const void* const* peer_q, int64_t q_base, int cap,
                          int* slot_of, int* dest_total, int* overflow, void* ws, size_t ws_bytes, int32_t* err_flag,
                          b2r_stream_t stream);
B2R_API int b2r_serve_rows(const float* T, int64_t n_t, const int64_t* req_rows, const int64_t* req_q, int64_t n,
                           const void* const* peer_dst, int W, int d, int32_t* err_flag, b2r_stream_t stream);
B2R_API int b2r_scatter_f32_to_peers(const float* val, const int* slot_of, int64_t n, const void* const* peer_dst, int W,
                                     int cap, float scale, b2r_stream_t stream);
B2R_API int b2r_scatter_rows_to_peers(const float* src, const int* slot_of, int64_t n, const void* const* peer_dst, int W,
                                      int cap, int d, b2r_stream_t stream);
B2R_API int b2r_sum_rows_from_peers(const void* const* peer_src, int W, int64_t offset_floats, float* out,
                                    int64_t n_floats, b2r_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200REC_H */
