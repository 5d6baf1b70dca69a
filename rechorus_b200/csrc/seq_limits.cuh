// seq_limits.cuh -- shape limits of SASRec's sequence kernels, in one place: the launchers (attention.cu, attention_rt.cu,
// attention_last.cu, attention_tiled.cu, dense.cu) refuse with these predicates and b2r_seq_train_check /
// b2r_seq_train_check_tiled (seq_check.cu) answer from them, so the construction-time check and the kernels cannot
// disagree.
#pragma once
#include <stddef.h>

namespace b2r {

constexpr size_t kAttnSmemMax = 227 * 1024;   // opt-in dynamic shared memory per CTA on sm_90
constexpr int kAttnBwdMaxL = 128;             // k_attention_bwd keeps at most 4 keys per lane (phase C)
constexpr int kALMaxL = 256;                  // k_attention_last_*: one [kALMaxL] score row per warp in shared memory
constexpr int kLNMaxD = 256;                  // k_add_layernorm_bwd: 8 columns per lane; the dropout masks: 8 keep bits

// register-resident attention (attention_rt.cu): head width, batch width and alignment class
static inline bool rt_shape_ok(int L, int d, int H, int ld) {
    if (H <= 0 || d % H != 0) return false;
    const int dk = d / H;
    return (dk == 8 || dk == 16 || dk == 32) && L <= 128 && d % 4 == 0 && ld % 4 == 0;
}

static inline size_t rt_fwd_smem(int L, int d) { return (size_t)3 * L * (d + 4) * sizeof(float); }
static inline size_t rt_bwd_smem(int L, int d, int H) {
    return ((size_t)5 * L * (d + 4) + (size_t)2 * L * H) * sizeof(float);
}

// tiled attention (attention_tiled.cu) and the long last-query form (attention_last.cu): shared memory does not depend
// on L.  The batch width stops where the dropout masks' 16-bit position field does (dropout.cuh, check_dropout).
constexpr int kTiledMaxL = 65535;

static inline bool tiled_shape_ok(int L, int d, int H, int ld) {
    if (H <= 0 || d % H != 0) return false;
    const int dk = d / H;
    return (dk == 8 || dk == 16 || dk == 32 || dk == 64) && L >= 1 && L <= kTiledMaxL && d <= kLNMaxD && d % 4 == 0 &&
           ld % 4 == 0;
}

static inline bool tiled_last_shape_ok(int L, int d, int H) {
    return H > 0 && d % H == 0 && L >= 1 && L <= kTiledMaxL;
}

// shared-memory operand attention (attention.cu)
static inline size_t attn_fwd_smem(int L, int d, int H) {
    return ((size_t)3 * L * (d + 1) + (size_t)8 * H * L) * sizeof(float);
}
static inline size_t attn_bwd_smem(int L, int d, int H) {
    return ((size_t)4 * L * (d + 1) + (size_t)H * L * (L + 1)) * sizeof(float);
}

}  // namespace b2r
