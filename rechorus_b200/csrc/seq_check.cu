// seq_check.cu -- b2r_seq_train_check: whether every kernel of a SASRec training step accepts the step's shapes, answered
// on the host from the launchers' own predicates (seq_limits.cuh) before anything is allocated or launched.  A model
// built outside that envelope would run its forward and then fail in the first backward.
#include "common.cuh"
#include "seq_limits.cuh"

using namespace b2r;

// Full causal attention at batch width L on the route ops._CausalAttention takes: the register-resident kernels when
// their shape class and forward shared memory allow (the backward then has to fit as well), the shared-memory kernels
// otherwise.  0, or B2R_E_UNSUPPORTED naming the launcher that refuses.
static int full_attention_check(int L, int d, int H) {
    if (rt_shape_ok(L, d, H, d) && rt_fwd_smem(L, d) <= kAttnSmemMax) {
        const size_t smem = rt_bwd_smem(L, d, H);
        B2R_REQUIRE(smem <= kAttnSmemMax, B2R_E_UNSUPPORTED,
                    "b2r_attention_bwd_rt: batch width L=%d with d=%d, H=%d needs %zu B of shared memory, more than %zu", L,
                    d, H, smem, kAttnSmemMax);
        return 0;
    }
    size_t smem = attn_fwd_smem(L, d, H);
    B2R_REQUIRE(smem <= kAttnSmemMax, B2R_E_UNSUPPORTED,
                "b2r_attention_fwd_live: batch width L=%d with d=%d, H=%d needs %zu B of shared memory, more than %zu", L, d,
                H, smem, kAttnSmemMax);
    B2R_REQUIRE(L <= kAttnBwdMaxL, B2R_E_UNSUPPORTED, "b2r_attention_bwd_live: batch width L=%d, the kernel needs L <= %d",
                L, kAttnBwdMaxL);
    smem = attn_bwd_smem(L, d, H);
    B2R_REQUIRE(smem <= kAttnSmemMax, B2R_E_UNSUPPORTED,
                "b2r_attention_bwd_live: batch width L=%d with d=%d, H=%d needs %zu B of shared memory, more than %zu", L, d,
                H, smem, kAttnSmemMax);
    return 0;
}

extern "C" int b2r_seq_train_check(int L, int d, int H, int full_blocks, int flags) {
    B2R_REQUIRE(L > 0 && d > 0 && d % 4 == 0 && H > 0 && d % H == 0 && full_blocks >= 0 &&
                    (flags & ~B2R_SEQ_LAST_QUERY) == 0,
                B2R_E_BADARG, "b2r_seq_train_check: bad arguments L=%d d=%d H=%d full_blocks=%d flags=%d", L, d, H,
                full_blocks, flags);
    B2R_REQUIRE(d <= kLNMaxD, B2R_E_UNSUPPORTED, "b2r_add_layernorm_bwd: d=%d, the kernel needs d <= %d", d, kLNMaxD);
    B2R_REQUIRE(!(flags & B2R_SEQ_LAST_QUERY) || L <= kALMaxL, B2R_E_UNSUPPORTED,
                "b2r_attention_last_fwd / _bwd: batch width L=%d, the kernels need L <= %d", L, kALMaxL);
    // a batch may be narrower than L (padded to its longest history): every width up to L must be accepted
    if (full_blocks > 0)
        for (int l = 1; l <= L; ++l) {
            const int rc = full_attention_check(l, d, H);
            if (rc != 0) return rc;
        }
    return 0;
}

// The envelope with --tiled_attention: what b2r_seq_train_check accepts runs on the same kernels; the rest may run on the
// tiled kernels (attention_tiled.cu) and the long last-query form (attention_last.cu, *_tiled), whose shared memory does
// not depend on L.  A superset of b2r_seq_train_check, monotone in L.
extern "C" int b2r_seq_train_check_tiled(int L, int d, int H, int full_blocks, int flags) {
    B2R_REQUIRE(L > 0 && d > 0 && d % 4 == 0 && H > 0 && d % H == 0 && full_blocks >= 0 &&
                    (flags & ~B2R_SEQ_LAST_QUERY) == 0,
                B2R_E_BADARG, "b2r_seq_train_check_tiled: bad arguments L=%d d=%d H=%d full_blocks=%d flags=%d", L, d, H,
                full_blocks, flags);
    if (b2r_seq_train_check(L, d, H, full_blocks, flags) == 0) return 0;
    B2R_REQUIRE(d <= kLNMaxD, B2R_E_UNSUPPORTED, "b2r_add_layernorm_bwd: d=%d, the kernel needs d <= %d", d, kLNMaxD);
    B2R_REQUIRE(L <= kTiledMaxL, B2R_E_UNSUPPORTED,
                "b2r_dropout: batch width L=%d, the masks' 16-bit position field needs L <= %d", L, kTiledMaxL);
    // a batch may be narrower than L: widths the default kernels take run on them, every other width on the tiled ones
    if (full_blocks > 0 && !tiled_shape_ok(L, d, H, d))
        for (int l = 1; l <= L; ++l) {
            if (full_attention_check(l, d, H) == 0) continue;
            return b2r::set_error(B2R_E_UNSUPPORTED,
                                  "b2r_attention_fwd_tiled / _bwd_tiled: head width d/H=%d at batch width L=%d, the kernels "
                                  "need d/H in {8, 16, 32, 64} (the shared-memory kernels stop at L=%d)", d / H, l, l - 1);
        }
    return 0;
}
