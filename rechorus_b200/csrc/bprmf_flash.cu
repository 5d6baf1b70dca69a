// bprmf_flash.cu -- K1+K2a as ONE streaming pass per sample, no second use of any candidate row.
//
// Contract: gather the user row and the C candidate rows of a sample, score them (models/general/BPRMF.py:39-42),
// evaluate the BPR loss (models/BaseModel.py:182-185) and its closed-form gradient g (SURVEY.md A.4), and reduce
// dQ = sum_c g_c * I[id_c] (the mul/sum half of loss.backward(), helpers/BaseRunner.py:205) -- every candidate row read
// from HBM exactly once.
//
// Why this structure: keeping all rows of a sample on chip between their two uses (score, then g * row once the softmax
// over the sample's negatives is known) is bound by that hand-over (barriers, cross-group statistics).  The gradient
// factorises instead.  With e_c = exp(x_c - M), s_c = sigmoid(p - x_c), Z = sum e_c, A = sum e_c s_c, S = A / Z,
// dS = -1 / (B S):
//     g_c = dS * (e_c / Z) * ((s_c - S) - s_c (1 - s_c)) = (dS / Z) * e_c * (s_c^2 - S)        (negatives)
//     dQ  = g_0 * r_0 + (dS / Z) * ( sum_c e_c s_c^2 r_c  -  S * sum_c e_c r_c )
// so two row-weighted sums (acc1, acc2) and three scalars (Z, A, D = sum e_c s_c (1 - s_c)) can be accumulated while
// the rows stream through, with the running-max rescaling of an online softmax -- the flash-attention recurrence
// applied to BPR.  A row is needed for one dot product and two FMAs and is then dead.
//
// Decomposition: ONE WARP per sample, no block-level barrier anywhere.  A row is read by LPR = d/4 lanes (16 B each);
// the warp's 32 / LPR lane groups take alternate negatives.  Rows travel global -> shared memory with cp.async (16 B per
// lane, nothing held in registers while in flight) through a per-warp ring of kFlStages stages of kFlRows rows per group,
// so (kFlStages - 1) * kFlRows rows per group are always in flight; each lane reads back only the 16 bytes it copied
// itself.  The sample's ids are fetched first (one coalesced pass) and parked in shared memory as checked 32-bit row
// indices.  The groups' partial states meet once per sample through shuffles (online-softmax combine, fixed order ->
// deterministic).  All 8 warps x 4 CTAs per SM of a B = 4096 batch are resident at once: a single wave, no tail.
// Two float4 per lane execute fewer instructions but spill under the 64-register cap that residency needs, and measured
// slower (0.152 vs 0.150 ms per config-2 step).
#include "common.cuh"

namespace b2r {

constexpr int kFlWarps = 8;       // samples in flight per CTA; 512 CTAs at B = 4096, 4 per SM, all of its shared memory
constexpr int kFlRows = 4;        // rows per lane group per chunk
constexpr int kFlStages = 3;      // ring stages

// sum each of the RCH per-lane values over the LPR lanes of a group with ~RCH + log2(LPR / RCH) shuffles: at every step
// the lanes split the live values in two halves and exchange the half they give up.  Afterwards lane `sub` holds the
// total of value sub / (LPR / RCH)  (the LPR / RCH lanes of one block hold copies).
template <int LPR, int RCH>
__device__ __forceinline__ float fl_group_sum_multi(float (&v)[RCH], int sub) {
    int n = RCH;
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
        if (n > 1) {
            const bool upper = (sub & o) != 0;
            n >>= 1;
#pragma unroll
            for (int i = 0; i < (RCH + 1) / 2; ++i) {
                if (i < n) {
                    const float send = upper ? v[i] : v[i + n];
                    const float keep = upper ? v[i + n] : v[i];
                    v[i] = keep + __shfl_xor_sync(B2R_FULL_MASK, send, o);
                }
            }
        } else {
            v[0] += __shfl_xor_sync(B2R_FULL_MASK, v[0], o);
        }
    }
    return v[0];
}

template <int LPR>
__device__ __forceinline__ float fl_group_max(float v) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(B2R_FULL_MASK, v, o));
    return v;
}

// 16-byte cp.async that reads nothing and writes zeros when `valid` is false (src-size operand): no branch, no separate
// zero store for the padding rows of a sample's last chunk
__device__ __forceinline__ void fl_cp16(void* smem_dst, const void* gsrc, bool valid) {
    const uint32_t sa = (uint32_t)__cvta_generic_to_shared(smem_dst);
    const int nbytes = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(gsrc), "r"(nbytes) : "memory");
}

// D floats per row.  Per warp the ring holds kFlStages * kFlRows * (32 / LPR) rows = kFlStages * kFlRows * 512 bytes.
template <int D>
__global__ void __launch_bounds__(kFlWarps * 32, 4)
k_bprmf_flash(const float* __restrict__ U, const int64_t* __restrict__ uid, int64_t n_users,
              const float* __restrict__ T, const int64_t* __restrict__ ids, int64_t n_t,
              float* __restrict__ pred, float* __restrict__ gout, float* __restrict__ row_loss,
              float* __restrict__ dQ, float* __restrict__ qout, int B, int C, int cpad, int32_t* err_flag,
              float* __restrict__ loss_out, unsigned int* __restrict__ done_counter) {
    constexpr int RCH = kFlRows, ST = kFlStages;
    constexpr int LPR = D / 4;
    constexpr int GPW = 32 / LPR;                 // lane groups (rows in parallel) per warp
    constexpr int RS = LPR / RCH;                 // lanes holding a copy of one row's score after the multi-sum
    static_assert(LPR >= 1 && LPR <= 32 && RCH <= LPR && (RCH & (RCH - 1)) == 0, "shape");
    constexpr int STAGE_F4 = RCH * 32;            // float4 per stage per warp
    extern __shared__ __align__(16) unsigned char fl_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane % LPR, grp = lane / LPR;
    // per-warp regions: ring [ST][RCH][32] float4, then cpad floats of scores, then cpad row indices
    unsigned char* wbase = fl_smem + (size_t)warp * ((size_t)ST * STAGE_F4 * 16 + (size_t)cpad * 8);
    float4* ring = reinterpret_cast<float4*>(wbase);
    float* xs = reinterpret_cast<float*>(wbase + (size_t)ST * STAGE_F4 * 16);
    uint32_t* sid = reinterpret_cast<uint32_t*>(xs + cpad);
    const float invB = 1.f / (float)B;

    for (int64_t b = (int64_t)blockIdx.x * kFlWarps + warp; b < B; b += (int64_t)gridDim.x * kFlWarps) {
        // ---- ids of the sample: one coalesced pass, range-checked once, parked as 32-bit row indices -------------
        const int64_t* idp = ids + b * C;
        for (int c = lane; c < C; c += 32) sid[c] = (uint32_t)checked_id(idp[c], n_t, err_flag);
        const int64_t qrow = checked_id(uid[b], n_users, lane == 0 ? err_flag : nullptr);
        __syncwarp();
        const float* r0p = T + (size_t)sid[0] * D + sub * 4;              // the positive's row (every group: same bytes)
        const float4 q = ld4(U + qrow * D + sub * 4);
        const float pp = 0.f + dot4(q, ld4(r0p));                         // r0 not kept: re-read (L2) for dQ at the end
        // negatives of this group: c = 1 + grp + GPW * k, k = 0 .. ; chunk j covers k in [j * RCH, (j + 1) * RCH)
        const int nneg = C - 1;
        const int nch = (nneg + GPW * RCH - 1) / (GPW * RCH);               // chunks per group (warp-uniform)

        auto issue = [&](int j, int stage) {                               // request chunk j into ring stage `stage`
            if (j < nch) {
                float4* st = ring + stage * STAGE_F4 + lane;
#pragma unroll
                for (int r = 0; r < RCH; ++r) {
                    const int c = 1 + grp + GPW * (j * RCH + r);
                    const bool ok = c < C;
                    fl_cp16(st + r * 32, T + (size_t)sid[ok ? c : 0] * D + sub * 4, ok);
                }
            }
            asm volatile("cp.async.commit_group;\n" ::: "memory");        // one (possibly empty) group per call
        };
#pragma unroll
        for (int j = 0; j < ST - 1; ++j) issue(j, j);

        if (qout != nullptr && grp == 0) st4(qout + b * D + sub * 4, q);
        const float p = group_sum<LPR>(pp);                               // positive's score, known to every group
        if (lane == 0) xs[0] = p;

        float M = -INFINITY, Zl = 0.f, Al = 0.f, Dl = 0.f;                 // running max; per-lane partial sums
        float4 acc1 = make_float4(0.f, 0.f, 0.f, 0.f);                    // sum e s^2 r (this lane's bytes)
        float4 acc2 = make_float4(0.f, 0.f, 0.f, 0.f);                    // sum e r
        int stage = 0, stage_in = ST - 1;
        for (int j = 0; j < nch; ++j) {
            issue(j + ST - 1, stage_in);
            stage_in = (stage_in + 1 == ST) ? 0 : stage_in + 1;
            asm volatile("cp.async.wait_group %0;\n" ::"n"(ST - 1) : "memory");
            const float4* st = ring + stage * STAGE_F4 + lane;
            stage = (stage + 1 == ST) ? 0 : stage + 1;
            float4 r[RCH];
            float d[RCH];
#pragma unroll
            for (int k = 0; k < RCH; ++k) {
                r[k] = st[k * 32];
                d[k] = 0.f + dot4(q, r[k]);
            }
            const float x = fl_group_sum_multi<LPR, RCH>(d, sub);          // score of row sub / RS of this chunk
            const int c_mine = 1 + grp + GPW * (j * RCH + sub / RS);
            const bool valid = c_mine < C;
            const bool speak = (sub % RS) == 0;
            if (valid && speak) xs[c_mine] = x;
            const float mx = fl_group_max<LPR>(valid ? x : -INFINITY);
            if (__any_sync(B2R_FULL_MASK, mx > M)) {                       // a new running max somewhere in the warp: rare
                const float Mn = fmaxf(M, mx);                             // after the first chunks -> rescale
                const float sc = (Mn == -INFINITY) ? 1.f : __expf(M - Mn); // M = -inf -> 0: nothing accumulated yet
                M = Mn;
                Zl *= sc; Al *= sc; Dl *= sc;
                acc1.x *= sc; acc1.y *= sc; acc1.z *= sc; acc1.w *= sc;
                acc2.x *= sc; acc2.y *= sc; acc2.z *= sc; acc2.w *= sc;
            }
            const float e = valid ? __expf(x - M) : 0.f;
            const float s = __fdividef(1.f, 1.f + __expf(x - p));
            const float es = e * s;
            if (speak) {
                Zl += e;
                Al += es;
                Dl = fmaf(es, 1.f - s, Dl);
            }
            const float ess = es * s;
#pragma unroll
            for (int k = 0; k < RCH; ++k) {
                const float ek = __shfl_sync(B2R_FULL_MASK, e, k * RS, LPR);
                const float wk = __shfl_sync(B2R_FULL_MASK, ess, k * RS, LPR);
                fma4(acc2, ek, r[k]);
                fma4(acc1, wk, r[k]);
            }
        }
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");

        // ---- combine: lanes of a group, then the warp's groups (online-softmax rescale), fixed order ---------------
        float Z = group_sum<LPR>(Zl), A = group_sum<LPR>(Al), Dp = group_sum<LPR>(Dl);
        if (GPW > 1) {
            float Mall = M;
#pragma unroll
            for (int o = LPR; o < 32; o <<= 1) Mall = fmaxf(Mall, __shfl_xor_sync(B2R_FULL_MASK, Mall, o));
            const float sg = (M == -INFINITY) ? 0.f : __expf(M - Mall);
            Z *= sg; A *= sg; Dp *= sg;
#pragma unroll
            for (int o = LPR; o < 32; o <<= 1) {
                Z += __shfl_xor_sync(B2R_FULL_MASK, Z, o);
                A += __shfl_xor_sync(B2R_FULL_MASK, A, o);
                Dp += __shfl_xor_sync(B2R_FULL_MASK, Dp, o);
            }
            float* a1 = &acc1.x;
            float* a2 = &acc2.x;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                a1[i] *= sg;
                a2[i] *= sg;
#pragma unroll
                for (int o = LPR; o < 32; o <<= 1) {
                    a1[i] += __shfl_xor_sync(B2R_FULL_MASK, a1[i], o);
                    a2[i] += __shfl_xor_sync(B2R_FULL_MASK, a2[i], o);
                }
            }
            M = Mall;
        }
        const float S = (C > 1) ? __fdividef(A, Z) : 0.f;
        const bool inside = (S >= 1e-8f) && (S <= 1.f - 1e-8f);
        const float dS = inside ? -__fdividef(invB, S) : 0.f;
        const float invZ = (C > 1) ? __fdividef(1.f, Z) : 0.f;
        const float g0 = dS * Dp * invZ;
        const float kz = dS * invZ;
        if (grp == 0) {
            const float4 r0 = ld4(r0p);
            float4 o;
            o.x = fmaf(g0, r0.x, kz * fmaf(-S, acc2.x, acc1.x));
            o.y = fmaf(g0, r0.y, kz * fmaf(-S, acc2.y, acc1.y));
            o.z = fmaf(g0, r0.z, kz * fmaf(-S, acc2.z, acc1.z));
            o.w = fmaf(g0, r0.w, kz * fmaf(-S, acc2.w, acc1.w));
            st4(dQ + b * D + sub * 4, o);
        }
        if (lane == 0) row_loss[b] = -logf(fminf(fmaxf(S, 1e-8f), 1.f - 1e-8f));
        __syncwarp();                                                      // xs[] complete
        // ---- per-candidate gradient (and scores), coalesced ----------------------------------------------------------
        for (int c = lane; c < C; c += 32) {
            const float x = xs[c];
            float g;
            if (c == 0) {
                g = g0;
            } else {
                const float e = __expf(x - M);
                const float s = __fdividef(1.f, 1.f + __expf(x - p));
                g = kz * e * ((s - S) - s * (1.f - s));
            }
            gout[b * C + c] = g;
            if (pred != nullptr) pred[b * C + c] = x;
        }
        __syncwarp();                                                      // before the next sample reuses xs / sid / ring
    }

    // mean of the per-sample losses by the last CTA to finish (fixed summation order -> deterministic)
    if (loss_out != nullptr) {
        constexpr int NT = kFlWarps * 32;
        __shared__ bool last;
        __shared__ float red[NT];
        static_assert((NT & (NT - 1)) == 0, "tree reduction over a power of two");
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) last = (atomicAdd(done_counter, 1u) == gridDim.x - 1);
        __syncthreads();
        if (last) {
            __threadfence();
            float a = 0.f;
            for (int i = threadIdx.x; i < B; i += NT) a += __ldcg(row_loss + i);
            red[threadIdx.x] = a;
            __syncthreads();
            for (int o = NT / 2; o > 0; o >>= 1) {
                if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
                __syncthreads();
            }
            if (threadIdx.x == 0) {
                loss_out[0] = red[0] / (float)B;
                *done_counter = 0u;                                        // ready for the next launch
            }
        }
    }
}

}  // namespace b2r

using namespace b2r;

static int flash_launch(const float* U, const int64_t* uid, int64_t n_users, const float* I, const int64_t* iid,
                        int64_t n_items, float* pred, float* grad_pred, float* row_loss, float* dQ, float* qout, int B,
                        int C, int d, int32_t* err_flag, float* loss_out, unsigned int* done_counter, b2r_stream_t stream) {
    B2R_REQUIRE(U && uid && I && iid && grad_pred && row_loss && dQ, B2R_E_BADARG, "b2r_bprmf_fused_fwd_bwd: null pointer");
    B2R_REQUIRE(B > 0 && C > 0, B2R_E_BADARG, "b2r_bprmf_fused_fwd_bwd: B=%d C=%d", B, C);
    B2R_REQUIRE(aligned16(U) && aligned16(I) && aligned16(dQ), B2R_E_BADARG, "b2r_bprmf_fused_fwd_bwd: alignment");
    // row indices travel as 32-bit values (sid, checked against n_t) and flat positions b * C + c stay below 2^32 - 1
    if (!(d == 32 || d == 64 || d == 128) || C > 1024 || n_items >= 0xffffffffLL || n_users >= 0xffffffffLL ||
        (int64_t)B * C >= 0xffffffffLL)
        return set_error(B2R_E_UNSUPPORTED, "b2r_bprmf_fused_fwd_bwd: d=%d C=%d", d, C);
    const int cpad = (C + 3) / 4 * 4;
    const int64_t need = ((int64_t)B + kFlWarps - 1) / kFlWarps;
    const int64_t cap = (int64_t)sm_count() * 32;                         // beyond that, warps loop over samples
    const int grid = (int)(need < cap ? need : cap);
    const int smem = kFlWarps * (kFlStages * kFlRows * 32 * 16 + cpad * 8);
#define B2R_FLASH_LAUNCH(D_)                                                                                         \
    do {                                                                                                             \
        static int attr_smem = 0;                                                                                    \
        if (smem > attr_smem) {                                                                                      \
            B2R_CUDA_OK(cudaFuncSetAttribute(k_bprmf_flash<D_>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
            attr_smem = smem;                                                                                        \
        }                                                                                                            \
        k_bprmf_flash<D_><<<grid, kFlWarps * 32, smem, as_stream(stream)>>>(                                         \
            U, uid, n_users, I, iid, n_items, pred, grad_pred, row_loss, dQ, qout, B, C, cpad, err_flag, loss_out,   \
            done_counter);                                                                                           \
    } while (0)
    switch (d) {
        case 32: B2R_FLASH_LAUNCH(32); break;
        case 64: B2R_FLASH_LAUNCH(64); break;
        default: B2R_FLASH_LAUNCH(128); break;
    }
#undef B2R_FLASH_LAUNCH
    B2R_LAUNCH_OK("k_bprmf_flash");
    return 0;
}

extern "C" int b2r_bprmf_fused_fwd_bwd(const float* U, const int64_t* uid, int64_t n_users, const float* I,
                                       const int64_t* iid, int64_t n_items, float* pred, float* grad_pred,
                                       float* row_loss, float* dQ, int B, int C, int d, int32_t* err_flag,
                                       b2r_stream_t stream) {
    return flash_launch(U, uid, n_users, I, iid, n_items, pred, grad_pred, row_loss, dQ, nullptr, B, C, d, err_flag, nullptr,
                        nullptr, stream);
}

// same, and the mean loss is produced by the kernel itself (done_counter: a zero-initialised device word the kernel
// leaves zero again) and the gathered user rows are kept (qout [B, d]: the item-side gradient's source, so that the
// user table may be updated while the item table still is); used by the step context
int b2r_bprmf_fused_fwd_bwd_loss(const float* U, const int64_t* uid, int64_t n_users, const float* I, const int64_t* iid,
                                 int64_t n_items, float* grad_pred, float* row_loss, float* dQ, float* qout, int B, int C,
                                 int d, int32_t* err_flag, float* loss_out, unsigned int* done_counter,
                                 b2r_stream_t stream) {
    return flash_launch(U, uid, n_users, I, iid, n_items, nullptr, grad_pred, row_loss, dQ, qout, B, C, d, err_flag, loss_out,
                        done_counter, stream);
}
