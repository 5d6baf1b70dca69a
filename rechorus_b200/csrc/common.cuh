// common.cuh -- shared device/host helpers for libb200rec.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <math.h>

#include "../../include/b200rec.h"

#define B2R_FULL_MASK 0xffffffffu

namespace b2r {

// ---- thread-local error string -------------------------------------------------------------------
char* err_buf();
int   set_error(int code, const char* fmt, ...);

#define B2R_REQUIRE(cond, code, ...)                        \
    do {                                                    \
        if (!(cond)) return b2r::set_error((code), __VA_ARGS__); \
    } while (0)

#define B2R_CUDA_OK(expr)                                                              \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess)                                                         \
            return b2r::set_error((int)_e, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

#define B2R_LAUNCH_OK(name)                                                            \
    do {                                                                               \
        b2r::count_launch();                                                           \
        cudaError_t _e = cudaGetLastError();                                           \
        if (_e != cudaSuccess)                                                         \
            return b2r::set_error((int)_e, "launch of %s failed: %s", name, cudaGetErrorString(_e)); \
    } while (0)

int sm_count();   // cached cudaDevAttrMultiProcessorCount of the current device

// bookkeeping for bench.py: number of kernel launches issued by this library, and optional CUDA-event brackets
// around one tagged kernel (armed per call with b2r_profile_arm, consumed by the next launch with that tag)
void count_launch();
void profile_begin(int tag, cudaStream_t s);
void profile_end(int tag, cudaStream_t s);

// fixed-order mean of B per-sample losses (loss.cu)
int launch_mean_rows(const float* row_loss, float* out, int B, cudaStream_t s);

static inline cudaStream_t as_stream(b2r_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- device helpers ---------------------------------------------------------------------------------

// streaming 128-bit load of a table row chunk: read-only path, do not allocate in L1 (each row chunk is
// used once per CTA; reuse across CTAs is served by the 50 MB L2)
__device__ __forceinline__ float4 ld_row4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

// cached 128-bit load (small, re-used operands such as the query row or the user-row block)
__device__ __forceinline__ float4 ld4(const float* p) {
    return *reinterpret_cast<const float4*>(p);
}

__device__ __forceinline__ void st4(float* p, const float4& v) {
    *reinterpret_cast<float4*>(p) = v;
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
    return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}

__device__ __forceinline__ void fma4(float4& acc, float c, const float4& x) {
    acc.x = fmaf(c, x.x, acc.x);
    acc.y = fmaf(c, x.y, acc.y);
    acc.z = fmaf(c, x.z, acc.z);
    acc.w = fmaf(c, x.w, acc.w);
}

// butterfly sum over the LPR lanes (a power of two <= 32) that share one embedding row
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(B2R_FULL_MASK, v, o);
    return v;
}

__device__ __forceinline__ float warp_sum(float v) { return group_sum<32>(v); }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(B2R_FULL_MASK, v, o));
    return v;
}

// Optimizer constants precomputed once on the host in double precision (1 - beta as torch computes it, the
// step size lr / bias_correction1 and 1 / sqrt(bias_correction2)) so that the per-element update costs one sqrt
// and one division instead of two square roots and three divisions.
struct OptK {
    int kind;          // 0 SGD, 1 Adam, 2 Adagrad
    int state_ld;
    float lr, beta1, beta2, eps, wd, omb1, omb2, step, isb2;
    const float* clock;   // device-side optimizer clock (b2r_optim.clock): step / isb2 are read from it when set
};

// kernels call this once on their private copy: Adam's step size and bias correction come from the device clock
__device__ __forceinline__ void optk_use_clock(OptK& o) {
    if (o.clock != nullptr) {
        o.step = __ldg(o.clock + 1);
        o.isb2 = __ldg(o.clock + 2);
    }
}

static inline OptK make_optk(const b2r_optim& o) {
    OptK k;
    k.kind = o.kind;
    k.state_ld = o.state_ld;
    k.lr = o.lr;
    k.beta1 = o.beta1;
    k.beta2 = o.beta2;
    k.eps = o.eps;
    k.wd = o.weight_decay;
    k.omb1 = (float)(1.0 - (double)o.beta1);
    k.omb2 = (float)(1.0 - (double)o.beta2);
    k.step = (o.kind == 1 && o.bc1 != 0.f) ? (float)((double)o.lr / (double)o.bc1) : o.lr;
    k.isb2 = (o.kind == 1 && o.bc2 > 0.f) ? (float)(1.0 / sqrt((double)o.bc2)) : 1.f;
    k.clock = (o.kind == 1) ? o.clock : nullptr;
    return k;
}

// one element of torch.optim.{SGD, Adam (amsgrad off), Adagrad}.step() with coupled L2 (g += wd * w)
__device__ __forceinline__ void optk_elem(const OptK& o, float& w, float& m, float& v, float gin) {
    const float g = fmaf(o.wd, w, gin);
    if (o.kind == 0) {
        w = fmaf(-o.lr, g, w);
    } else if (o.kind == 1) {
        m = fmaf(o.beta1, m, o.omb1 * g);
        v = fmaf(o.beta2, v, o.omb2 * g * g);
        const float denom = fmaf(sqrtf(v), o.isb2, o.eps);
        w = fmaf(-o.step, m / denom, w);
    } else {
        v = fmaf(g, g, v);
        w = fmaf(-o.lr, g / (sqrtf(v) + o.eps), w);
    }
}

// Same update with hardware-approximate sqrt / reciprocal (MUFU.RSQ / MUFU.RCP, <= 2 ulp each) for the row-sparse
// kernels, which are otherwise instruction-bound on the IEEE sqrt and division sequences: the relative deviation of
// a step is <= ~5e-7, i.e. ~1e-10 absolute at lr = 1e-3.  b2r_dense_optim (exact-reference mode) keeps optk_elem.
__device__ __forceinline__ void optk_elem_fast(const OptK& o, float& w, float& m, float& v, float gin) {
    const float g = fmaf(o.wd, w, gin);
    if (o.kind == 0) {
        w = fmaf(-o.lr, g, w);
    } else if (o.kind == 1) {
        m = fmaf(o.beta1, m, o.omb1 * g);
        v = fmaf(o.beta2, v, o.omb2 * g * g);
        const float sq = v * rsqrtf(fmaxf(v, 1e-38f));                  // sqrt(v), 0 at v = 0
        w = fmaf(-o.step, __fdividef(m, fmaf(sq, o.isb2, o.eps)), w);
    } else {
        v = fmaf(g, g, v);
        const float sq = v * rsqrtf(fmaxf(v, 1e-38f));
        w = fmaf(-o.lr, __fdividef(g, sq + o.eps), w);
    }
}

__device__ __forceinline__ void optk_update4_fast(const OptK& o, float4& w, float4& m, float4& v, const float4& g) {
    optk_elem_fast(o, w.x, m.x, v.x, g.x);
    optk_elem_fast(o, w.y, m.y, v.y, g.y);
    optk_elem_fast(o, w.z, m.z, v.z, g.z);
    optk_elem_fast(o, w.w, m.w, v.w, g.w);
}

// unsigned division by a runtime constant as multiply-high + shift (exact for all 32-bit numerators)
struct FastDiv {
    uint32_t mul, sh1, sh2, div;
};

static inline FastDiv make_fastdiv(uint32_t d) {
    FastDiv f;
    f.div = d < 1 ? 1 : d;
    uint32_t l = 0;
    while (l < 32 && ((uint64_t)1 << l) < f.div) ++l;                    // ceil(log2 d)
    f.mul = (uint32_t)((((uint64_t)1 << 32) * (((uint64_t)1 << l) - f.div)) / f.div + 1);
    f.sh1 = l < 1 ? l : 1;
    f.sh2 = l < 1 ? 0 : l - 1;
    return f;
}

__device__ __forceinline__ uint32_t fastdiv(uint32_t n, const FastDiv& f) {
    const uint32_t t = __umulhi(n, f.mul);
    return (t + ((n - t) >> f.sh1)) >> f.sh2;
}

__device__ __forceinline__ void optk_update4(const OptK& o, float4& w, float4& m, float4& v, const float4& g) {
    optk_elem(o, w.x, m.x, v.x, g.x);
    optk_elem(o, w.y, m.y, v.y, g.y);
    optk_elem(o, w.z, m.z, v.z, g.z);
    optk_elem(o, w.w, m.w, v.w, g.w);
}

// id range check: clamp to row 0 and count the violation (reference: ATen index error)
__device__ __forceinline__ int64_t checked_id(int64_t id, int64_t n_rows, int32_t* err_flag) {
    if (id < 0 || id >= n_rows) {
        if (err_flag) atomicAdd(err_flag, 1);
        return 0;
    }
    return id;
}

}  // namespace b2r
