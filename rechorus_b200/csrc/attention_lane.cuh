// attention_lane.cuh -- the per-lane arithmetic of the lane-per-(row, head) attention kernels (attention_rt.cu,
// attention_tiled.cu).  Both files run their rows through these functions, so a lane's sequence of roundings is the
// same whichever kernel stages its operands.
#pragma once
#include "common.cuh"

namespace b2r {

static constexpr float kLog2e = 1.4426950408889634f;

template <int DK>
__device__ __forceinline__ void load_vec(float (&dst)[DK], const float* src) {
#pragma unroll
    for (int c = 0; c < DK; c += 4) {
        const float4 t = *reinterpret_cast<const float4*>(src + c);
        dst[c] = t.x; dst[c + 1] = t.y; dst[c + 2] = t.z; dst[c + 3] = t.w;
    }
}

template <int DK>
__device__ __forceinline__ void store_vec(float* dst, const float (&src)[DK]) {
#pragma unroll
    for (int c = 0; c < DK; c += 4) *reinterpret_cast<float4*>(dst + c) = make_float4(src[c], src[c + 1], src[c + 2], src[c + 3]);
}

// dot of a register vector with a shared-memory row chunk (broadcast loads when the address is warp-uniform)
template <int DK>
__device__ __forceinline__ float dot_sm(const float (&a)[DK], const float* b) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < DK; c += 4) {
        const float4 t = *reinterpret_cast<const float4*>(b + c);
        s = fmaf(a[c], t.x, s); s = fmaf(a[c + 1], t.y, s); s = fmaf(a[c + 2], t.z, s); s = fmaf(a[c + 3], t.w, s);
    }
    return s;
}

template <int DK>
__device__ __forceinline__ void axpy_sm(float (&acc)[DK], float w, const float* b) {
#pragma unroll
    for (int c = 0; c < DK; c += 4) {
        const float4 t = *reinterpret_cast<const float4*>(b + c);
        acc[c] = fmaf(w, t.x, acc[c]); acc[c + 1] = fmaf(w, t.y, acc[c + 1]);
        acc[c + 2] = fmaf(w, t.z, acc[c + 2]); acc[c + 3] = fmaf(w, t.w, acc[c + 3]);
    }
}

__device__ __forceinline__ int live_rows(const int64_t* live, int b, int L) {
    if (live == nullptr) return L;
    const int64_t lv = live[b];
    return lv < 0 ? 0 : (lv > L ? L : (int)lv);
}

}  // namespace b2r
