// wgmma_tf32.cuh -- Hopper warpgroup MMA (wgmma.mma_async, sm_90a) for TF32 operands in shared memory, fp32 accumulator
// in registers, plus the descriptor / fence helpers the Linear kernels share.
//
// Both operands are K-major tiles in the SWIZZLE_128B layout: one 128-byte row holds 32 floats of K, the 16-byte chunk index
// is XORed with (row & 7), 8-row groups are 1024 bytes apart, and the tile base is 1024-byte aligned.  One wgmma consumes
// K = 8 floats (32 bytes) of every row; the next K step is the same descriptor with the start address advanced by 32 bytes.
//
// Accumulator fragment of m64nNk8 (thread t of the warpgroup, warp w = t / 32, lane l = t % 32): d[4 j + 2 h + c] holds
// row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + c.
#pragma once
#include <stdint.h>

namespace b2r {

__device__ __forceinline__ uint32_t wg_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// shared-memory matrix descriptor: start address >> 4 in [0,14), LBO (unused for swizzled K-major) = 1 in [16,30),
// SBO = 1024 B >> 4 in [32,46), layout type 1 = SWIZZLE_128B in [62,64)
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)64 << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T; scale_d = 0 overwrites D
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, int scale_d);

#define WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])

template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\twgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7"
        "}, %8, %9, p, 1, 1;\n\t}\n"
        : WG_D8(0)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
        "}, %16, %17, p, 1, 1;\n\t}\n"
        : WG_D8(0), WG_D8(8)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

template <>
__device__ __forceinline__ void wgmma_tf32<48>(float (&d)[24], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\twgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23"
        "}, %24, %25, p, 1, 1;\n\t}\n"
        : WG_D8(0), WG_D8(8), WG_D8(16)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
        "%27,%28,%29,%30,%31"
        "}, %32, %33, p, 1, 1;\n\t}\n"
        : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

template <>
__device__ __forceinline__ void wgmma_tf32<80>(float (&d)[40], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\twgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
        "%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39"
        "}, %40, %41, p, 1, 1;\n\t}\n"
        : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
        "%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,"
        "%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p, 1, 1;\n\t}\n"
        : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

template <>
__device__ __forceinline__ void wgmma_tf32<256>(float (&d)[128], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
        "%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,"
        "%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,"
        "%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,"
        "%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,"
        "%121,%122,%123,%124,%125,%126,%127"
        "}, %128, %129, p, 1, 1;\n\t}\n"
        : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56), WG_D8(64), WG_D8(72), WG_D8(80), WG_D8(88), WG_D8(96), WG_D8(104), WG_D8(112), WG_D8(120)
        : "l"(adesc), "l"(bdesc), "r"(scale_d) : "memory");
}

#undef WG_D8

}  // namespace b2r
