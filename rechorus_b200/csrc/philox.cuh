// philox.cuh -- Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; Random123 constants),
// the one counter-based generator of the library: the device negative sampler (sampler.cu) and the dropout masks
// (dropout.cuh) draw from it in disjoint counter domains (bit 31 of counter word 2 is 0 for the sampler, 1 for dropout).
// oracle.philox4x32_10 restates it and is pinned by the Random123 known-answer vectors.
#pragma once
#include <stdint.h>

namespace b2r {

__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                               uint32_t k1) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
        const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0;
        c1 = lo1;
        c2 = n2;
        c3 = lo0;
        k0 += W0;
        k1 += W1;
    }
    return make_uint4(c0, c1, c2, c3);
}

}  // namespace b2r
