// tma_gather4_probe.cu -- stand-alone probe (not product code): can the (1+K) x d candidate block of a sample be fetched
// with TMA tile::gather4 (4 table rows per instruction, one issuing lane, mbarrier completion) faster than per-lane
// 16-byte cp.async?  Config-2 shape: 4096 samples x 100 random rows of a [1M, 64] fp32 table; gather + dot.
// Blackwell-only: tile::gather4 does not exist on Hopper, so this design probe does not build for sm_90a and nothing
// in the project builds or runs it (the product kernels use the cp.async path).
// One warp per sample, 8 warps per CTA: lane 0 arms the warp's mbarrier with 25 x 1024 bytes and issues 25 gather4
// copies into the warp's 25.6 KB of shared memory; the warp waits and reduces (16 lanes per row).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

constexpr int D = 64, C = 100, WARPS = 8, ROWB = D * 4, SAMPLE_B = C * ROWB;

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(WARPS * 32, 1)
k_gather4(const __grid_constant__ CUtensorMap tmap, const float* __restrict__ Q, const int64_t* __restrict__ ids,
          float* __restrict__ pred, int B) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bars[WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* mine = smem + (size_t)warp * SAMPLE_B;
    if (lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&bars[warp])) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    uint32_t parity = 0;
    for (int b = blockIdx.x * WARPS + warp; b < B; b += gridDim.x * WARPS) {
        const int64_t* idp = ids + (int64_t)b * C;
        if (lane == 0) {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&bars[warp])), "r"(SAMPLE_B) : "memory");
            for (int g = 0; g < C / 4; ++g) {
                const int r0 = (int)idp[4 * g], r1 = (int)idp[4 * g + 1], r2 = (int)idp[4 * g + 2], r3 = (int)idp[4 * g + 3];
                asm volatile(
                    "cp.async.bulk.tensor.2d.shared::cta.global.tile::gather4.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
                    ::"r"(s32(mine + g * 4 * ROWB)), "l"(&tmap), "r"(0), "r"(r0), "r"(r1), "r"(r2), "r"(r3), "r"(s32(&bars[warp]))
                    : "memory");
            }
        }
        const float4 q = *reinterpret_cast<const float4*>(Q + (int64_t)b * D + (lane & 15) * 4);
        uint32_t done = 0;
        while (!done) {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                         : "=r"(done) : "r"(s32(&bars[warp])), "r"(parity) : "memory");
        }
        parity ^= 1;
        for (int c = lane >> 4; c < C; c += 2) {
            const float4 r = *reinterpret_cast<const float4*>(mine + c * ROWB + (lane & 15) * 16);
            float v = q.x * r.x + q.y * r.y + q.z * r.z + q.w * r.w;
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if ((lane & 15) == 0) pred[(int64_t)b * C + c] = v;
        }
        __syncwarp();
    }
}

// the same decomposition with per-lane 16-byte cp.async (LDGSTS) for comparison
__global__ void __launch_bounds__(WARPS * 32, 1)
k_ldgsts(const float* __restrict__ T, const float* __restrict__ Q, const int64_t* __restrict__ ids, float* __restrict__ pred, int B) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* mine = smem + (size_t)warp * SAMPLE_B;
    for (int b = blockIdx.x * WARPS + warp; b < B; b += gridDim.x * WARPS) {
        const int64_t* idp = ids + (int64_t)b * C;
        for (int c = lane >> 4; c < C; c += 2) {
            const float* src = T + idp[c] * D + (lane & 15) * 4;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s32(mine + c * ROWB + (lane & 15) * 16)), "l"(src) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        const float4 q = *reinterpret_cast<const float4*>(Q + (int64_t)b * D + (lane & 15) * 4);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
        for (int c = lane >> 4; c < C; c += 2) {
            const float4 r = *reinterpret_cast<const float4*>(mine + c * ROWB + (lane & 15) * 16);
            float v = q.x * r.x + q.y * r.y + q.z * r.z + q.w * r.w;
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if ((lane & 15) == 0) pred[(int64_t)b * C + c] = v;
        }
        __syncwarp();
    }
}

int main() {
    const int64_t n_items = 1000000;
    const int B = 4096, ITERS = 20, POOL = 4;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    float *T, *Q, *pred, *pred2;
    int64_t* ids;
    CK(cudaMalloc(&T, n_items * D * 4));
    CK(cudaMalloc(&Q, (size_t)B * D * 4));
    CK(cudaMalloc(&pred, (size_t)B * C * 4));
    CK(cudaMalloc(&pred2, (size_t)B * C * 4));
    CK(cudaMalloc(&ids, (size_t)POOL * B * C * 8));
    std::vector<float> h((size_t)n_items * D);
    uint64_t st = 88172645463325252ull;
    auto rnd = [&]() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return st; };
    for (auto& x : h) x = (float)((rnd() % 2001) - 1000) * 1e-3f;
    CK(cudaMemcpy(T, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(Q, h.data(), (size_t)B * D * 4, cudaMemcpyHostToDevice));
    std::vector<int64_t> hid((size_t)POOL * B * C);
    for (auto& x : hid) x = 1 + (int64_t)(rnd() % (n_items - 1));
    CK(cudaMemcpy(ids, hid.data(), hid.size() * 8, cudaMemcpyHostToDevice));

    CUtensorMap tmap;
    cuuint64_t gdim[2] = {(cuuint64_t)D, (cuuint64_t)n_items};
    cuuint64_t gstr[1] = {(cuuint64_t)ROWB};
    cuuint32_t estr[2] = {1, 1};
    CUresult rc = CUDA_ERROR_UNKNOWN;
    int used_box1 = -1;
    for (int box1 : {1, 4}) {                                  // which box height does gather4 want? try both
        cuuint32_t box[2] = {(cuuint32_t)D, (cuuint32_t)box1};
        rc = cuTensorMapEncodeTiled(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, T, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        printf("cuTensorMapEncodeTiled box {%d, %d}: rc=%d\n", D, box1, (int)rc);
        if (rc == CUDA_SUCCESS) { used_box1 = box1; break; }
    }
    if (rc != CUDA_SUCCESS) return 1;
    const int smem = WARPS * SAMPLE_B;
    CK(cudaFuncSetAttribute(k_gather4, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(k_ldgsts, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const double bytes = (double)B * C * (D * 4 + 8 + 4) + (double)B * D * 4;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    auto timeit = [&](const char* name, auto launch) {
        for (int i = 0; i < 3; ++i) launch(ids + (size_t)(i % POOL) * B * C);
        CK(cudaDeviceSynchronize());
        CK(cudaEventRecord(e0));
        for (int i = 0; i < ITERS; ++i) launch(ids + (size_t)(i % POOL) * B * C);
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        CK(cudaGetLastError());
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        ms /= ITERS;
        printf("%-52s %8.4f ms  %8.1f GB/s\n", name, ms, bytes / ms * 1e-6);
    };
    timeit("per-lane cp.async 16 B (LDGSTS), warp per sample", [&](const int64_t* id) { k_ldgsts<<<sms, WARPS * 32, smem>>>(T, Q, id, pred2, B); });
    k_ldgsts<<<sms, WARPS * 32, smem>>>(T, Q, ids, pred2, B);
    CK(cudaDeviceSynchronize());
    k_gather4<<<sms, WARPS * 32, smem>>>(tmap, Q, ids, pred, B);
    cudaError_t e = cudaDeviceSynchronize();
    printf("gather4 (box height %d) first launch: %s\n", used_box1, cudaGetErrorString(e));
    if (e != cudaSuccess) return 2;
    std::vector<float> a((size_t)B * C), b2((size_t)B * C);
    CK(cudaMemcpy(a.data(), pred, a.size() * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(b2.data(), pred2, b2.size() * 4, cudaMemcpyDeviceToHost));
    double worst = 0;
    for (size_t i = 0; i < a.size(); ++i) { double d = fabs((double)a[i] - b2[i]); if (d > worst) worst = d; }
    printf("gather4 vs cp.async scores: max abs diff %.3e\n", worst);
    timeit("TMA tile::gather4 (4 rows / instruction, 1 issuing lane)", [&](const int64_t* id) { k_gather4<<<sms, WARPS * 32, smem>>>(tmap, Q, id, pred, B); });
    return worst < 1e-6 ? 0 : 3;
}
