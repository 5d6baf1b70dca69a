// gather_bench.cu -- stand-alone design-space probe for the K1 gather+dot kernel (not product code).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o build/gather_bench tools/gather_bench.cu
// Times, with CUDA events after warm-up and with a fresh id set per iteration (table 256 MB > 50 MB L2):
//   V0  sequential read of the same number of bytes (what "HBM peak" looks like for this byte count)
//   V1  register-staged LDG.128 gather+dot, RCH rows in flight per lane group, several grid caps
//   V2  bulk-copy (cp.async.bulk -> shared memory, mbarrier completion) staged gather+dot, 2-stage ring
// Prints one line per variant: name, ms, GB/s of algorithmic bytes (rows*256 + ids*8 + preds*4).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)
#define FULL 0xffffffffu

__device__ __forceinline__ float4 ld_nc_na(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 ld_plain(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float dot4(float4 a, float4 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w))); }
template <int LPR> __device__ __forceinline__ float gsum(float v) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// ---------------- V0: streaming read ----------------
__global__ void __launch_bounds__(256) k_stream(const float4* __restrict__ src, int64_t n4, float* out) {
    float acc = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = ld_nc_na(reinterpret_cast<const float*>(src + i));
        acc += v.x + v.y + v.z + v.w;
    }
    if (acc == 123.456f) out[0] = acc;
}

// ---------------- V1: register-staged gather + dot ----------------
template <int LPR, int RCH, bool NA>
__global__ void __launch_bounds__(256) k_v1(const float* __restrict__ Q, const float* __restrict__ T,
                                            const int64_t* __restrict__ ids, float* __restrict__ pred, int B, int C, int nchunk) {
    constexpr int D = LPR * 4, GPC = 256 / LPR, GPW = 32 / LPR;
    const int sub = threadIdx.x % LPR, grp = threadIdx.x / LPR;
    const int64_t total = (int64_t)B * nchunk;
    const int64_t wfirst = (int64_t)blockIdx.x * GPC + (grp / GPW) * GPW;
    for (int64_t wb = wfirst; wb < total; wb += (int64_t)gridDim.x * GPC) {
        const int64_t item = wb + (grp % GPW);
        const bool act = item < total;
        const int b = act ? (int)(item / nchunk) : 0;
        const int c0 = act ? (int)(item % nchunk) * RCH : 0;
        const int nr = act ? min(RCH, C - c0) : 0;
        const float4 q = ld_plain(Q + (int64_t)b * D + sub * 4);
        int64_t my = 0;
        if (sub < nr) my = ids[(int64_t)b * C + c0 + sub];
        float4 r[RCH];
#pragma unroll
        for (int k = 0; k < RCH; ++k) {
            const int64_t idk = __shfl_sync(FULL, my, k, LPR);
            if (k < nr) r[k] = NA ? ld_nc_na(T + idk * D + sub * 4) : ld_plain(T + idk * D + sub * 4);
            else r[k] = make_float4(0, 0, 0, 0);
        }
        float mine = 0.f;
#pragma unroll
        for (int k = 0; k < RCH; ++k) {
            const float s = gsum<LPR>(dot4(q, r[k]));
            if (sub == k) mine = s;
        }
        if (sub < nr) pred[(int64_t)b * C + c0 + sub] = mine;
    }
}

// ---------------- V2: bulk-copy staged gather + dot ----------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nWAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\nbra WAIT_LOOP;\nDONE:\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// CTA walks samples b = blockIdx.x, += gridDim.x; per sample all C rows are staged into one of STAGES smem buffers
template <int LPR, int STAGES, int THREADS>
__global__ void __launch_bounds__(THREADS) k_v2(const float* __restrict__ Q, const float* __restrict__ T,
                                                const int64_t* __restrict__ ids, float* __restrict__ pred, int B, int C) {
    constexpr int D = LPR * 4, GPC = THREADS / LPR;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* rows = reinterpret_cast<float*>(smem_raw);                       // [STAGES][C][D]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (size_t)STAGES * C * D * 4);
    const int sub = threadIdx.x % LPR, grp = threadIdx.x / LPR;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(&bars[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int b, int stage) {
        if (threadIdx.x == 0) mbar_expect_tx(&bars[stage], (uint32_t)C * D * 4);
        for (int c = threadIdx.x; c < C; c += THREADS) {
            const int64_t id = ids[(int64_t)b * C + c];
            bulk_g2s(rows + ((size_t)stage * C + c) * D, T + id * D, D * 4, &bars[stage]);
        }
    };
    int it = 0;
    for (int b = blockIdx.x, s = 0; s < STAGES - 1 && b < B; b += gridDim.x, ++s) issue(b, s);
    for (int b = blockIdx.x; b < B; b += gridDim.x, ++it) {
        const int stage = it % STAGES;
        const int bn = b + (STAGES - 1) * gridDim.x;
        if (bn < B) issue(bn, (it + STAGES - 1) % STAGES);
        mbar_wait(&bars[stage], (it / STAGES) & 1);
        const float4 q = ld_plain(Q + (int64_t)b * D + sub * 4);
        const float* base = rows + (size_t)stage * C * D;
        for (int c0 = 0; c0 < C; c0 += GPC) {           // uniform trip count over the CTA
            const int c = c0 + grp;
            float s = 0.f;
            if (c < C) s = dot4(q, *reinterpret_cast<const float4*>(base + (size_t)c * D + sub * 4));
            s = gsum<LPR>(s);
            if (c < C && sub == 0) pred[(int64_t)b * C + c] = s;
        }
        __syncthreads();     // all reads of this stage done before it is refilled
    }
}

int main(int argc, char** argv) {
    const int64_t n_items = 1000000;
    const int D = 64, B = 4096, C = 100, ITERS = 20, POOL = 6;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    printf("SMs=%d\n", sms);
    float *T, *Q, *pred, *sink;
    int64_t* ids;
    CK(cudaMalloc(&T, n_items * D * 4));
    CK(cudaMalloc(&Q, (size_t)B * D * 4));
    CK(cudaMalloc(&pred, (size_t)B * C * 4));
    CK(cudaMalloc(&sink, 4));
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
    const double bytes = (double)B * C * (D * 4 + 8 + 4) + (double)B * D * 4;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    std::vector<float> ref((size_t)B * C), got((size_t)B * C);

    auto timeit = [&](const char* name, auto launch, bool check) {
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
        double maxerr = -1;
        if (check) {
            launch(ids);
            CK(cudaMemcpy(got.data(), pred, got.size() * 4, cudaMemcpyDeviceToHost));
            maxerr = 0;
            for (size_t i = 0; i < got.size(); ++i) { double e = fabs((double)got[i] - ref[i]); if (e > maxerr) maxerr = e; }
        }
        printf("%-44s %8.4f ms  %8.1f GB/s  maxerr %.2e\n", name, ms, bytes / ms * 1e-6, maxerr);
    };

    // reference result for ids pool 0 from V1<16,8>
    k_v1<16, 8, true><<<sms * 16, 256>>>(Q, T, ids, pred, B, C, (C + 7) / 8);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(ref.data(), pred, ref.size() * 4, cudaMemcpyDeviceToHost));
    {   // spot-check the reference itself on the host
        double worst = 0;
        for (int t = 0; t < 200; ++t) {
            size_t i = rnd() % ref.size();
            int b = (int)(i / C);
            int64_t id = hid[i];
            double s = 0;
            for (int k = 0; k < D; ++k) s += (double)h[(size_t)b * D + k] * h[(size_t)id * D + k];
            if (fabs(s - ref[i]) > worst) worst = fabs(s - ref[i]);
        }
        printf("host spot-check of reference kernel: max |err| = %.3e\n", worst);
    }

    timeit("V0 stream read (same bytes)", [&](const int64_t*) { k_stream<<<sms * 8, 256>>>((const float4*)T, (int64_t)(bytes / 16), sink); }, false);
    for (int cap : {4, 8, 16, 32}) {
        char nm[96];
        snprintf(nm, 96, "V1 LPR16 RCH8 nc.na grid=%dxSM", cap);
        timeit(nm, [&](const int64_t* id) { k_v1<16, 8, true><<<sms * cap, 256>>>(Q, T, id, pred, B, C, (C + 7) / 8); }, true);
    }
    timeit("V1 LPR16 RCH4 nc.na grid=16xSM", [&](const int64_t* id) { k_v1<16, 4, true><<<sms * 16, 256>>>(Q, T, id, pred, B, C, (C + 3) / 4); }, true);
    timeit("V1 LPR16 RCH16 nc.na grid=16xSM", [&](const int64_t* id) { k_v1<16, 16, true><<<sms * 16, 256>>>(Q, T, id, pred, B, C, (C + 15) / 16); }, true);
    timeit("V1 LPR16 RCH8 plain-ld grid=16xSM", [&](const int64_t* id) { k_v1<16, 8, false><<<sms * 16, 256>>>(Q, T, id, pred, B, C, (C + 7) / 8); }, true);
    timeit("V1 LPR16 RCH8 nc.na full grid", [&](const int64_t* id) { k_v1<16, 8, true><<<(B * 13 + 15) / 16, 256>>>(Q, T, id, pred, B, C, (C + 7) / 8); }, true);

    {
        auto run_v2 = [&](auto kern, int stages, int threads, int ctas_per_sm, const char* nm) {
            size_t smem = (size_t)stages * C * D * 4 + 64;
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            timeit(nm, [&](const int64_t* id) { kern<<<sms * ctas_per_sm, threads, smem>>>(Q, T, id, pred, B, C); }, true);
        };
        run_v2(k_v2<16, 2, 128>, 2, 128, 4, "V2 bulk->smem 2 stages 128thr 4 CTA/SM");
        run_v2(k_v2<16, 2, 128>, 2, 128, 3, "V2 bulk->smem 2 stages 128thr 3 CTA/SM");
        run_v2(k_v2<16, 3, 128>, 3, 128, 2, "V2 bulk->smem 3 stages 128thr 2 CTA/SM");
        run_v2(k_v2<16, 2, 256>, 2, 256, 4, "V2 bulk->smem 2 stages 256thr 4 CTA/SM");
        run_v2(k_v2<16, 4, 256>, 4, 256, 2, "V2 bulk->smem 4 stages 256thr 2 CTA/SM");
    }
    return 0;
}
