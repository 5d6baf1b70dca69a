// rmw_bench.cu -- what HBM can deliver for the access pattern of the row-sparse optimizer (not product code).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o build/rmw_bench tools/rmw_bench.cu
// k_apply_sorted (config 2) touches ~336 k of 1 M rows per step: per row it reads 256 B of weights and 512 B of
// interleaved Adam state and writes the same 768 B back.  This probe strips everything else away (no pair walk, no
// contribution gather, trivial arithmetic, registers low enough for full occupancy) and times exactly that traffic,
// with a fresh sorted random row set per iteration, next to a sequential copy of the same byte count -- the ceiling
// the kernel's roofline fraction should be read against.
//   seqcopy   sequential read + write of the same bytes
//   rmw       read w, m|v of each listed row, write them back      (sorted unique rows / unsorted rows)
//   ronly     the reads alone;  wonly  the writes alone
// One line per variant: name, microseconds, GB/s of bytes moved.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <algorithm>
#include <random>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

constexpr int D = 64, LPR = 16, BT = 256, GPC = BT / LPR;

__global__ void __launch_bounds__(BT) k_seqcopy(const float4* __restrict__ src, float4* __restrict__ dst, int64_t n4) {
    for (int64_t i = (int64_t)blockIdx.x * BT + threadIdx.x; i < n4; i += (int64_t)gridDim.x * BT) {
        float4 v = src[i];
        v.x += 1.f;
        dst[i] = v;
    }
}

// MODE 0: read + write, 1: read only, 2: write only.  U rows per lane group in flight.
template <int MODE, int U>
__global__ void __launch_bounds__(BT) k_rmw(const int* __restrict__ rows, int n, float* __restrict__ W,
                                            float* __restrict__ MV, float* sink) {
    const int sub = threadIdx.x % LPR, grp = threadIdx.x / LPR;
    float keep = 0.f;
    for (int j = (blockIdx.x * GPC + grp) * U; j < n; j += gridDim.x * GPC * U) {
        int64_t r[U];
        float4 w[U], m[U], v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) r[u] = j + u < n ? rows[j + u] : -1;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (r[u] < 0) continue;
            if (MODE != 2) {
                w[u] = *reinterpret_cast<const float4*>(W + r[u] * D + sub * 4);
                m[u] = *reinterpret_cast<const float4*>(MV + r[u] * 2 * D + sub * 4);
                v[u] = *reinterpret_cast<const float4*>(MV + r[u] * 2 * D + D + sub * 4);
            } else {
                w[u] = m[u] = v[u] = make_float4(1.f, 2.f, 3.f, (float)j);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (r[u] < 0) continue;
            w[u].x += 1e-3f * m[u].x; m[u].y *= 0.9f; v[u].z *= 0.999f;
            if (MODE != 1) {
                *reinterpret_cast<float4*>(W + r[u] * D + sub * 4) = w[u];
                *reinterpret_cast<float4*>(MV + r[u] * 2 * D + sub * 4) = m[u];
                *reinterpret_cast<float4*>(MV + r[u] * 2 * D + D + sub * 4) = v[u];
            } else {
                keep += w[u].x + m[u].y + v[u].z;
            }
        }
    }
    if (keep == 123.456f) sink[0] = keep;
}

int main(int argc, char** argv) {
    const int64_t n_rows = 1000000;
    const int n_touch = argc > 1 ? atoi(argv[1]) : 336000;
    const int iters = 20, sets = 4;
    float *W, *MV, *sink, *copy_src, *copy_dst;
    CK(cudaMalloc(&W, n_rows * D * 4));
    CK(cudaMalloc(&MV, n_rows * 2 * D * 4));
    CK(cudaMalloc(&sink, 4));
    CK(cudaMemset(W, 0, n_rows * D * 4));
    CK(cudaMemset(MV, 0, n_rows * 2 * D * 4));
    const int64_t bytes_one_way = (int64_t)n_touch * 3 * D * 4;
    CK(cudaMalloc(&copy_src, bytes_one_way));
    CK(cudaMalloc(&copy_dst, bytes_one_way));
    CK(cudaMemset(copy_src, 0, bytes_one_way));
    std::mt19937_64 rng(1);
    std::vector<int*> d_sorted(sets), d_unsorted(sets);
    for (int s = 0; s < sets; ++s) {
        std::vector<int> all(n_rows);
        for (int64_t i = 0; i < n_rows; ++i) all[i] = (int)i;
        std::shuffle(all.begin(), all.end(), rng);
        std::vector<int> pick(all.begin(), all.begin() + n_touch);
        CK(cudaMalloc(&d_unsorted[s], n_touch * 4));
        CK(cudaMemcpy(d_unsorted[s], pick.data(), n_touch * 4, cudaMemcpyHostToDevice));
        std::sort(pick.begin(), pick.end());
        CK(cudaMalloc(&d_sorted[s], n_touch * 4));
        CK(cudaMemcpy(d_sorted[s], pick.data(), n_touch * 4, cudaMemcpyHostToDevice));
    }
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    auto time_it = [&](const char* name, double bytes, auto launch) {
        for (int i = 0; i < 3; ++i) launch(i % sets);
        CK(cudaDeviceSynchronize());
        CK(cudaEventRecord(e0));
        for (int i = 0; i < iters; ++i) launch(i % sets);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        CK(cudaGetLastError());
        printf("%-28s %8.2f us  %8.1f GB/s\n", name, ms / iters * 1e3, bytes / (ms / iters * 1e-3) / 1e9);
    };
    const double rw = 2.0 * bytes_one_way + n_touch * 4.0, ro = bytes_one_way + n_touch * 4.0;
    time_it("seqcopy (same bytes)", 2.0 * bytes_one_way, [&](int) {
        k_seqcopy<<<sms * 8, BT>>>((const float4*)copy_src, (float4*)copy_dst, bytes_one_way / 16);
    });
    for (int ctas : {4, 8, 16}) {
        char nm[64];
        snprintf(nm, sizeof nm, "rmw sorted U=1 grid=%dxSM", ctas);
        time_it(nm, rw, [&](int s) { k_rmw<0, 1><<<sms * ctas, BT>>>(d_sorted[s], n_touch, W, MV, sink); });
        snprintf(nm, sizeof nm, "rmw sorted U=2 grid=%dxSM", ctas);
        time_it(nm, rw, [&](int s) { k_rmw<0, 2><<<sms * ctas, BT>>>(d_sorted[s], n_touch, W, MV, sink); });
    }
    time_it("rmw sorted U=4 grid=8xSM", rw, [&](int s) { k_rmw<0, 4><<<sms * 8, BT>>>(d_sorted[s], n_touch, W, MV, sink); });
    time_it("rmw unsorted U=2 grid=8xSM", rw, [&](int s) { k_rmw<0, 2><<<sms * 8, BT>>>(d_unsorted[s], n_touch, W, MV, sink); });
    time_it("read-only sorted U=2", ro, [&](int s) { k_rmw<1, 2><<<sms * 8, BT>>>(d_sorted[s], n_touch, W, MV, sink); });
    time_it("write-only sorted U=2", ro, [&](int s) { k_rmw<2, 2><<<sms * 8, BT>>>(d_sorted[s], n_touch, W, MV, sink); });
    return 0;
}
