// What one GPU sustains for the row traffic of the CSR-fed BPR/SGD step, per form of the in-place row update.
// Standalone (not part of the library):
//
//     nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o row_update_probe profiles/row_update_probe.cu
//     ./row_update_probe            # one JSON object per (row law, update form) on stdout
//
// A 12.5 M x 128 fp32 table (the benchmark's item table) and 3 x 2^20 row ids per launch (the rows of one
// 2^20-triplet step).  One warp per row, lane l owns floats [4l, 4l + 4): it reads the row, reduces it across the
// warp (so the update depends on the whole row, as the step's does) and then, by mode,
//   read        does nothing more;
//   store       writes the updated row back with plain float4 stores;
//   red_v4      adds the delta with one float4 RED.ADD per lane;
//   bulk_reduce stages the delta row in shared memory and adds it with ONE cp.reduce.async.bulk .add.f32, waiting
//               for the copy engine to have read the previous row before staging the next (as the step did).
// Each warp keeps two rows in flight.  Row laws: uniform over the table; the benchmark's positive-item law
// (continuous Zipf(1.05) inverse CDF, the 16384 most popular ids first, the rest spread by a multiplicative hash);
// and the step's mix (user and negative uniform, positive Zipf).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#define CK(x)                                                                             \
    do {                                                                                  \
        cudaError_t e_ = (x);                                                             \
        if (e_ != cudaSuccess) {                                                          \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));   \
            return 1;                                                                     \
        }                                                                                 \
    } while (0)

constexpr int D = 128;
constexpr int64_t kRows = 12500000, kIds = 3ll << 20;
constexpr int kHead = 16384;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int MODE>
__device__ __forceinline__ void update(float* p, float4 v, float s, float* stage, int lane) {
    const float4 d = make_float4(1e-7f * s, -1e-7f * s, 1e-7f * v.x, -1e-7f * v.y);
    if constexpr (MODE == 1) {
        *reinterpret_cast<float4*>(p) = make_float4(v.x + d.x, v.y + d.y, v.z + d.z, v.w + d.w);
    } else if constexpr (MODE == 2) {
        atomicAdd(reinterpret_cast<float4*>(p), d);
    } else if constexpr (MODE == 3) {
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        __syncwarp();
        *reinterpret_cast<float4*>(stage + lane * 4) = d;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
            const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(stage);
            asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
                         ::"l"(p), "r"(saddr), "r"((uint32_t)(D * 4)) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(256) probe_kernel(float* __restrict__ table, const int32_t* __restrict__ ids, int64_t n,
                                                    float* __restrict__ sink) {
    __shared__ __align__(16) float stage[8][2][D];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float acc = 0.f;
    for (int64_t r = ((int64_t)blockIdx.x * 8 + warp) * 2; r < n; r += (int64_t)gridDim.x * 16) {
        float* p0 = table + (size_t)ids[r] * D + lane * 4;
        float* p1 = table + (size_t)ids[r + 1 < n ? r + 1 : r] * D + lane * 4;
        const float4 v0 = *reinterpret_cast<const float4*>(p0), v1 = *reinterpret_cast<const float4*>(p1);
        const float s0 = warp_sum(v0.x + v0.y + v0.z + v0.w), s1 = warp_sum(v1.x + v1.y + v1.z + v1.w);
        if constexpr (MODE == 0) {
            acc += s0 + s1;
        } else {
            update<MODE>(p0, v0, s0, stage[warp][0], lane);
            if (r + 1 < n) update<MODE>(p1, v1, s1, stage[warp][1], lane);
        }
    }
    if constexpr (MODE == 3) {
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
    if (acc == 1234.5f) *sink = acc;      // keeps the read-only mode's loads
}

static int64_t zipf_id(double x) {       // bench.synth_shard_csr's law and relabelling
    const double a = 1.05, ni = (double)kRows;
    int64_t r = (int64_t)std::pow((std::pow(ni, 1 - a) - 1) * x + 1, 1 / (1 - a));
    r = std::min<int64_t>(std::max<int64_t>(r, 1), kRows) - 1;
    return r < kHead ? r : kHead + (int64_t)(((uint64_t)(r - kHead) * 2654435761ull) % (uint64_t)(kRows - kHead));
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    float* table;
    int32_t* ids;
    float* sink;
    CK(cudaMalloc(&table, (size_t)kRows * D * sizeof(float)));
    CK(cudaMalloc(&ids, kIds * sizeof(int32_t)));
    CK(cudaMalloc(&sink, sizeof(float)));
    CK(cudaMemset(table, 0, (size_t)kRows * D * sizeof(float)));
    const char* laws[3] = {"uniform", "zipf", "step_mix"};
    const char* modes[4] = {"read", "store", "red_v4", "bulk_reduce"};
    std::mt19937_64 rng(7);
    std::uniform_real_distribution<double> u01(0.0, 1.0);
    std::uniform_int_distribution<int64_t> uni(0, kRows - 1);
    std::vector<int32_t> h(kIds);
    const int grid = prop.multiProcessorCount * 8;
    for (int law = 0; law < 3; ++law) {
        for (int64_t k = 0; k < kIds; ++k) {
            const bool z = law == 1 || (law == 2 && k % 3 == 1);      // step_mix: (user, positive, negative)
            h[k] = (int32_t)(z ? zipf_id(u01(rng)) : uni(rng));
        }
        CK(cudaMemcpy(ids, h.data(), kIds * sizeof(int32_t), cudaMemcpyHostToDevice));
        for (int mode = 0; mode < 4; ++mode) {
            auto launch = [&]() {
                if (mode == 0) probe_kernel<0><<<grid, 256>>>(table, ids, kIds, sink);
                else if (mode == 1) probe_kernel<1><<<grid, 256>>>(table, ids, kIds, sink);
                else if (mode == 2) probe_kernel<2><<<grid, 256>>>(table, ids, kIds, sink);
                else probe_kernel<3><<<grid, 256>>>(table, ids, kIds, sink);
            };
            for (int w = 0; w < 3; ++w) launch();
            CK(cudaGetLastError());
            const int K = 10;
            cudaEvent_t a, b;
            CK(cudaEventCreate(&a));
            CK(cudaEventCreate(&b));
            CK(cudaEventRecord(a));
            for (int k = 0; k < K; ++k) launch();
            CK(cudaEventRecord(b));
            CK(cudaEventSynchronize(b));
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, a, b));
            const double us = ms * 1e3 / K;
            const double bytes = (double)kIds * D * 4 * (mode == 0 ? 1 : 2);   // rows read (+ rows updated)
            printf("{\"law\": \"%s\", \"mode\": \"%s\", \"launch_us\": %.1f, \"rows_per_s\": %.4g, \"GBps_read_plus_update\": %.1f}\n",
                   laws[law], modes[mode], us, kIds / (us * 1e-6), bytes / (us * 1e-6) / 1e9);
            CK(cudaEventDestroy(a));
            CK(cudaEventDestroy(b));
        }
    }
    CK(cudaFree(table));
    CK(cudaFree(ids));
    CK(cudaFree(sink));
    return 0;
}
