// Shared helpers for the neurec_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/neurec_b200.h"

namespace nrc {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;

void set_error(const char* fmt, ...);

#define NRC_CUDA_CHECK(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            nrc::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                           __LINE__);                                                     \
            return NRC_E_CUDA;                                                            \
        }                                                                                 \
    } while (0)

#define NRC_REQUIRE(cond, code, ...)     \
    do {                                 \
        if (!(cond)) {                   \
            nrc::set_error(__VA_ARGS__); \
            return (code);               \
        }                                \
    } while (0)

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Number of SMs of the current device (132 on H100 SXM); cached.
int sm_count();

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// A load that is ld.global.cg when CG (through L2 only: for the persistent kernels, whose tables change between
// grid barriers), an ordinary load otherwise.
template <bool CG, class T>
__device__ __forceinline__ T ld(const T* p) {
    if constexpr (CG) return __ldcg(p);
    else return *p;
}

// One lane's slice of a row, VEC = dim / 32 consecutive floats: one float4 / float2 / float access.
template <int VEC, bool CG = false>
__device__ __forceinline__ void ld_vec(const float* p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 x = ld<CG>(reinterpret_cast<const float4*>(p));
        v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
    } else if constexpr (VEC == 2) {
        const float2 x = ld<CG>(reinterpret_cast<const float2*>(p));
        v[0] = x.x; v[1] = x.y;
    } else {
        v[0] = ld<CG>(p);
    }
}

template <int VEC>
__device__ __forceinline__ void st_vec(float* p, const float (&v)[VEC]) {
    if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else if constexpr (VEC == 2) *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
    else *p = v[0];
}

// p[t] += d[t] with one vector RED.ADD (float4 / float2 atomics, sm_90+)
template <int VEC>
__device__ __forceinline__ void red_vec(float* p, const float (&d)[VEC]) {
    if constexpr (VEC == 4) atomicAdd(reinterpret_cast<float4*>(p), make_float4(d[0], d[1], d[2], d[3]));
    else if constexpr (VEC == 2) atomicAdd(reinterpret_cast<float2*>(p), make_float2(d[0], d[1]));
    else atomicAdd(p, d[0]);
}

// Membership in an ascending int32 array.  Rows of up to 8 entries (the common case for the sampler's
// rejection test on sparse users) are compared with independent loads -- one memory round trip instead
// of log2(n) dependent ones; longer rows by binary search.
__device__ __forceinline__ bool sorted_contains(const int32_t* __restrict__ a, int64_t n,
                                                int32_t x) {
    if (n <= 0) return false;
    if (n <= 8) {
        bool hit = false;
#pragma unroll
        for (int i = 0; i < 8; ++i) hit |= (i < n) && (__ldg(a + (i < n ? i : 0)) == x);
        return hit;
    }
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < x) lo = mid + 1; else hi = mid;
    }
    return lo < n && __ldg(a + lo) == x;
}

}  // namespace nrc
