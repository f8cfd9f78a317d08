// Shared helpers for the mmrec_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/mmrec_b200.h"

namespace mmrec {

void set_error(const char* fmt, ...);

#define MMREC_CHECK_ARG(cond, ...)                 \
    do {                                           \
        if (!(cond)) {                             \
            mmrec::set_error(__VA_ARGS__);         \
            return MMREC_EINVAL;                   \
        }                                          \
    } while (0)

#define MMREC_CUDA(call)                                                                          \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            mmrec::set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return MMREC_ECUDA;                                                                   \
        }                                                                                         \
    } while (0)

extern long long g_launches;   // kernels launched (mmrec_launch_count)
#define MMREC_LAUNCH_CHECK()            \
    do {                                \
        ++::mmrec::g_launches;          \
        MMREC_CUDA(cudaGetLastError()); \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// number of SMs of the current device (cached)
int sm_count();

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// order-preserving float -> uint32 key (ascending); +0 > -0, NaN (positive) largest
__device__ __forceinline__ uint32_t float_key(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}

}  // namespace mmrec
