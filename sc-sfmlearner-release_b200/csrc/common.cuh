// Shared host/device helpers for libscsfm (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/scsfm.h"

namespace scsfm {

void set_error(const char* fmt, ...);

#define SCSFM_CHECK_ARG(cond, ...)               \
    do {                                         \
        if (!(cond)) {                           \
            scsfm::set_error(__VA_ARGS__);       \
            return SCSFM_ERR_ARG;                \
        }                                        \
    } while (0)

#define SCSFM_CHECK_CUDA(expr)                                                            \
    do {                                                                                  \
        cudaError_t e__ = (expr);                                                         \
        if (e__ != cudaSuccess) {                                                         \
            scsfm::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),     \
                             __FILE__, __LINE__);                                         \
            return SCSFM_ERR_CUDA;                                                        \
        }                                                                                 \
    } while (0)

// every kernel launch site ends with this macro: it also feeds scsfm_launch_count() (bench.py's "gpu_launches")
extern long long g_launch_count;
#define SCSFM_CHECK_LAUNCH()                                   \
    do {                                                       \
        __atomic_add_fetch(&scsfm::g_launch_count, 1, __ATOMIC_RELAXED); \
        SCSFM_CHECK_CUDA(cudaGetLastError());                  \
    } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum `v` over the block; result valid in thread 0.  `scratch` holds >= 32 floats.
template <int NWARPS>
__device__ __forceinline__ float block_sum(float v, float* scratch) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) scratch[wid] = v;
    __syncthreads();
    float r = 0.f;
    if (wid == 0) {
        r = lane < NWARPS ? scratch[lane] : 0.f;
        r = warp_sum(r);
    }
    return r;
}

// fire-and-forget fp32 add (RED.E.ADD.F32)
__device__ __forceinline__ void red_add(float* p, float v) { atomicAdd(p, v); }

__host__ __device__ __forceinline__ int reflect_index(int i, int n) {
    // ReflectionPad2d(1): -1 -> 1, n -> n-2 (edge sample not repeated)
    return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i);
}

}  // namespace scsfm
