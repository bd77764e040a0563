// Shared helpers for libgen6d_b200.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/gen6d_b200.h"

namespace g6d {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

inline cudaStream_t as_stream(g6d_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// call after every kernel launch
#define G6D_CHECK_LAUNCH(name)                                                        \
    do {                                                                              \
        cudaError_t e__ = cudaGetLastError();                                         \
        if (e__ != cudaSuccess) {                                                     \
            g6d::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
            return G6D_ECUDA;                                                         \
        }                                                                             \
        g6d::count_launch();                                                          \
    } while (0)

#define G6D_REQUIRE(cond, ...)            \
    do {                                  \
        if (!(cond)) {                    \
            g6d::set_error(__VA_ARGS__);  \
            return G6D_EINVAL;            \
        }                                 \
    } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// streaming (read-once) 128-bit load that does not pollute L1
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

}  // namespace g6d
