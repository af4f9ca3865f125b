// common.cuh — shared host/device helpers for libngp_b200 (sm_90a only).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ngp_b200.h"

// ---- host side: error reporting + launch accounting -------------------------------------
namespace ngp {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

int sm_count();

}  // namespace ngp

#define NGP_REQUIRE(cond, msg)                       \
    do {                                             \
        if (!(cond)) {                               \
            ngp::set_error("%s: %s", __func__, msg); \
            return -1;                               \
        }                                            \
    } while (0)

#define NGP_LAUNCHED(name)                 \
    do {                                   \
        ngp::count_launch();               \
        int rc_ = ngp::check_launch(name); \
        if (rc_) return rc_;               \
    } while (0)

// ---- device side --------------------------------------------------------------------------
#ifdef __CUDACC__

// Strict IEEE fp32 in source order: the marching code must be bit-identical to the CPU oracle
// (gcc -ffp-contract=off), so every arithmetic op is an explicit round-to-nearest intrinsic
// that nvcc may not contract into an FMA.
__device__ __forceinline__ float f_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float f_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float f_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float f_div(float a, float b) { return __fdiv_rn(a, b); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// inclusive prefix sum / product across the warp
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    return v;
}
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v *= n;
    }
    return v;
}

template <typename T>
__device__ __forceinline__ float load_as_float(const T* p, int64_t i);
template <>
__device__ __forceinline__ float load_as_float<float>(const float* p, int64_t i) { return p[i]; }
template <>
__device__ __forceinline__ float load_as_float<__half>(const __half* p, int64_t i) { return __half2float(p[i]); }

template <typename T>
__device__ __forceinline__ void store_from_float(T* p, int64_t i, float v);
template <>
__device__ __forceinline__ void store_from_float<float>(float* p, int64_t i, float v) { p[i] = v; }
template <>
__device__ __forceinline__ void store_from_float<__half>(__half* p, int64_t i, float v) { p[i] = __float2half_rn(v); }

#endif  // __CUDACC__
