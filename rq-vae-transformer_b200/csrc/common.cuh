// rqb200 -- shared helpers for the sm_90a kernels (error plumbing, warp/block reductions, launch counter).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <algorithm>
#include <atomic>
#include <string>

#include "../../include/rqb200.h"

namespace rqb {

void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
extern thread_local int64_t g_launches;          // kernels launched on this thread since the last reset

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    g_launches++;
    if (e != cudaSuccess) return fail(RQB200_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
    return 0;
}

#define RQB_TRY(expr)            \
    do {                         \
        int _rc = (expr);        \
        if (_rc != 0) return _rc; \
    } while (0)

#define RQB_CUDA(expr)                                                                     \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) return rqb::fail(RQB200_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: remember it per (call site, device), thread-safe.
// usage: RQB_ENSURE_SMEM(bytes, kernel<template, args>);
#define RQB_ENSURE_SMEM(bytes, ...)                                                                               \
    do {                                                                                                          \
        static std::atomic<uint64_t> _done{0};                                                                    \
        int _dev = 0;                                                                                             \
        RQB_CUDA(cudaGetDevice(&_dev));                                                                           \
        const uint64_t _bit = 1ull << (_dev & 63);                                                                \
        if (!(_done.load(std::memory_order_acquire) & _bit)) {                                                    \
            RQB_CUDA(cudaFuncSetAttribute(__VA_ARGS__, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
            _done.fetch_or(_bit, std::memory_order_release);                                                      \
        }                                                                                                         \
    } while (0)

// cudaLaunchKernelEx with the programmatic-stream-serialization attribute `pdl`: the kernel may start before the previous kernel on
// the stream has finished, so it must read upstream data only after griddepcontrol.wait.
template <typename... KArgs, typename... Args>
int launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    RQB_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
    g_launches++;
    return 0;
}

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

// the grid of a 256-thread grid-stride launch over n elements: one CTA per 256 elements, at least 1 and at most 8192
inline unsigned grid_1d(int64_t n) { return (unsigned)std::min<int64_t>(std::max<int64_t>(ceil_div(n, 256), 1), 8192); }
// the items (images, pairs) a layer-plan call runs at once: as many as fit in 2 GiB of workspace, at least 1 and at most B; a larger
// batch runs in chunks of that many inside one call
inline int chunk_items(int B, size_t bytes_per_item) {
    const int64_t fit = std::max<int64_t>(1, (int64_t)((size_t(2) << 30) / bytes_per_item));
    return (int)std::min<int64_t>(B, fit);
}

// bump allocator over the caller's workspace
struct Arena {
    char* base;
    size_t cap, off;
    Arena(void* p, size_t c) : base(reinterpret_cast<char*>(p)), cap(c), off(0) {}
    template <typename T>
    T* take(size_t n) {
        off = align_up(off, 256);
        T* r = reinterpret_cast<T*>(base + off);
        off += n * sizeof(T);
        return r;
    }
    bool ok() const { return off <= cap; }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// block-wide reductions through shared scratch (>= 33 floats); all threads get the result
__device__ __forceinline__ float block_sum(float v, float* scratch) {
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) scratch[wid] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : 0.f;
    r = warp_sum(r);
    return r;
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) scratch[wid] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : -INFINITY;
    r = warp_max(r);
    return r;
}

// 16-bit tensor-core operand storage of the fast tier.  `bf` selects the format at run time (uniform per launch): 0 = IEEE fp16
// (the reference's autocast class, transformers.py:114,206), 1 = bf16.  Same bytes, same wgmma rate.
typedef uint16_t h16;
__device__ __forceinline__ uint32_t pack_h16x2(float a, float b, int bf) {
    if (bf) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_h16x2(uint32_t v, int bf) {
    if (bf) return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v));
    return __half22float2(*reinterpret_cast<__half2*>(&v));
}
__device__ __forceinline__ h16 pack_h16(float a, int bf) {
    if (bf) {
        __nv_bfloat16 h = __float2bfloat16(a);
        return *reinterpret_cast<h16*>(&h);
    }
    __half h = __float2half_rn(a);
    return *reinterpret_cast<h16*>(&h);
}

// The split-fp16 form of the fast tier's conv operands and weights: hi = fp16(v), lo = fp16(v - hi)
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}
__device__ __forceinline__ void split_f16x2(float a, float b, __half2& hi, __half2& lo) {
    hi = __floats2half2_rn(a, b);
    const float2 f = __half22float2(hi);
    lo = __floats2half2_rn(a - f.x, b - f.y);
}

// GELU in the exact erf form (F.gelu's default, the reference's gelu='v1')
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// CLIP's QuickGELU, x * sigmoid(1.702 x), with an IEEE division so the exact tier's value does not depend on build flags
__device__ __forceinline__ float quick_gelu(float x) { return __fdiv_rn(x, 1.0f + expf(-1.702f * x)); }

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }

}  // namespace rqb
