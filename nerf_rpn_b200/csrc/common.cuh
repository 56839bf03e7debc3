// Shared host/device helpers for libnerf_rpn_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <atomic>
#include "../../include/nerf_rpn_b200.h"

namespace nrpn {

extern thread_local int g_last_cuda_error;
extern std::atomic<unsigned long long> g_launch_count;

inline int cuda_fail(cudaError_t e) {
    g_last_cuda_error = (int)e;
    return NRPN_ERR_CUDA;
}

// Every kernel launch goes through this so that nrpn_launch_count() is an honest count.
#define NRPN_LAUNCH_CHECK()                                         \
    do {                                                            \
        ::nrpn::g_launch_count.fetch_add(1, std::memory_order_relaxed); \
        cudaError_t e__ = cudaGetLastError();                       \
        if (e__ != cudaSuccess) return ::nrpn::cuda_fail(e__);      \
    } while (0)

#define NRPN_CUDA_TRY(expr)                                         \
    do {                                                            \
        cudaError_t e__ = (expr);                                   \
        if (e__ != cudaSuccess) return ::nrpn::cuda_fail(e__);      \
    } while (0)

inline int num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
    }
    return sms;
}

// 16-bit activation format of a launch: 0 = bf16 (default, BASELINE config 2), 1 = fp16 (same tensor-core rate, 11-bit
// significand: the higher-parity mode of DESIGN.md section 4).  Storage is 2 bytes either way; only conversions differ.
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t pack_act2(float a, float b, int fp16) {
    if (fp16) { __half2 v = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&v); }
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float load_act(const __nv_bfloat16* p, int fp16) {
    return fp16 ? __half2float(*reinterpret_cast<const __half*>(p)) : __bfloat162float(*p);
}
__device__ __forceinline__ void store_act(__nv_bfloat16* p, float v, int fp16) {
    if (fp16) *reinterpret_cast<__half*>(p) = __float2half_rn(v);
    else *p = __float2bfloat16(v);
}
__device__ __forceinline__ float2 unpack_act2(uint32_t u, int fp16) {
    if (fp16) return __half22float2(*reinterpret_cast<const __half2*>(&u));
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}

// One window of nn.MaxPool3d(kernel 2, stride 2, ceil_mode=True): output voxel (b,i,j,k), channels [8g, 8g+8) of a channels-last
// (n,X,Y,Z,C) 16-bit map.  Only positions inside the map are candidates (the last window along an odd extent is partial).
// m: the maximum, fmaxf of the candidates except that a NaN wins (nn.MaxPool3d propagates it).  pos: window position dx*4 + dy*2 + dz of
// the FIRST maximum in PyTorch's scan order (x outer, z inner): a candidate takes it when it exceeds the running maximum or is the first
// NaN.  The inference pool ignores pos; the training pool records it for the backward pass.
__device__ __forceinline__ void maxpool_k2s2_window(const __nv_bfloat16* __restrict__ in, int X, int Y, int Z, int C, int b, int i, int j, int k,
                                                    int g, int fp16, float (&m)[8], int (&pos)[8]) {
#pragma unroll
    for (int q = 0; q < 8; ++q) { m[q] = -INFINITY; pos[q] = 0; }
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
        const int x = 2 * i + dx; if (x >= X) continue;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            const int y = 2 * j + dy; if (y >= Y) continue;
#pragma unroll
            for (int dz = 0; dz < 2; ++dz) {
                const int z = 2 * k + dz; if (z >= Z) continue;
                const uint4 raw = __ldg(reinterpret_cast<const uint4*>(in + ((((size_t)b * X + x) * Y + y) * Z + z) * C + g * 8));
                const uint32_t* h = reinterpret_cast<const uint32_t*>(&raw);
                const int p = dx * 4 + dy * 2 + dz;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float2 f = unpack_act2(h[q >> 1], fp16);
                    const float v = (q & 1) ? f.y : f.x;
                    const bool mnan = m[q] != m[q], vnan = v != v;
                    if (v > m[q] || (vnan && !mnan)) pos[q] = p;
                    m[q] = mnan ? m[q] : (vnan ? v : fmaxf(m[q], v));
                }
            }
        }
    }
}
#endif

template <typename T>
__host__ __device__ inline T ceil_div(T a, T b) { return (a + b - 1) / b; }

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Monotone map float -> uint32 (larger float => larger key); -0 < +0, NaNs sort to the ends.
__host__ __device__ inline uint32_t float_to_ordered(float f) {
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(f);
#else
    union { float f; uint32_t u; } c; c.f = f; uint32_t u = c.u;
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

}  // namespace nrpn
