// Shared host/device helpers for the hipie_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "../../include/hipie_b200.h"

namespace hipie {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launch_count;

inline void count_launch(int n = 1) { g_launch_count.fetch_add(n, std::memory_order_relaxed); }

#define HIPIE_CHECK_ARG(cond, ...)                \
    do {                                          \
        if (!(cond)) {                            \
            ::hipie::set_error(__VA_ARGS__);      \
            return HIPIE_EINVAL;                  \
        }                                         \
    } while (0)

#define HIPIE_CHECK_CUDA(expr)                                                              \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            ::hipie::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                               __FILE__, __LINE__);                                         \
            return HIPIE_ECUDA;                                                             \
        }                                                                                   \
    } while (0)

#define HIPIE_CHECK_LAUNCH()                                                                \
    do {                                                                                    \
        cudaError_t _e = cudaGetLastError();                                                \
        if (_e != cudaSuccess) {                                                            \
            ::hipie::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),  \
                               __FILE__, __LINE__);                                         \
            return HIPIE_ECUDA;                                                             \
        }                                                                                   \
        ::hipie::count_launch();                                                            \
    } while (0)

// Dynamic shared-memory opt-in (a per-device function attribute): raise it on the CURRENT device when a launch needs more.
#define HIPIE_ENSURE_SMEM(func, bytes)                                                                          \
    do {                                                                                                        \
        static int _smem_set[64] = {};                                                                          \
        int _dev = 0;                                                                                           \
        HIPIE_CHECK_CUDA(cudaGetDevice(&_dev));                                                                 \
        if (_dev < 0 || _dev >= 64) _dev = 0;                                                                   \
        if ((int)(bytes) > _smem_set[_dev]) {                                                                   \
            HIPIE_CHECK_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
            _smem_set[_dev] = (int)(bytes);                                                                     \
        }                                                                                                       \
    } while (0)

static inline int num_sms() {
    static int n[64] = {};          // per device (several devices in one process see their own SM count)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (n[dev] == 0) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        n[dev] = v > 0 ? v : 132;
    }
    return n[dev];
}

// ---- device helpers ------------------------------------------------------------------------
__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ float bf16_round(float x) {
    return __bfloat162float(__float2bfloat16_rn(x));
}

// hi = bf16(x), lo = bf16(x - hi) for a pair of floats; packed conversions (one F2FP per pair, ALU pipe)
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const uint32_t hu = *reinterpret_cast<uint32_t*>(&h);
    const float ha = __uint_as_float(hu << 16), hb = __uint_as_float(hu & 0xffff0000u);
    __nv_bfloat162 l = __floats2bfloat162_rn(a - ha, b - hb);
    hi = hu;
    lo = *reinterpret_cast<uint32_t*>(&l);
}

__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
// hi/lo planes of a pair: bf16 split, or (fp16 != 0) one IEEE fp16 plane
// ---- fp16 + e4m3 split (prec 6 of hipie_gemm): x = h + l, h = fp16(x); planes fp16(h), e4m3(h), e4m3(2^10 l) -----------------
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
    return lo | (hi << 16);
}
// Layout of an e4m3 operand plane (rows, 2K bytes): the two slots (hi-like / lo-like factor of the cross terms) are interleaved in
// groups of 32 columns -- element k of slot 0 at byte (k / 32) * 64 + k % 32, of slot 1 at +32 -- so that a producer's 32-column
// chunk is ONE 64-byte row segment (one TMA box with 64-byte rows in the GEMM epilogue).  The contraction over 2K is order-free as
// long as A8 and W8 use the same order; K % 32 == 0.
__host__ __device__ __forceinline__ int64_t e4m3_slot0(int64_t k) { return (k >> 5) * 64 + (k & 31); }

__device__ __forceinline__ void split4_f16_e4m3(const float4& x, uint2& h16, uint32_t& hi8, uint32_t& lo8) {
    const __half2 h0 = __floats2half2_rn(x.x, x.y), h1 = __floats2half2_rn(x.z, x.w);
    h16.x = *reinterpret_cast<const uint32_t*>(&h0);
    h16.y = *reinterpret_cast<const uint32_t*>(&h1);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    hi8 = pack_e4m3x4(f0.x, f0.y, f1.x, f1.y);
    lo8 = pack_e4m3x4((x.x - f0.x) * 1024.f, (x.y - f0.y) * 1024.f, (x.z - f1.x) * 1024.f, (x.w - f1.y) * 1024.f);
}

__device__ __forceinline__ void split2m(float a, float b, uint32_t& hi, uint32_t& lo, int fp16) {
    if (fp16) { hi = pack_f16x2(a, b); lo = 0u; }
    else split2(a, b, hi, lo);
}

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace hipie
