// half.cuh -- fp16 / bf16 inputs for the element-wise and collector kernels.
//
// Every statistic and every fake-quantised value of a half tensor x is defined as the fp32 result on X = x.float(): the upcast is exact
// and order-preserving, so the kernels load 16 bytes (8 elements) per vector, convert in registers and run the fp32 operators unchanged.
// A fake-quantised half output is that fp32 result rounded once to the output type (round-to-nearest-even, fp16 overflow to +-inf),
// which is what torch's `.to(dtype)` does.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <string.h>
#include <type_traits>

#include "common.cuh"
#include "../../include/ppq_b200.h"

namespace ppqb {

template <class T> struct is_half_t : std::integral_constant<bool, std::is_same<T, __half>::value || std::is_same<T, __nv_bfloat16>::value> {};

static inline bool valid_dtype(int dtype) { return dtype == PPQ_B200_F32 || dtype == PPQ_B200_F16 || dtype == PPQ_B200_BF16; }
static inline bool valid_half_dtype(int dtype) { return dtype == PPQ_B200_F16 || dtype == PPQ_B200_BF16; }

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

template <class T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// f(T()) with T the element type of a dtype code: with_half_type for fp16 / bf16 only, with_elem_type for all three
template <class F> static int with_half_type(int dtype, F &&f) {
    if (dtype == PPQ_B200_F16) return f(__half());
    if (dtype == PPQ_B200_BF16) return f(__nv_bfloat16());
    return (int)cudaErrorInvalidValue;
}
template <class F> static int with_elem_type(int dtype, F &&f) {
    if (dtype == PPQ_B200_F32) return f(float());
    return with_half_type(dtype, f);
}

// one element through the read-only, no-L1-allocate path, as fp32
template <class T> __device__ __forceinline__ float ld_stream1_f(const T *p) {
    unsigned short u;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(u) : "l"(p));
    T v; memcpy(&v, &u, 2);
    return to_f(v);
}
__device__ __forceinline__ float ld_stream1_f(const float *p) { return ld_stream1(p); }

__device__ __forceinline__ uint4 ld_stream_u4(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// 8 packed half elements -> two float4 (elements 0-3, 4-7), exact
template <class T> __device__ __forceinline__ void unpack8(const uint4 &r, float4 &a, float4 &b) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
    float f[8];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        if constexpr (std::is_same<T, __nv_bfloat16>::value) {                 // bf16 -> fp32 is a 16-bit shift
            f[2 * i] = __uint_as_float(w[i] << 16);
            f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
        } else {
            __half2 h; memcpy(&h, &w[i], 4);
            const float2 g = __half22float2(h);
            f[2 * i] = g.x; f[2 * i + 1] = g.y;
        }
    }
    a = make_float4(f[0], f[1], f[2], f[3]);
    b = make_float4(f[4], f[5], f[6], f[7]);
}

// two float4 -> 8 packed half elements, each rounded once to nearest even
template <class T> __device__ __forceinline__ uint4 pack8(const float4 &a, const float4 &b) {
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const unsigned short lo = [&] { T t = from_f<T>(f[2 * i]); unsigned short u; memcpy(&u, &t, 2); return u; }();
        const unsigned short hi = [&] { T t = from_f<T>(f[2 * i + 1]); unsigned short u; memcpy(&u, &t, 2); return u; }();
        w[i] = (uint32_t)lo | ((uint32_t)hi << 16);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// Elements before the first 16-byte boundary of a 2-byte-aligned half pointer (0..7).
template <class T> __host__ __device__ __forceinline__ int64_t head_elems(const T *p) {
    return (int64_t)(((16u - (uint32_t)(reinterpret_cast<uintptr_t>(p) & 15u)) & 15u) >> 1);
}

}  // namespace ppqb
