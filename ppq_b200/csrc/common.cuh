// common.cuh -- device helpers shared by the sm_90a kernels of libppq_b200.
//
// Numerics contract (restated in DESIGN.md, proven against oracle/ and the reference's own CUDA build):
//   round2int<mode>   == _round2int            (/root/reference/ppq/csrc/cuda/common.cuh:88-114)
//   ExactDiv          == IEEE fp32 division    (the reference insists on x / s, never x * (1/s): linear.cu:73-74)
// No torch here: this translation unit family only needs the CUDA runtime.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ppqb {

// SM count of the CURRENT device (H100 SXM: 132), queried once per device ordinal; every persistent grid is sized from it.
inline int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    int v = cached[dev];
    if (v == 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        cached[dev] = v;
    }
    return v;
}
constexpr int RND_HALF_EVEN = 0, RND_HALF_UP = 1, RND_HALF_DOWN = 2, RND_HALF_TOWARDS_ZERO = 3,
              RND_HALF_FAR_FROM_ZERO = 4, RND_TO_NEAR_INT = 5, RND_UP = 6, RND_DOWN = 7;

// ---- rounding ---------------------------------------------------------------------------------------
// All conversions saturate and send NaN to 0 (PTX cvt.*.s32.*), which is what the reference's implicit
// float->int / double->int conversions compile to.
// The reference evaluates its "+ .5" modes in double (`floor(value + .5)` promotes the float).  fp64 throughput on this part is a
// small fraction of fp32, so the same integers are produced in fp32: with t = floor(v), floor(v + .5) = t + [v - t >= .5].  The
// subtraction may round (tiny negative v: 1 - 1e-30 -> 1), but rounding is monotonic and .5 is representable, so the comparison
// `>= .5` is decided correctly; a `> .5` comparison would not be, which is why the "half down" form is built on ceil() instead
// of reusing floor().  Saturation and NaN -> 0 come from the F2I conversion exactly as in the double path (the fraction of a
// saturated or non-finite v is 0 or NaN, so nothing is added).
__device__ __forceinline__ int round_half_up(float v)   { return __float2int_rd(v) + (__fsub_rn(v, floorf(v)) >= 0.5f ? 1 : 0); }   // floor(v + .5)
__device__ __forceinline__ int round_half_down(float v) { return __float2int_ru(v) - (__fsub_rn(ceilf(v), v) >= 0.5f ? 1 : 0); }    // ceil(v - .5)

template <int MODE>
__device__ __forceinline__ int round2int(float v) {
    if constexpr (MODE == RND_HALF_EVEN) {
        return __float2int_rn(v);                                   // nearbyint -> int  (one F2I)
    } else if constexpr (MODE == RND_HALF_UP) {
        return round_half_up(v);
    } else if constexpr (MODE == RND_HALF_DOWN) {
        return round_half_down(v);
    } else if constexpr (MODE == RND_HALF_TOWARDS_ZERO) {
        return v > 0.f ? round_half_down(v) : round_half_up(v);
    } else if constexpr (MODE == RND_UP) {
        return __float2int_ru(v);
    } else if constexpr (MODE == RND_DOWN) {
        return __float2int_rd(v);
    } else {                                                        // HALF_FAR_FROM_ZERO, and TO_NEAR_INT = round(): the same function
        return v > 0.f ? round_half_up(v) : round_half_down(v);
    }
}

// Run-time mode (warp-uniform): the four half-way modes share one branch-free body selected by two uniform flags.
__device__ __forceinline__ int round2int_dyn(float v, int mode) {
    if (mode == RND_HALF_EVEN) return __float2int_rn(v);
    if (mode == RND_UP)        return __float2int_ru(v);
    if (mode == RND_DOWN)      return __float2int_rd(v);
    const bool pos_up = (mode != RND_HALF_DOWN) && (mode != RND_HALF_TOWARDS_ZERO);       // HALF_UP, FAR_FROM_ZERO, TO_NEAR_INT
    const bool neg_up = (mode == RND_HALF_UP) || (mode == RND_HALF_TOWARDS_ZERO);
    const int up = round_half_up(v), down = round_half_down(v);
    return ((v > 0.f) ? pos_up : neg_up) ? up : down;
}

// `int o = std::round(offset)` (linear.cu:51): half away from zero, saturating.
__device__ __forceinline__ int offset_to_int(float o) { return __float2int_rz(roundf(o)); }

// ---- exact fp32 division by a (warp-)uniform divisor ------------------------------------------------------
// x / s must be the correctly rounded IEEE quotient.  div.rn.f32 costs ~30 issue slots per element on sm_90a
// (MUFU.RCP + 6 FFMA + FCHK + guarded slow-path call, measured from SASS), which would make an 8 B/element
// streaming kernel issue-bound at HBM3e speed.  The divisor is constant per tensor (or per channel row), so we
// hoist r = RN(1/s) and run Markstein's correction twice per element (1 FMUL + 4 FFMA):
//     q0 = x * r;  e0 = fma(-q0, s, x);  q1 = fma(e0, r, q0);     // q1 is a faithful quotient
//     e1 = fma(-q1, s, x);               q  = fma(e1, r, q1);     // == RN(x / s)   (Markstein's theorem)
// The theorem needs r correctly rounded (we use __frcp_rn), exact residuals (FMA) and no over/underflow of the
// intermediates.  `ok` is false when s is outside [2^-60, 2^60] (or NaN): callers then use __fdiv_rn everywhere.
// For elements whose quotient is huge, infinite or NaN the caller's range test fails and it redoes that element
// with __fdiv_rn (rare, warp-divergent only there).  Tiny quotients (|x/s| < 2^-40, where a residual could
// underflow) are harmless: everything downstream only distinguishes them from 0 through rint()/sub-normal
// rounding, both of which give 0 for any value of that magnitude.
// Out-of-line IEEE division: keeps the ~25-instruction div.rn expansion (and its slow-path call) out of the hot loops.
static __device__ __noinline__ float ieee_div_slow(float x, float s) { return __fdiv_rn(x, s); }

// max(|a|, |b|, |c|, |d|), NaN if any lane is NaN
__device__ __forceinline__ float max_abs_nan4(const float4 &q) {
    float m, n;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(m) : "f"(fabsf(q.x)), "f"(fabsf(q.y)));
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(n) : "f"(fabsf(q.z)), "f"(fabsf(q.w)));
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(m) : "f"(m), "f"(n));
    return m;
}

struct ExactDiv {
    float s, r;
    __device__ __forceinline__ ExactDiv() {}
    __device__ __forceinline__ explicit ExactDiv(float scale) { init(scale); }
    __device__ __forceinline__ void init(float scale) {
        s = scale;
        const float a = fabsf(scale);
        const bool ok = (a >= 8.6736174e-19f) && (a <= 1.1529215e18f);     // 2^-60 .. 2^60 (false for NaN)
        // A NaN reciprocal makes every fast quotient NaN, which fails the range test in div() and so routes every
        // element of a badly scaled tensor through the IEEE slow path without a second branch in the hot loop.
        r = ok ? __frcp_rn(scale) : __int_as_float(0x7FC00000);
    }
    __device__ __forceinline__ float fast(float x) const {
        const float q0 = __fmul_rn(x, r);
        const float e0 = __fmaf_rn(-q0, s, x);
        const float q1 = __fmaf_rn(e0, r, q0);
        const float e1 = __fmaf_rn(-q1, s, x);
        return __fmaf_rn(e1, r, q1);
    }
    // Exact quotient whenever |result| < limit; otherwise (huge / inf / NaN) falls back to div.rn.
    __device__ __forceinline__ float div(float x, float limit = 2147483648.f) const {
        float q = fast(x);
        if (!(fabsf(q) < limit)) q = ieee_div_slow(x, s);
        return q;
    }
    // Four quotients, one range test: the NaN-propagating maximum of the four magnitudes (three FMNMX.NAN with |.| operand
    // modifiers) fails `< limit` for huge, infinite and NaN lanes alike.
    __device__ __forceinline__ float4 div4(const float4 &x, float limit = 2147483648.f) const {
        float4 q = make_float4(fast(x.x), fast(x.y), fast(x.z), fast(x.w));
        if (!(max_abs_nan4(q) < limit)) {
            q.x = ieee_div_slow(x.x, s); q.y = ieee_div_slow(x.y, s); q.z = ieee_div_slow(x.z, s); q.w = ieee_div_slow(x.w, s);
        }
        return q;
    }
};

// Four quotients by four different divisors (channel-last layouts: neighbouring elements belong to different channels), one range test.
__device__ __forceinline__ float4 exact_div4x(const ExactDiv &a, const ExactDiv &b, const ExactDiv &c, const ExactDiv &d,
                                              const float4 &x, float limit = 2147483648.f) {
    float4 q = make_float4(a.fast(x.x), b.fast(x.y), c.fast(x.z), d.fast(x.w));
    if (!(max_abs_nan4(q) < limit)) {
        q.x = ieee_div_slow(x.x, a.s); q.y = ieee_div_slow(x.y, b.s); q.z = ieee_div_slow(x.z, c.s); q.w = ieee_div_slow(x.w, d.s);
    }
    return q;
}

// ---- streaming global memory access -----------------------------------------------------------------------
// Inputs are read exactly once: bypass L1 allocation (ld.global.nc.L1::no_allocate).  Outputs are written with
// the default policy so that they stay in the 50 MB L2 for the consumer kernel (the next operator of the graph).
__device__ __forceinline__ float4 ld_stream4(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float ld_stream1(const float *p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// ---- fast division of a 64-bit index by a runtime 32-bit constant (channel index arithmetic) ---------------
// d < 2^31.  For n < 2^63 computes floor(n / d) exactly with one 64x64->128 high multiply and a correction.
struct FastDiv {
    uint64_t magic; uint32_t d;
    __host__ __device__ FastDiv() : magic(0), d(1) {}
    __host__ explicit FastDiv(uint32_t div) : d(div) {
        magic = div <= 1 ? 0 : (~0ull) / div;                       // floor((2^64 - 1) / d)
    }
    __device__ __forceinline__ uint64_t quot(uint64_t n) const {
        if (d == 1) return n;
        uint64_t q = __umul64hi(n, magic);                          // q <= n/d, off by at most 1 (n < 2^63)
        if (n - q * d >= d) ++q;
        return q;
    }
};

// 32-bit variant for indices < 2^31 (every tensor on this path has numel <= 2^31 - 1): IMAD.HI + IMAD + compare.
struct FastDiv32 {
    uint32_t magic, d;
    __host__ __device__ FastDiv32() : magic(0), d(1) {}
    __host__ __device__ explicit FastDiv32(uint32_t div) : magic(div <= 1 ? 0u : 0xFFFFFFFFu / div), d(div) {}
    __device__ __forceinline__ uint32_t quot(uint32_t n) const {
        if (d == 1) return n;
        uint32_t q = __umulhi(n, magic);                            // floor(n/d) - 1 <= q <= floor(n/d) for n < 2^31
        if (n - q * d >= d) ++q;
        return q;
    }
};

// ---- atomics --------------------------------------------------------------------------------------------------------------
// Float atomic min/max on raw IEEE bits (works for mixed signs; see DESIGN.md "statistics arena").
// NaN is encoded by the caller: for the max slot +NaN (0x7FC00000) wins every signed-int max; for the min slot
// -NaN (0xFFC00000) wins every unsigned max among negatives and is below every positive as a signed int.
__device__ __forceinline__ void atomic_max_float(float *addr, float v) {
    if (!(__float_as_uint(v) >> 31)) atomicMax(reinterpret_cast<int *>(addr), __float_as_int(v));          // +x, +0, +NaN
    else                             atomicMin(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v)); // -x, -0
}
__device__ __forceinline__ void atomic_min_float(float *addr, float v) {
    if (!(__float_as_uint(v) >> 31)) atomicMin(reinterpret_cast<int *>(addr), __float_as_int(v));
    else                             atomicMax(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v)); // -x, -0, -NaN
}

inline int grid_for(int64_t work_items, int threads, int items_per_thread, int ctas_per_sm) {
    const int64_t per_cta = (int64_t)threads * items_per_thread;
    int64_t g = (work_items + per_cta - 1) / per_cta;
    const int64_t cap = (int64_t)sm_count() * ctas_per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace ppqb
