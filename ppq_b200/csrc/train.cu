// train.cu -- the training-pass helpers that share the scalar quantizer (sm_90a), behind the C ABI of include/ppq_b200.h.
// These are the "next" rows of the scope table (SURVEY.md §8f-2, §8f-4): callers on either side of the fake-quant path.
//
//   ppq_b200_linear_quant_t_backward / _c_backward   replace QuantizeTensor_LT_B / _LC_B (/root/reference/ppq/csrc/cuda/linear.cu:235-433)
//   ppq_b200_float_quant_t_backward  / _c_backward   replace QuantizeTensor_FT_B / _FC_B (ppq/csrc/cuda/floating.cu:133-331)
//   ppq_b200_tensor_clip_t / _c                      replace TensorClip_T / _C            (ppq/csrc/cuda/train.cu:34-113)
//   ppq_b200_rounding_loss_lt / _lc (+ _backward)    replace RoundingLoss_LT/_LC(_B)      (train.cu:115-338)
//
// Element-wise outputs (grad_x, clipped tensors, rounding-loss gradients) are bit-identical to the reference kernels.  The
// scalar reductions (grad_s, loss) are fp32 sums whose association order differs (warp shuffle tree + one atomic per CTA here,
// 1024-thread tree + atomic per block upstream -- itself launch-order dependent), so they agree to fp32 rounding only; the
// reference's own test asks for SNR <= 1e-3 / 1e-5 on them (tests/test_cuda_kernel.py:91-96, 136-141).  The normaliser is applied
// as the reference applies it -- LSQ multiplies each block sum by the host's double-precision rsqrtf, the float backward and the
// rounding loss divide each block sum by sqrtf(...) -- so a sum that is exact in fp32 gives the reference's bits.
#include "ops.cuh"
#include "../../include/ppq_b200.h"

namespace ppqb {

constexpr int kTThreads = 256;

__device__ __forceinline__ float block_sum_f(float v) {
    __shared__ float part[kTThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 32) {
        t = threadIdx.x < kTThreads / 32 ? part[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    return t;     // valid in thread 0
}

struct Channel {                       // channel of flat element i for a [outer, C, epc] tensor; C == 1 && epc == n -> per tensor
    FastDiv32 de, dc; uint32_t C;
    __device__ __forceinline__ uint32_t of(uint32_t i) const { const uint32_t row = de.quot(i); return row - dc.quot(row) * C; }
};

// ---- LSQ backward (integer) -------------------------------------------------------------------------------------------------
// linear.cu:251-275 / 343-370.  PER_CHANNEL selects the _LC_B formula, which differs in the association of (q - v), s and dy.
template <bool PER_CHANNEL>
__global__ void __launch_bounds__(kTThreads)
linear_backward_kernel(const float *__restrict__ x, const float *__restrict__ dy, uint32_t n, Channel ch,
                       const float *__restrict__ scale, const float *__restrict__ offset, int lo, int hi, int mode, float grad_factor,
                       float *__restrict__ grad_x, float *__restrict__ grad_s) {
    // one CTA handles whole rows of one channel at a time so that its partial sum belongs to a single grad_s slot
    const uint32_t epc = ch.de.d, rows = n / epc;
    for (uint32_t row = blockIdx.x; row < rows; row += gridDim.x) {
        const uint32_t c = PER_CHANNEL ? row - ch.dc.quot(row) * ch.C : 0u;
        const float s = __ldg(scale + c);
        const float o = roundf(__ldg(offset + c));                     // float o = std::round(offset)
        float part = 0.f;
        for (uint32_t j = threadIdx.x; j < epc; j += kTThreads) {
            const uint32_t i = row * epc + j;
            const float v = __ldg(x + i), g = __ldg(dy + i);
            const int qt = __float2int_rz(__fadd_rn(__int2float_rn(round2int_dyn(__fdiv_rn(v, s), mode)), o));   // int + float -> float -> int
            float gx;
            if (qt > hi)      { part = __fadd_rn(part, __fmul_rn(__fsub_rn(__int2float_rn(hi), o), g)); gx = 0.f; }
            else if (qt < lo) { part = __fadd_rn(part, __fmul_rn(__fsub_rn(__int2float_rn(lo), o), g)); gx = 0.f; }
            else {
                const float q = __fmul_rn(__int2float_rn(qt - __float2int_rz(o)), s);                              // DequantizeScalar<int,float,int>
                if (PER_CHANNEL) part = __fadd_rn(part, __fmul_rn(__fdiv_rn(__fsub_rn(q, v), s), g));              // (q - v) / s * dy
                else             part = __fadd_rn(part, __fdiv_rn(__fmul_rn(__fsub_rn(q, v), g), s));              // (q - v) * dy / s
                gx = g;
            }
            grad_x[i] = gx;
        }
        const float total = block_sum_f(part);
        if (threadIdx.x == 0) atomicAdd(grad_s + c, __fmul_rn(total, grad_factor));
    }
}

// ---- backward of the float fake-quant ----------------------------------------------------------------------------------------
// floating.cu:148-183 / 241-283: quantise with the clip range widened by one, saturated values take the clip-bound gradient.
__global__ void __launch_bounds__(kTThreads)
float_backward_kernel(const float *__restrict__ x, const float *__restrict__ dy, uint32_t n, Channel ch, bool per_channel,
                      const float *__restrict__ scale, const float *__restrict__ offset, FloatOp<-1>::Params p, float cmin, float cmax,
                      float norm, float *__restrict__ grad_x, float *__restrict__ grad_s) {
    const FloatOp<-1>::Plan plan(p);                                   // p carries clip_min - 1 / clip_max + 1
    const uint32_t epc = ch.de.d, rows = n / epc;
    for (uint32_t row = blockIdx.x; row < rows; row += gridDim.x) {
        const uint32_t c = per_channel ? row - ch.dc.quot(row) * ch.C : 0u;
        const float s = __ldg(scale + c), o = __ldg(offset + c);
        const float inv_s = __fdiv_rn(1.0f, s);
        const float bmin = __fmul_rn(s, __fsub_rn(cmin, o)), bmax = __fmul_rn(s, __fsub_rn(cmax, o));
        const FloatOp<-1> op(plan, s, o);
        float part = 0.f;
        for (uint32_t j = threadIdx.x; j < epc; j += kTThreads) {
            const uint32_t i = row * epc + j;
            const float v = __ldg(x + i), g = __ldg(dy + i);
            const float qt = op.grid(__fdiv_rn(v, s));
            const float q = op.dequant(qt);
            float gx;
            if (qt == p.cmax)      { part = __fadd_rn(part, __fmul_rn(__fmul_rn(bmax, g), inv_s)); gx = 0.f; }
            else if (qt == p.cmin) { part = __fadd_rn(part, __fmul_rn(__fmul_rn(bmin, g), inv_s)); gx = 0.f; }
            else                   { part = __fadd_rn(part, __fmul_rn(__fmul_rn(__fsub_rn(q, v), inv_s), g)); gx = g; }
            grad_x[i] = gx;
        }
        const float total = block_sum_f(part);
        if (threadIdx.x == 0) atomicAdd(grad_s + c, __fdiv_rn(total, norm));                // reduced / sqrtf(...), floating.cu:181
    }
}

// ---- TensorClip: out = CLIP(value, reference - limit[c], reference + limit[c])  (train.cu:44-48, 89-92) -----------------------------
__global__ void __launch_bounds__(kTThreads)
tensor_clip_kernel(const float *__restrict__ v, const float *__restrict__ ref, const float *__restrict__ limit, uint32_t n, Channel ch,
                   bool per_channel, float *__restrict__ out) {
    for (uint32_t i = blockIdx.x * kTThreads + threadIdx.x; i < n; i += gridDim.x * kTThreads) {
        const float l = __ldg(limit + (per_channel ? ch.of(i) : 0u));
        const float r = __ldg(ref + i), x = __ldg(v + i);
        const float lo = __fsub_rn(r, l), hi = __fadd_rn(r, l);
        out[i] = x > hi ? hi : (x < lo ? lo : x);
    }
}

// ---- RoundingLoss (train.cu:125-141, 178-191, 241-257, 299-313) ---------------------------------------------------------------------
// `int o = nearbyint(offset)` for the quantiser (half-even, unlike the fake-quant kernels), but the "was it clipped" test of the
// per-channel variants uses the UNROUNDED float offset -- both quirks kept.
__global__ void __launch_bounds__(kTThreads)
rounding_loss_kernel(const float *__restrict__ x, uint32_t n, Channel ch, bool per_channel,
                     const float *__restrict__ scale, const float *__restrict__ offset, int lo, int hi, int mode, float sqrt_n,
                     float *__restrict__ out) {
    float part = 0.f;
    for (uint32_t i = blockIdx.x * kTThreads + threadIdx.x; i < n; i += gridDim.x * kTThreads) {
        const uint32_t c = per_channel ? ch.of(i) : 0u;
        const float s = __ldg(scale + c), of = __ldg(offset + c);
        const int o = __float2int_rn(of);
        const float v = __ldg(x + i);
        int q = round2int_dyn(__fdiv_rn(v, s), mode) + o;
        q = q > hi ? hi : (q < lo ? lo : q);
        const float deq = __fmul_rn(__int2float_rn(q - o), s);
        const float up = per_channel ? __fmul_rn(s, __fsub_rn(__int2float_rn(hi), of)) : __fmul_rn(s, __int2float_rn(hi - o));
        const float dn = per_channel ? __fmul_rn(s, __fsub_rn(__int2float_rn(lo), of)) : __fmul_rn(s, __int2float_rn(lo - o));
        const bool clipped = (v > up) || (v < dn);
        part = __fadd_rn(part, clipped ? 0.f : fabsf(__fsub_rn(deq, v)));
    }
    const float total = block_sum_f(part);
    if (threadIdx.x == 0) atomicAdd(out, __fdiv_rn(total, sqrt_n));                           // diff_reduced / sqrtf(n), train.cu:140
}

// exact `grad / sqrtf(n)` for the backward variant (a division, not a multiplication by the reciprocal)
__global__ void __launch_bounds__(kTThreads)
rounding_loss_backward_kernel(const float *__restrict__ x, const float *__restrict__ dy, uint32_t n, Channel ch, bool per_channel,
                              const float *__restrict__ scale, const float *__restrict__ offset, int lo, int hi, int mode, float sqrt_n,
                              float *__restrict__ out) {
    const float g0 = __ldg(dy);
    for (uint32_t i = blockIdx.x * kTThreads + threadIdx.x; i < n; i += gridDim.x * kTThreads) {
        const uint32_t c = per_channel ? ch.of(i) : 0u;
        const float s = __ldg(scale + c), of = __ldg(offset + c);
        const int o = __float2int_rn(of);
        const float v = __ldg(x + i);
        int q = round2int_dyn(__fdiv_rn(v, s), mode) + o;
        q = q > hi ? hi : (q < lo ? lo : q);
        const float deq = __fmul_rn(__int2float_rn(q - o), s);
        const float up = per_channel ? __fmul_rn(s, __fsub_rn(__int2float_rn(hi), of)) : __fmul_rn(s, __int2float_rn(hi - o));
        const float dn = per_channel ? __fmul_rn(s, __fsub_rn(__int2float_rn(lo), of)) : __fmul_rn(s, __int2float_rn(lo - o));
        float grad = __fmul_rn(v > deq ? 1.f : -1.f, g0);
        if (v > up) grad = 0.f;
        if (v < dn) grad = 0.f;
        out[i] = __fdiv_rn(grad, sqrt_n);
    }
}

static inline Channel make_channel(int64_t n, int64_t epc, int C) {
    Channel ch;
    ch.de = FastDiv32((uint32_t)epc); ch.dc = FastDiv32((uint32_t)C); ch.C = (uint32_t)C;
    (void)n;
    return ch;
}
static inline bool geom_ok(int64_t n, int64_t epc, int C) { return n > 0 && n <= 0x7fffffffLL && epc > 0 && C > 0 && n % epc == 0; }
static inline int flat_grid(int64_t n) { int64_t g = (n + kTThreads * 8 - 1) / (kTThreads * 8); return (int)(g > sm_count() * 8 ? sm_count() * 8 : (g < 1 ? 1 : g)); }
// the host's rsqrtf (crt/math_functions.hpp): the reciprocal square root in double, rounded once to float
static inline float host_rsqrtf(float a) { return (float)(1.0 / sqrt((double)a)); }
static inline int row_grid(int64_t rows) { return (int)(rows > sm_count() * 8 ? sm_count() * 8 : rows); }

}  // namespace ppqb

using namespace ppqb;

extern "C" {

int ppq_b200_linear_quant_t_backward(const float *x, const float *dy, int64_t n, const float *scale, const float *offset,
                                     int qmin, int qmax, int rounding, float *grad_x, float *grad_s, void *stream) {
    if (!geom_ok(n, n, 1) || !x || !dy || !scale || !offset || !grad_x || !grad_s) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(grad_s, 0, sizeof(float), st);
    // per tensor: treat the tensor as rows of 8192 elements so that many CTAs share the work (any divisor keeps the sum a sum)
    int64_t epc = n;
    for (int64_t cand = 8192; cand >= 256; cand >>= 1) if (n % cand == 0) { epc = cand; break; }
    const float gf = host_rsqrtf((float)((double)n * (double)(int)((uint32_t)qmax - (uint32_t)qmin)));   // rsqrtf((double) n * (clip_max - clip_min)), linear.cu:306
    linear_backward_kernel<false><<<row_grid(n / epc), kTThreads, 0, st>>>(x, dy, (uint32_t)n, make_channel(n, epc, 1), scale, offset, qmin, qmax,
                                                                            rounding, gf, grad_x, grad_s);
    return (int)cudaGetLastError();
}

int ppq_b200_linear_quant_c_backward(const float *x, const float *dy, int64_t n, int64_t epc, int C, const float *scale, const float *offset,
                                     int qmin, int qmax, int rounding, float *grad_x, float *grad_s, void *stream) {
    if (!geom_ok(n, epc, C) || !x || !dy || !scale || !offset || !grad_x || !grad_s) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(grad_s, 0, sizeof(float) * C, st);
    const float gf = host_rsqrtf((float)((double)n * (double)qmax));                    // rsqrtf((double) n * clip_max), linear.cu:402
    linear_backward_kernel<true><<<row_grid(n / epc), kTThreads, 0, st>>>(x, dy, (uint32_t)n, make_channel(n, epc, C), scale, offset, qmin, qmax,
                                                                           rounding, gf, grad_x, grad_s);
    return (int)cudaGetLastError();
}

static bool fp_format_ok(int E, int M) {
    if (E < 1 || E > 5 || M < 0 || M > 22) return false;
    const int k = (1 << (E - 1)) + M - 2;
    return k >= 0 && k <= 30;
}

int ppq_b200_float_quant_t_backward(const float *x, const float *dy, int64_t n, const float *scale, const float *offset, int exponent,
                                    int mantissa, float clip_min, float clip_max, int rounding, float *grad_x, float *grad_s, void *stream) {
    if (!geom_ok(n, n, 1) || !fp_format_ok(exponent, mantissa) || !x || !dy || !scale || !offset || !grad_x || !grad_s) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(grad_s, 0, sizeof(float), st);
    int64_t epc = n;
    for (int64_t cand = 8192; cand >= 256; cand >>= 1) if (n % cand == 0) { epc = cand; break; }
    const float norm = sqrtf((float)n * clip_max);                                         // sqrtf((float)(num_of_elements * clip_max)), floating.cu:181
    float_backward_kernel<<<row_grid(n / epc), kTThreads, 0, st>>>(x, dy, (uint32_t)n, make_channel(n, epc, 1), false, scale, offset,
                                                                    {exponent, mantissa, rounding, clip_min - 1, clip_max + 1}, clip_min, clip_max,
                                                                    norm, grad_x, grad_s);
    return (int)cudaGetLastError();
}

int ppq_b200_float_quant_c_backward(const float *x, const float *dy, int64_t n, int64_t epc, int C, const float *scale, const float *offset,
                                    int exponent, int mantissa, float clip_min, float clip_max, int rounding, float *grad_x, float *grad_s,
                                    void *stream) {
    if (!geom_ok(n, epc, C) || !fp_format_ok(exponent, mantissa) || !x || !dy || !scale || !offset || !grad_x || !grad_s) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(grad_s, 0, sizeof(float) * C, st);
    const float norm = sqrtf((float)n * clip_max);
    float_backward_kernel<<<row_grid(n / epc), kTThreads, 0, st>>>(x, dy, (uint32_t)n, make_channel(n, epc, C), true, scale, offset,
                                                                    {exponent, mantissa, rounding, clip_min - 1, clip_max + 1}, clip_min, clip_max,
                                                                    norm, grad_x, grad_s);
    return (int)cudaGetLastError();
}

int ppq_b200_tensor_clip_t(const float *value, const float *reference, const float *limit, int64_t n, float *out, void *stream) {
    if (!geom_ok(n, n, 1) || !value || !reference || !limit || !out) return (int)cudaErrorInvalidValue;
    tensor_clip_kernel<<<flat_grid(n), kTThreads, 0, (cudaStream_t)stream>>>(value, reference, limit, (uint32_t)n, make_channel(n, n, 1), false, out);
    return (int)cudaGetLastError();
}

int ppq_b200_tensor_clip_c(const float *value, const float *reference, const float *limit, int64_t n, int64_t epc, int C, float *out, void *stream) {
    if (!geom_ok(n, epc, C) || !value || !reference || !limit || !out) return (int)cudaErrorInvalidValue;
    tensor_clip_kernel<<<flat_grid(n), kTThreads, 0, (cudaStream_t)stream>>>(value, reference, limit, (uint32_t)n, make_channel(n, epc, C), true, out);
    return (int)cudaGetLastError();
}

int ppq_b200_rounding_loss(const float *x, int64_t n, int64_t epc, int C, int per_channel, const float *scale, const float *offset,
                           int qmin, int qmax, int rounding, float *loss, void *stream) {
    if (!geom_ok(n, epc, C) || !x || !scale || !offset || !loss) return (int)cudaErrorInvalidValue;
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(loss, 0, sizeof(float), st);
    rounding_loss_kernel<<<flat_grid(n), kTThreads, 0, st>>>(x, (uint32_t)n, make_channel(n, epc, C), per_channel != 0, scale, offset,
                                                                   qmin, qmax, rounding, sqrtf((float)n), loss);
    return (int)cudaGetLastError();
}

int ppq_b200_rounding_loss_backward(const float *x, const float *dy, int64_t n, int64_t epc, int C, int per_channel, const float *scale,
                                    const float *offset, int qmin, int qmax, int rounding, float *grad_x, void *stream) {
    if (!geom_ok(n, epc, C) || !x || !dy || !scale || !offset || !grad_x) return (int)cudaErrorInvalidValue;
    rounding_loss_backward_kernel<<<flat_grid(n), kTThreads, 0, (cudaStream_t)stream>>>(x, dy, (uint32_t)n, make_channel(n, epc, C), per_channel != 0,
                                                                                        scale, offset, qmin, qmax, rounding, sqrtf((float)n), grad_x);
    return (int)cudaGetLastError();
}

}  // extern "C"
