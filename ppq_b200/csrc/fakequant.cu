// fakequant.cu -- sm_90a fake-quant kernels (quantize -> clamp -> dequantize) behind the C ABI of include/ppq_b200.h.
//
//   ppq_b200_linear_quant_t / _c   replace QuantizeTensor_LT / _LC  (/root/reference/ppq/csrc/cuda/linear.cu:38-233)
//   ppq_b200_float_quant_t  / _c   replace QuantizeTensor_FT / _FC  (ppq/csrc/cuda/floating.cu:36-131, common.cuh:154-226)
//   ppq_b200_linear_quant_*_toint  device twin of PPQLinearQuant_toInt (ppq/quantization/qfunction/linear.py:218-238)
//
// Design (DESIGN.md §kernels): pure streaming kernels, 8 B/element of algorithmic HBM traffic (4 read + 4 write),
// no reuse -> no shared-memory staging in the default variant.  Each thread keeps 4 independent 128-bit loads in flight
// (64 B), 256 threads per CTA, persistent grid of (SM count) x 8 CTAs, grid-stride over float4 vectors, so ~128 KB are in
// flight per SM -- enough to cover HBM3e latency x bandwidth.  The arithmetic per element is kept under ~15 issue slots
// (hoisted exact reciprocal + 2 Markstein corrections instead of div.rn, see common.cuh) so the kernel stays
// bandwidth-bound rather than issue-bound.  Variant 1 (ppq_b200_set_variant("linear_quant_t", 1)) is the
// TMA-staged pipeline (cp.async.bulk global->shared ring with mbarriers, bulk store back) kept for comparison.
#include "ops.cuh"
#include "../../include/ppq_b200.h"
#include "variants.h"
#include <string.h>

namespace ppqb {

// ---- output writers ------------------------------------------------------------------------------------------------
template <class Op, class OutT> struct Emit;
template <class Op> struct Emit<Op, float> {
    static __device__ __forceinline__ float one(const Op &op, float x) { return op.apply(x); }
    static __device__ __forceinline__ void store4(float *y, int64_t vi, float a, float b, float c, float d) {
        reinterpret_cast<float4 *>(y)[vi] = make_float4(a, b, c, d);
    }
    static __device__ __forceinline__ void vec(const Op &op, const float4 &v, float *y, int64_t vi) {
        reinterpret_cast<float4 *>(y)[vi] = op.apply4(v);
    }
    static __device__ __forceinline__ void vecx(const Op (&ops)[4], const float4 &v, float *y, int64_t vi) {
        reinterpret_cast<float4 *>(y)[vi] = Op::apply4x(ops, v);
    }
};
template <class Op> struct Emit<Op, int32_t> {
    static __device__ __forceinline__ int32_t one(const Op &op, float x) { return op.quant(x); }
    static __device__ __forceinline__ void store4(int32_t *y, int64_t vi, int32_t a, int32_t b, int32_t c, int32_t d) {
        reinterpret_cast<int4 *>(y)[vi] = make_int4(a, b, c, d);
    }
    static __device__ __forceinline__ void vec(const Op &op, const float4 &v, int32_t *y, int64_t vi) {
        reinterpret_cast<int4 *>(y)[vi] = op.quant4(v);
    }
    static __device__ __forceinline__ void vecx(const Op (&ops)[4], const float4 &v, int32_t *y, int64_t vi) {
        reinterpret_cast<int4 *>(y)[vi] = Op::quant4x(ops, v);
    }
};
template <class Op> struct Emit<Op, int8_t> {       // also used for uint8 (same low byte)
    static __device__ __forceinline__ int8_t one(const Op &op, float x) { return (int8_t)op.quant(x); }
    static __device__ __forceinline__ void store4(int8_t *y, int64_t vi, int8_t a, int8_t b, int8_t c, int8_t d) {
        reinterpret_cast<uint32_t *>(y)[vi] = ((uint32_t)(uint8_t)a) | ((uint32_t)(uint8_t)b << 8) | ((uint32_t)(uint8_t)c << 16) | ((uint32_t)(uint8_t)d << 24);
    }
    static __device__ __forceinline__ void vec(const Op &op, const float4 &v, int8_t *y, int64_t vi) {
        const int4 q = op.quant4(v);
        reinterpret_cast<uint32_t *>(y)[vi] = ((uint32_t)q.x & 0xFFu) | (((uint32_t)q.y & 0xFFu) << 8) |
                                              (((uint32_t)q.z & 0xFFu) << 16) | (((uint32_t)q.w & 0xFFu) << 24);
    }
    static __device__ __forceinline__ void vecx(const Op (&ops)[4], const float4 &v, int8_t *y, int64_t vi) {
        const int4 q = Op::quant4x(ops, v);
        reinterpret_cast<uint32_t *>(y)[vi] = ((uint32_t)q.x & 0xFFu) | (((uint32_t)q.y & 0xFFu) << 8) |
                                              (((uint32_t)q.z & 0xFFu) << 16) | (((uint32_t)q.w & 0xFFu) << 24);
    }
};

constexpr int kThreads = 256;
constexpr int kUnroll = 4;          // independent 128-bit loads in flight per thread

// ---- per-tensor: one (scale, offset) for the whole tensor ---------------------------------------------------------------
// VEC: x and y are 16-byte aligned -> float4 main loop + scalar tail; otherwise everything scalar.
// Every round issues kUnroll predicated 128-bit loads before the first use, also in the ragged last round.
template <class Op, class OutT, bool VEC, int U = kUnroll, int TPB = kThreads, int MINB = 1>
__global__ void __launch_bounds__(TPB, MINB)
ew_tensor_kernel(const float *__restrict__ x, OutT *__restrict__ y, int64_t n,
                 const float *__restrict__ scale, const float *__restrict__ offset, typename Op::Params p) {
    const typename Op::Plan plan(p);
    const Op op(plan, __ldg(scale), __ldg(offset));
    const int64_t tid = (int64_t)blockIdx.x * TPB + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * TPB;
    if constexpr (VEC) {
        const int64_t n4 = n >> 2;
        const float4 *x4 = reinterpret_cast<const float4 *>(x);
        // Each warp walks contiguous segments of 32 x U vectors (lane-interleaved): the U loads of a thread hit one 2 KB span of
        // HBM instead of U pages a grid-stride apart (measured +4 points of HBM peak on the per-channel twin of this loop).
        constexpr int64_t kSeg = 32 * U;
        const int64_t lane = threadIdx.x & 31;
        const int64_t warp = tid >> 5, warps = stride >> 5;
        const int64_t segs = (n4 + kSeg - 1) / kSeg;
        for (int64_t sg = warp; sg < segs; sg += warps) {
            const int64_t base = sg * kSeg + lane;
            float4 v[U];
#pragma unroll
            for (int j = 0; j < U; j++) if (base + j * 32 < n4) v[j] = ld_stream4(x4 + base + j * 32);
#pragma unroll
            for (int j = 0; j < U; j++) if (base + j * 32 < n4) Emit<Op, OutT>::vec(op, v[j], y, base + j * 32);
        }
        const int64_t t = (n4 << 2) + tid;                          // <= 3 leftover elements
        if (t < n) y[t] = Emit<Op, OutT>::one(op, x[t]);
    } else {
        for (int64_t i = tid; i < n; i += stride) y[i] = Emit<Op, OutT>::one(op, x[i]);
    }
}

// ---- per-channel, vectorised: epc % 4 == 0 and 16-byte aligned bases, so a float4 never straddles a channel row ----------
// Flat grid-stride over float4 vectors exactly like the per-tensor kernel (same memory-level parallelism); the channel of
// vector vi is (vi / (epc/4)) % C, from two 32-bit multiply-high divisions (numel < 2^31 is part of the contract), and the
// operator (exact reciprocal, integer offset) is rebuilt per vector.
template <class Op, class OutT>
__device__ __forceinline__ void channel_vec_body(const float *__restrict__ x, OutT *__restrict__ y, uint32_t n4, int C,
                                                 const FastDiv32 &div_epc4, const FastDiv32 &div_C,
                                                 const float *__restrict__ scale, const float *__restrict__ offset,
                                                 const typename Op::Plan &plan, uint32_t first, uint32_t stride) {
    const float4 *x4 = reinterpret_cast<const float4 *>(x);
    for (uint64_t i = first; i < n4; i += (uint64_t)kUnroll * stride) {
        float4 v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; j++) if (i + (uint64_t)j * stride < n4) v[j] = ld_stream4(x4 + i + (uint64_t)j * stride);
#pragma unroll
        for (int j = 0; j < kUnroll; j++) {
            const uint64_t vi = i + (uint64_t)j * stride;
            if (vi < n4) {
                const uint32_t row = div_epc4.quot((uint32_t)vi);
                const uint32_t c = row - div_C.quot(row) * (uint32_t)C;
                const Op op(plan, __ldg(scale + c), __ldg(offset + c));
                Emit<Op, OutT>::vec(op, v[j], y, (int64_t)vi);
            }
        }
    }
}

// Long rows (epc/4 >= 128): each warp walks contiguous 128-vector segments (lane-interleaved, 4 x 128-bit loads in flight per lane).
// A segment touches at most two channel rows, so the operator is built once (twice when the segment straddles a row end, a
// warp-uniform branch) per 16 elements of a thread instead of once per vector.
template <class Op, class OutT>
__global__ void __launch_bounds__(kThreads)
ew_channel_seg_kernel(const float *__restrict__ x, OutT *__restrict__ y, uint32_t n4, int C, uint32_t epc4,
                      FastDiv32 div_epc4, FastDiv32 div_C,
                      const float *__restrict__ scale, const float *__restrict__ offset, typename Op::Params p) {
    const typename Op::Plan plan(p);
    const float4 *x4 = reinterpret_cast<const float4 *>(x);
    constexpr uint32_t kSeg = 32 * kUnroll;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (kThreads / 32);
    const uint32_t segs = (n4 + kSeg - 1) / kSeg;
    for (uint32_t sg = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); sg < segs; sg += warps) {
        const uint32_t base = sg * kSeg;
        float4 v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; j++) if (base + j * 32 + lane < n4) v[j] = ld_stream4(x4 + base + j * 32 + lane);
        const uint32_t r0 = div_epc4.quot(base);
        const uint32_t c0 = r0 - div_C.quot(r0) * (uint32_t)C;
        const uint32_t next_row = (r0 + 1) * epc4;                   // first vector of the following row (no overflow: n4 < 2^29)
        const Op op0(plan, __ldg(scale + c0), __ldg(offset + c0));
        if (next_row >= base + kSeg) {                               // whole segment in one row (warp-uniform)
#pragma unroll
            for (int j = 0; j < kUnroll; j++) if (base + j * 32 + lane < n4) Emit<Op, OutT>::vec(op0, v[j], y, (int64_t)(base + j * 32 + lane));
        } else {
            const uint32_t c1 = (c0 + 1 == (uint32_t)C) ? 0u : c0 + 1;
            const Op op1(plan, __ldg(scale + c1), __ldg(offset + c1));
#pragma unroll
            for (int j = 0; j < kUnroll; j++) {
                const uint32_t vi = base + j * 32 + lane;
                if (vi < n4) { if (vi < next_row) Emit<Op, OutT>::vec(op0, v[j], y, (int64_t)vi); else Emit<Op, OutT>::vec(op1, v[j], y, (int64_t)vi); }
            }
        }
    }
}

template <class Op, class OutT>
__global__ void __launch_bounds__(kThreads)
ew_channel_vec_kernel(const float *__restrict__ x, OutT *__restrict__ y, uint32_t n4, int C,
                      FastDiv32 div_epc4, FastDiv32 div_C,
                      const float *__restrict__ scale, const float *__restrict__ offset, typename Op::Params p) {
    const typename Op::Plan plan(p);
    channel_vec_body<Op, OutT>(x, y, n4, C, div_epc4, div_C, scale, offset, plan, blockIdx.x * kThreads + threadIdx.x, gridDim.x * kThreads);
}

// ---- per-channel, short rows (4 <= epc < 512): per-row operators from a shared-memory table -------------------------------------------
// A CTA walks contiguous tiles of 1024 vectors (16 KB; tiles round-robin over the grid, inside a tile every warp owns a contiguous 2 KB
// segment, 4 x 128-bit loads in flight per lane).  The rows a tile touches are known from two divisions per TILE; their operators -- exact
// reciprocal with its range check, integer offset -- are built ONCE per row by the first threads of the CTA into a 16-byte-per-row table
// while the tile's loads are in flight, so an element pays one table read per vector (VEC4: rows are a multiple of 4 elements, a vector
// never straddles a row) or per element (any epc >= 4: the walker steps to the next entry at a row end) instead of two multiply-high
// divisions, two global loads, a reciprocal and a float->int conversion per vector.
constexpr int kTileVec = kThreads * kUnroll;                            // 1024 vectors = 4096 elements
constexpr int kTabRows = 4 * kTileVec / 4 + 2;                          // rows a tile can touch when epc >= 4
template <class Op, class OutT, bool VEC4>
__global__ void __launch_bounds__(kThreads)
ew_channel_table_kernel(const float *__restrict__ x, OutT *__restrict__ y, uint32_t n, uint32_t epc, int C, FastDiv32 div_epc, FastDiv32 div_C,
                        const float *__restrict__ scale, const float *__restrict__ offset, typename Op::Params p) {
    // Two tables: tile t builds into tab[t & 1] and needs ONE barrier (after the build).  Every warp passes the barrier of tile t + 1 only after its
    // own apply stage of tile t, so when a table is rebuilt (tile t + 2) nobody reads it any more -- and a warp that runs ahead has already issued
    // the loads of the next tile when it waits at that barrier, so the memory pipe of the CTA never drains at a tile boundary.
    __shared__ float4 tab[2][kTabRows];
    const typename Op::Plan plan(p);
    const float4 *x4 = reinterpret_cast<const float4 *>(x);
    const uint32_t groups = (n + 3u) >> 2;                              // VEC4: n % 4 == 0
    const uint32_t n4 = n >> 2;                                         // whole vectors
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t which = 0;
    for (uint32_t base = blockIdx.x * (uint32_t)kTileVec; base < groups; base += gridDim.x * (uint32_t)kTileVec, which ^= 1u) {
        float4 *t = tab[which];
        const uint32_t v0 = base + warp * (32 * kUnroll) + lane;
        float4 v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; j++) if (v0 + j * 32 < n4) v[j] = ld_stream4(x4 + v0 + j * 32);
        const uint32_t e_first = base << 2;
        const uint32_t e_last = min(n, (base + (uint32_t)kTileVec) << 2) - 1u;
        const uint32_t r0 = div_epc.quot(e_first), rows = div_epc.quot(e_last) - r0 + 1u;
        for (uint32_t i = threadIdx.x; i < rows; i += kThreads) {
            const uint32_t row = r0 + i, c = row - div_C.quot(row) * (uint32_t)C;
            t[i] = Op::entry(__ldg(scale + c), __ldg(offset + c));
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kUnroll; j++) {
            const uint32_t vi = v0 + j * 32;
            if (vi >= groups) continue;
            const uint32_t e0 = vi << 2;
            const uint32_t row = div_epc.quot(e0);
            if constexpr (VEC4) {
                const Op op(plan, t[row - r0]);
                Emit<Op, OutT>::vec(op, v[j], y, (int64_t)vi);
            } else {
                uint32_t col = e0 - row * epc, idx = row - r0;
                if (vi < n4) {
                    // epc >= 4: the four elements of a vector lie in at most two rows.  Both table entries are read, every lane picks its row with
                    // a select, and the four quotients share one range test (the 4-operator form of the channel-last kernel) -- no branch per element.
                    const uint32_t left = epc - col;                    // elements of the vector that still belong to row `idx` (>= 1)
                    const float4 E0 = t[idx], E1 = t[min(idx + 1u, rows - 1u)];
                    const Op ops[4] = {Op(plan, E0), Op(plan, left > 1u ? E0 : E1), Op(plan, left > 2u ? E0 : E1), Op(plan, left > 3u ? E0 : E1)};
                    Emit<Op, OutT>::vecx(ops, v[j], y, (int64_t)vi);
                } else {                                                // the <= 3 elements after the last whole vector
                    Op op(plan, t[idx]);
                    for (uint32_t e = e0; e < n; e++) {
                        y[e] = Emit<Op, OutT>::one(op, ld_stream1(x + e));
                        if (++col == epc) { col = 0; ++idx; if (e + 1 < n) op.rebind(t[idx]); }
                    }
                }
            }
        }
    }
}

// ---- per-channel, channel-last (epc == 1, C % 4 == 0): x is [rows, C], element (r, c) belongs to channel c ---------------------
// The grid-stride is rounded down to a multiple of C/4, so every thread keeps meeting the same four channels: their operators
// (exact reciprocals, integer offsets) are built once per thread and the loop body costs what the per-tensor kernel costs.
template <class Op, class OutT>
__global__ void __launch_bounds__(kThreads)
ew_channel_last_kernel(const float *__restrict__ x, OutT *__restrict__ y, int64_t n4, uint32_t C4, uint32_t active,
                       const float *__restrict__ scale, const float *__restrict__ offset, typename Op::Params p) {
    const typename Op::Plan plan(p);
    const uint32_t tid = blockIdx.x * kThreads + threadIdx.x;
    if (tid >= active) return;
    const uint32_t c = (tid % C4) * 4;
    const Op ops[4] = {Op(plan, __ldg(scale + c), __ldg(offset + c)), Op(plan, __ldg(scale + c + 1), __ldg(offset + c + 1)),
                       Op(plan, __ldg(scale + c + 2), __ldg(offset + c + 2)), Op(plan, __ldg(scale + c + 3), __ldg(offset + c + 3))};
    const float4 *x4 = reinterpret_cast<const float4 *>(x);
    for (int64_t base = tid; base < n4; base += (int64_t)active * kUnroll) {
        float4 v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; j++) if (base + (int64_t)j * active < n4) v[j] = ld_stream4(x4 + base + (int64_t)j * active);
#pragma unroll
        for (int j = 0; j < kUnroll; j++) if (base + (int64_t)j * active < n4) Emit<Op, OutT>::vecx(ops, v[j], y, base + (int64_t)j * active);
    }
}

// ---- per-channel, generic: any epc (1, 9, 27, ...), any alignment ---------------------------------------------------------
// Each thread owns 4 consecutive elements; (row, col) of the first comes from one fast division, the rest by walking.
template <class Op, class OutT>
__device__ __forceinline__ void channel_generic_body(const float *__restrict__ x, OutT *__restrict__ y, int64_t n, int64_t epc, int C,
                                                     const FastDiv &div_epc, const FastDiv &div_C,
                                                     const float *__restrict__ scale, const float *__restrict__ offset,
                                                     const typename Op::Plan &plan, int64_t first, int64_t stride) {
    const int64_t groups = (n + 3) >> 2;
    // 16-byte aligned bases: one 128-bit load / store per group even though the four elements may belong to different channels
    // (four scalar no-allocate loads of the same 128-byte line would fetch it from L2 four times)
    const bool al = ((reinterpret_cast<uintptr_t>(x) & 15u) == 0) && ((reinterpret_cast<uintptr_t>(y) & (4 * sizeof(OutT) - 1)) == 0);
    for (int64_t g = first; g < groups; g += stride) {
        const int64_t e0 = g << 2;
        int64_t row = (int64_t)div_epc.quot((uint64_t)e0);
        int64_t col = e0 - row * epc;
        int c = (int)(row - (int64_t)div_C.quot((uint64_t)row) * C);
        const int cnt = (int)((n - e0) < 4 ? (n - e0) : 4);
        if (al && cnt == 4) {
            const float4 v = ld_stream4(reinterpret_cast<const float4 *>(x) + g);
            const float in[4] = {v.x, v.y, v.z, v.w};
            OutT out[4];
            Op op(plan, __ldg(scale + c), __ldg(offset + c));
#pragma unroll
            for (int j = 0; j < 4; j++) {
                out[j] = Emit<Op, OutT>::one(op, in[j]);
                if (++col == epc) {                                  // next element starts a new channel row
                    col = 0; if (++c == C) c = 0;
                    if (j < 3) op.rebind(__ldg(scale + c), __ldg(offset + c));
                }
            }
            Emit<Op, OutT>::store4(y, g, out[0], out[1], out[2], out[3]);
        } else if (col + cnt <= epc) {                               // all in one row: one operator for the group
            const Op op(plan, __ldg(scale + c), __ldg(offset + c));
            for (int j = 0; j < cnt; j++) y[e0 + j] = Emit<Op, OutT>::one(op, ld_stream1(x + e0 + j));
        } else {
            for (int j = 0; j < cnt; j++) {
                const Op op(plan, __ldg(scale + c), __ldg(offset + c));
                y[e0 + j] = Emit<Op, OutT>::one(op, ld_stream1(x + e0 + j));
                if (++col == epc) { col = 0; if (++c == C) c = 0; }
            }
        }
    }
}

template <class Op, class OutT>
__global__ void __launch_bounds__(kThreads)
ew_channel_generic_kernel(const float *__restrict__ x, OutT *__restrict__ y, int64_t n, int64_t epc, int C,
                          FastDiv div_epc, FastDiv div_C,
                          const float *__restrict__ scale, const float *__restrict__ offset, typename Op::Params p) {
    const typename Op::Plan plan(p);
    channel_generic_body<Op, OutT>(x, y, n, epc, C, div_epc, div_C, scale, offset, plan,
                                   (int64_t)blockIdx.x * kThreads + threadIdx.x, (int64_t)gridDim.x * kThreads);
}

// ---- multi-tensor per-channel fake-quant: every Conv/Gemm weight of a network in ONE launch ------------------------------------
// The tensors are cut into warp segments of 128 vectors (512 elements); the concatenation of all segments is split evenly over the
// CTAs (the per-tensor segment counts are prefix-summed in shared memory by every CTA, so no host-side table is needed and no CTA
// visits an empty work item).  Inside a span the 8 warps of a CTA take segments round-robin.  A segment of a tensor with rows of
// >= 128 vectors lies in one channel row (or straddles one row end): the operator -- exact reciprocal, integer offset -- is built
// once per 16 elements of a thread.  Shorter rows build one operator per vector; rows that are not a multiple of 4 elements, or
// unaligned tensors, walk (row, col) element by element but still move 128 bits per access when the bases allow it.
constexpr int kSegVec = 32 * kUnroll;
constexpr int kMaxMultiTensors = 4096;              // (count + 1) x 8 bytes of shared memory
template <class Op>
__global__ void __launch_bounds__(kThreads)
multi_channel_kernel(const ppq_b200_lc_desc *__restrict__ descs, int count, typename Op::Params p) {
    extern __shared__ long long seg_prefix[];                          // [count + 1], in segments
    for (int t = threadIdx.x; t < count; t += kThreads) {
        const int64_t n = descs[t].n;
        seg_prefix[t + 1] = n > 0 ? (n + 4 * kSegVec - 1) / (4 * kSegVec) : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long run = 0; seg_prefix[0] = 0;
        for (int t = 1; t <= count; t++) { run += seg_prefix[t]; seg_prefix[t] = run; }
    }
    __syncthreads();
    const int64_t total = seg_prefix[count];
    const int64_t span = (total + gridDim.x - 1) / gridDim.x;
    const int64_t s0 = (int64_t)blockIdx.x * span, s1 = (s0 + span) < total ? (s0 + span) : total;
    if (s0 >= total) return;
    int t;
    { int lo = 0, hi = count - 1; while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (seg_prefix[mid] <= s0) lo = mid; else hi = mid - 1; } t = lo; }
    const typename Op::Plan plan(p);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (; t < count && seg_prefix[t] < s1; t++) {
        const int64_t first = seg_prefix[t], segs = seg_prefix[t + 1] - first;
        if (segs == 0) continue;
        const ppq_b200_lc_desc d = descs[t];
        const uint32_t a = (uint32_t)(s0 > first ? s0 - first : 0), b = (uint32_t)((s1 - first) < segs ? (s1 - first) : segs);
        const bool al = ((reinterpret_cast<uintptr_t>(d.x) | reinterpret_cast<uintptr_t>(d.y)) & 15u) == 0;
        const float4 *x4 = reinterpret_cast<const float4 *>(d.x);
        if (al && d.epc % 4 == 0) {
            const uint32_t n4 = (uint32_t)(d.n >> 2), epc4 = (uint32_t)(d.epc >> 2);
            const FastDiv32 de(epc4), dc((uint32_t)d.C);
            for (uint32_t sg = a + warp; sg < b; sg += kThreads / 32) {
                const uint32_t base = sg * kSegVec;
                float4 v[kUnroll];
#pragma unroll
                for (int j = 0; j < kUnroll; j++) if (base + j * 32 + lane < n4) v[j] = ld_stream4(x4 + base + j * 32 + lane);
                const uint32_t r0 = de.quot(base);
                const uint32_t c0 = r0 - dc.quot(r0) * (uint32_t)d.C;
                if ((r0 + 1) * epc4 >= base + kSegVec) {                 // whole segment inside one channel row (warp-uniform)
                    const Op op(plan, __ldg(d.scale + c0), __ldg(d.offset + c0));
#pragma unroll
                    for (int j = 0; j < kUnroll; j++) if (base + j * 32 + lane < n4) Emit<Op, float>::vec(op, v[j], d.y, (int64_t)(base + j * 32 + lane));
                } else {
#pragma unroll
                    for (int j = 0; j < kUnroll; j++) {
                        const uint32_t vi = base + j * 32 + lane;
                        if (vi < n4) {
                            const uint32_t row = de.quot(vi);
                            const uint32_t c = row - dc.quot(row) * (uint32_t)d.C;
                            const Op op(plan, __ldg(d.scale + c), __ldg(d.offset + c));
                            Emit<Op, float>::vec(op, v[j], d.y, (int64_t)vi);
                        }
                    }
                }
            }
        } else {
            const uint32_t n = (uint32_t)d.n, epc = (uint32_t)d.epc;
            const FastDiv32 de(epc), dc((uint32_t)d.C);
            for (uint32_t sg = a + warp; sg < b; sg += kThreads / 32) {
                const uint32_t base = sg * kSegVec;
                float4 v[kUnroll];
                if (al) {
#pragma unroll
                    for (int j = 0; j < kUnroll; j++) if ((uint64_t)(base + j * 32 + lane) * 4 + 4 <= n) v[j] = ld_stream4(x4 + base + j * 32 + lane);
                }
#pragma unroll
                for (int j = 0; j < kUnroll; j++) {
                    const uint32_t g = base + j * 32 + lane;
                    const uint64_t e0 = (uint64_t)g * 4;
                    if (e0 >= n) continue;
                    const uint32_t row = de.quot((uint32_t)e0);
                    uint32_t col = (uint32_t)e0 - row * epc;
                    uint32_t c = row - dc.quot(row) * (uint32_t)d.C;
                    Op op(plan, __ldg(d.scale + c), __ldg(d.offset + c));
                    if (al && e0 + 4 <= n) {
                        const float in[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
                        float out[4];
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            out[k] = op.apply(in[k]);
                            if (++col == epc) { col = 0; if (++c == (uint32_t)d.C) c = 0; if (k < 3) op.rebind(__ldg(d.scale + c), __ldg(d.offset + c)); }
                        }
                        reinterpret_cast<float4 *>(d.y)[g] = make_float4(out[0], out[1], out[2], out[3]);
                    } else {
                        const int cnt = (int)((n - e0) < 4 ? (n - e0) : 4);
                        for (int k = 0; k < cnt; k++) {
                            d.y[e0 + k] = op.apply(ld_stream1(d.x + e0 + k));
                            if (++col == epc) { col = 0; if (++c == (uint32_t)d.C) c = 0; op.rebind(__ldg(d.scale + c), __ldg(d.offset + c)); }
                        }
                    }
                }
            }
        }
    }
}

// ---- multi-tensor per-tensor fake-quant: the activation tensors of a quantised graph in ONE launch -----------------------------------------
// Same partition as multi_channel_kernel (512-element warp segments, the concatenation of all segments split evenly over the CTAs), but one
// operator per tensor: it is built once per (CTA, tensor) visit and the loop body is the per-tensor kernel's.
template <class Op>
__global__ void __launch_bounds__(kThreads)
multi_tensor_kernel(const ppq_b200_lt_desc *__restrict__ descs, int count, typename Op::Params p) {
    extern __shared__ long long seg_prefix[];                          // [count + 1], in segments
    for (int t = threadIdx.x; t < count; t += kThreads) {
        const int64_t n = descs[t].n;
        seg_prefix[t + 1] = n > 0 ? (n + 4 * kSegVec - 1) / (4 * kSegVec) : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long run = 0; seg_prefix[0] = 0;
        for (int t = 1; t <= count; t++) { run += seg_prefix[t]; seg_prefix[t] = run; }
    }
    __syncthreads();
    const int64_t total = seg_prefix[count];
    const int64_t span = (total + gridDim.x - 1) / gridDim.x;
    const int64_t s0 = (int64_t)blockIdx.x * span, s1 = (s0 + span) < total ? (s0 + span) : total;
    if (s0 >= total) return;
    int t;
    { int lo = 0, hi = count - 1; while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (seg_prefix[mid] <= s0) lo = mid; else hi = mid - 1; } t = lo; }
    const typename Op::Plan plan(p);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (; t < count && seg_prefix[t] < s1; t++) {
        const int64_t first = seg_prefix[t], segs = seg_prefix[t + 1] - first;
        if (segs == 0) continue;
        const ppq_b200_lt_desc d = descs[t];
        const uint32_t a = (uint32_t)(s0 > first ? s0 - first : 0), b = (uint32_t)((s1 - first) < segs ? (s1 - first) : segs);
        const Op op(plan, __ldg(d.scale), __ldg(d.offset));
        const uint32_t n = (uint32_t)d.n;
        if (((reinterpret_cast<uintptr_t>(d.x) | reinterpret_cast<uintptr_t>(d.y)) & 15u) == 0) {
            const uint32_t n4 = n >> 2;
            const float4 *x4 = reinterpret_cast<const float4 *>(d.x);
            for (uint32_t sg = a + warp; sg < b; sg += kThreads / 32) {
                const uint32_t base = sg * kSegVec + lane;
                float4 v[kUnroll];
#pragma unroll
                for (int j = 0; j < kUnroll; j++) if (base + j * 32 < n4) v[j] = ld_stream4(x4 + base + j * 32);
#pragma unroll
                for (int j = 0; j < kUnroll; j++) if (base + j * 32 < n4) Emit<Op, float>::vec(op, v[j], d.y, (int64_t)(base + j * 32));
                if (sg == (uint32_t)segs - 1) {                          // <= 3 elements after the last whole vector
                    const uint32_t e = (n4 << 2) + lane;
                    if (e < n) d.y[e] = op.apply(ld_stream1(d.x + e));
                }
            }
        } else {
            for (uint32_t sg = a + warp; sg < b; sg += kThreads / 32) {
                const uint32_t e0 = sg * (4 * kSegVec);
                for (uint32_t e = e0 + lane; e < min(n, e0 + 4 * kSegVec); e += 32) d.y[e] = op.apply(ld_stream1(d.x + e));
            }
        }
    }
}

// ---- host-side launch helpers --------------------------------------------------------------------------------------------
static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
template <class OutT> static inline bool out_aligned(const void *p) {
    return (reinterpret_cast<uintptr_t>(p) & (4 * sizeof(OutT) - 1)) == 0;
}

template <class Op, class OutT>
static int launch_tensor(const float *x, OutT *y, int64_t n, const float *scale, const float *offset,
                         typename Op::Params p, cudaStream_t st) {
    if (n <= 0 || !x || !y || !scale || !offset) return (int)cudaErrorInvalidValue;
    const bool vec = aligned16(x) && out_aligned<OutT>(y);
    if (vec && Op::kLight && sizeof(OutT) == 4 && n >= (int64_t)1 << 25) {
        // >= 32 M elements: 8 loads in flight per thread (4 KB contiguous per warp) measured 92 % vs 89 % of HBM peak; below that the
        // coarser work granularity costs more in the tail than the extra memory-level parallelism gains (82 % vs 71 % at 8 M elements)
        ew_tensor_kernel<Op, OutT, true, 8><<<grid_for((n + 3) / 4, kThreads, 8, 16), kThreads, 0, st>>>(x, y, n, scale, offset, p);
        return (int)cudaGetLastError();
    }
    const int grid = grid_for(vec ? (n + 3) / 4 : n, kThreads, vec ? kUnroll : 4, 8);       // persistent: SM count x 8 CTAs
    if (vec) ew_tensor_kernel<Op, OutT, true><<<grid, kThreads, 0, st>>>(x, y, n, scale, offset, p);
    else     ew_tensor_kernel<Op, OutT, false><<<grid, kThreads, 0, st>>>(x, y, n, scale, offset, p);
    return (int)cudaGetLastError();
}

template <class Op, class OutT>
static int launch_channel(const float *x, OutT *y, int64_t n, int64_t epc, int C, const float *scale, const float *offset,
                          typename Op::Params p, cudaStream_t st) {
    if (n <= 0 || epc <= 0 || C <= 0 || !x || !y || !scale || !offset) return (int)cudaErrorInvalidValue;
    if (epc > 0x7fffffffLL || n % epc != 0) return (int)cudaErrorInvalidValue;
    const bool al = aligned16(x) && out_aligned<OutT>(y);
    const auto table_grid = [&]() {
        int64_t tiles = ((n + 3) / 4 + kTileVec - 1) / kTileVec;
        const int64_t cap = (int64_t)sm_count() * 5;                    // 44 registers, 2 x 16.4 KB of tables: five CTAs per SM
        return (int)(tiles < cap ? tiles : cap);
    };
    if (epc % 4 == 0 && al) {
        const int64_t n4 = n / 4;
        if (n4 <= 0x1fffffffLL && epc / 4 >= 128) {
            const int grid = grid_for(n4, kThreads, kUnroll, 16);
            ew_channel_seg_kernel<Op, OutT><<<grid, kThreads, 0, st>>>(x, y, (uint32_t)n4, C, (uint32_t)(epc / 4), FastDiv32((uint32_t)(epc / 4)),
                                                                          FastDiv32((uint32_t)C), scale, offset, p);
            return (int)cudaGetLastError();
        }
        if (n <= 0x7fffffffLL && variant_of(kVarChannel) == 0) {        // short rows: per-row operators from a shared-memory table
            ew_channel_table_kernel<Op, OutT, true><<<table_grid(), kThreads, 0, st>>>(x, y, (uint32_t)n, (uint32_t)epc, C, FastDiv32((uint32_t)epc),
                                                                                       FastDiv32((uint32_t)C), scale, offset, p);
            return (int)cudaGetLastError();
        }
        if (n4 <= 0x7fffffffLL) {
            const int grid = grid_for(n4, kThreads, kUnroll, 16);
            ew_channel_vec_kernel<Op, OutT><<<grid, kThreads, 0, st>>>(x, y, (uint32_t)n4, C, FastDiv32((uint32_t)(epc / 4)), FastDiv32((uint32_t)C),
                                                                          scale, offset, p);
            return (int)cudaGetLastError();
        }
    }
    if (epc == 1 && C % 4 == 0 && al) {
        const int64_t n4 = n / 4, C4 = C / 4;
        const int grid = grid_for(n4, kThreads, kUnroll, 8);
        const int64_t threads = (int64_t)grid * kThreads;
        if (threads >= C4) {
            ew_channel_last_kernel<Op, OutT><<<grid, kThreads, 0, st>>>(x, y, n4, (uint32_t)C4, (uint32_t)(threads / C4 * C4), scale, offset, p);
            return (int)cudaGetLastError();
        }
    }
    if (epc >= 4 && al && n <= 0x7fffffffLL && variant_of(kVarChannel) == 0) {      // ragged short rows (depth-wise 3x3: epc 9)
        ew_channel_table_kernel<Op, OutT, false><<<table_grid(), kThreads, 0, st>>>(x, y, (uint32_t)n, (uint32_t)epc, C, FastDiv32((uint32_t)epc),
                                                                                    FastDiv32((uint32_t)C), scale, offset, p);
        return (int)cudaGetLastError();
    }
    const int grid = grid_for((n + 3) / 4, kThreads, 1, 8);
    ew_channel_generic_kernel<Op, OutT><<<grid, kThreads, 0, st>>>(x, y, n, epc, C, FastDiv((uint32_t)epc), FastDiv((uint32_t)C),
                                                                      scale, offset, p);
    return (int)cudaGetLastError();
}

// Host twin of the fast-path condition (see FloatOp<MODE, FAST> in ops.cuh).
static inline bool float_fast_path_ok(int E, int M, float cmin, float cmax) {
    auto f2u = [](float f) { uint32_t u; memcpy(&u, &f, 4); return u; };
    auto u2f = [](uint32_t u) { float f; memcpy(&f, &u, 4); return f; };
    const int emin = -(1 << (E - 1)) + 1, emax = 1 << (E - 1);
    const uint32_t top = ~(0x007FFFFFu >> M) & 0x007FFFFFu;
    const float tmax = u2f((uint32_t)((emax + 127) << 23) + top);
    const float hi = cmax < tmax ? cmax : tmax, lo = cmin > -tmax ? cmin : -tmax;
    const uint32_t thresh = (uint32_t)(emin + 1 + 127) << 23, half_minus1 = (1u << (22 - M)) - 1u, keep = ~((1u << (23 - M)) - 1u);
    const uint32_t hb = f2u(hi) & 0x7FFFFFFFu, lb = f2u(lo) & 0x7FFFFFFFu;
    return hi > 0.f && lo < 0.f && hb >= thresh && lb >= thresh && ((hb + half_minus1) & keep) == hb && ((lb + half_minus1) & keep) == lb;
}

static inline bool valid_fp_format(int E, int M) {
    // The reference forms min_subnormal with an int shift `1 << (2^(E-1) + M - 2)` (common.cuh:209): defined only
    // while that shift is in 0..30, which also keeps every constant a normal fp32.  E4M3, E5M2, E5M10 (fp16) are inside.
    if (E < 1 || E > 5 || M < 0 || M > 22) return false;
    const int k = (1 << (E - 1)) + M - 2;
    return k >= 0 && k <= 30;
}

}  // namespace ppqb

using namespace ppqb;

// TMA-staged variant lives in fakequant_tma.cu
int launch_linear_quant_t_tma(const float *x, float *y, int64_t n, const float *scale, const float *offset,
                              int qmin, int qmax, cudaStream_t st);

extern "C" {

// Every rounding policy is a compile-time instantiation behind one switch (the run-time-mode operator, LinearOp<-1>, costs 20 points of
// HBM peak: its uniform branches and the fp32 "+ .5" forms of all four half-way modes stay live in the loop).
#define PPQB_DISPATCH_MODE(rounding, ...)                           \
    switch (rounding) {                                             \
    case RND_HALF_EVEN:          { constexpr int M_ = RND_HALF_EVEN; __VA_ARGS__; }          \
    case RND_HALF_UP:            { constexpr int M_ = RND_HALF_UP; __VA_ARGS__; }            \
    case RND_HALF_DOWN:          { constexpr int M_ = RND_HALF_DOWN; __VA_ARGS__; }          \
    case RND_HALF_TOWARDS_ZERO:  { constexpr int M_ = RND_HALF_TOWARDS_ZERO; __VA_ARGS__; }  \
    case RND_HALF_FAR_FROM_ZERO: { constexpr int M_ = RND_HALF_FAR_FROM_ZERO; __VA_ARGS__; } \
    case RND_TO_NEAR_INT:        { constexpr int M_ = RND_TO_NEAR_INT; __VA_ARGS__; }        \
    case RND_UP:                 { constexpr int M_ = RND_UP; __VA_ARGS__; }                 \
    case RND_DOWN:               { constexpr int M_ = RND_DOWN; __VA_ARGS__; }               \
    default: break;                                                 \
    }

int ppq_b200_linear_quant_t(const float *x, float *y, int64_t n, const float *scale, const float *offset,
                            int qmin, int qmax, int rounding, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (qmin > qmax) return (int)cudaErrorInvalidValue;
    if (rounding == RND_HALF_EVEN) {
        const int var = variant_of(kVarLinearT);
        if (var == 1 && n >= 4096 && aligned16(x) && aligned16(y))
            return launch_linear_quant_t_tma(x, y, n, scale, offset, qmin, qmax, st);
        if (var >= 2 && n >= 4096 && aligned16(x) && aligned16(y)) {          // launch-shape A/B knobs (tools/kbench.py; results in DESIGN.md)
            using Op = LinearOp<0>;
            const Op::Params p{qmin, qmax, 0};
            const int64_t n4 = (n + 3) / 4;
            if (var == 2) ew_tensor_kernel<Op, float, true, 8, 256><<<grid_for(n4, 256, 8, 16), 256, 0, st>>>(x, y, n, scale, offset, p);      // 8 loads in flight
            else ew_tensor_kernel<Op, float, true, 4, 256><<<grid_for(n4, 256, 4, 8), 256, 0, st>>>(x, y, n, scale, offset, p);                 // 4 loads, persistent
            return (int)cudaGetLastError();
        }
    }
    PPQB_DISPATCH_MODE(rounding, return (launch_tensor<LinearOp<M_>, float>(x, y, n, scale, offset, {qmin, qmax, M_}, st)))
    return launch_tensor<LinearOp<-1>, float>(x, y, n, scale, offset, {qmin, qmax, rounding}, st);     // unknown ids: the reference's `default` branch
}

int ppq_b200_linear_quant_c(const float *x, float *y, int64_t n, int64_t epc, int C, const float *scale, const float *offset,
                            int qmin, int qmax, int rounding, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (qmin > qmax) return (int)cudaErrorInvalidValue;
    PPQB_DISPATCH_MODE(rounding, return (launch_channel<LinearOp<M_>, float>(x, y, n, epc, C, scale, offset, {qmin, qmax, M_}, st)))
    return launch_channel<LinearOp<-1>, float>(x, y, n, epc, C, scale, offset, {qmin, qmax, rounding}, st);
}

static int toint_bits_ok(int out_bits) { return out_bits == 8 || out_bits == 32; }

int ppq_b200_linear_quant_t_toint(const float *x, void *q, int out_bits, int64_t n, const float *scale, const float *offset,
                                  int qmin, int qmax, int rounding, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (qmin > qmax) return (int)cudaErrorInvalidValue;
    if (!toint_bits_ok(out_bits)) return (int)cudaErrorInvalidValue;
    if (rounding == RND_HALF_EVEN) {                                   // the policy every shipped quantizer but one selects: compile-time
        if (out_bits == 8) return launch_tensor<LinearOp<0>, int8_t>(x, (int8_t *)q, n, scale, offset, {qmin, qmax, 0}, st);
        return launch_tensor<LinearOp<0>, int32_t>(x, (int32_t *)q, n, scale, offset, {qmin, qmax, 0}, st);
    }
    if (out_bits == 8) return launch_tensor<LinearOp<-1>, int8_t>(x, (int8_t *)q, n, scale, offset, {qmin, qmax, rounding}, st);
    return launch_tensor<LinearOp<-1>, int32_t>(x, (int32_t *)q, n, scale, offset, {qmin, qmax, rounding}, st);
}

int ppq_b200_linear_quant_c_toint(const float *x, void *q, int out_bits, int64_t n, int64_t epc, int C,
                                  const float *scale, const float *offset, int qmin, int qmax, int rounding, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (qmin > qmax) return (int)cudaErrorInvalidValue;
    if (!toint_bits_ok(out_bits)) return (int)cudaErrorInvalidValue;
    if (rounding == RND_HALF_EVEN) {
        if (out_bits == 8) return launch_channel<LinearOp<0>, int8_t>(x, (int8_t *)q, n, epc, C, scale, offset, {qmin, qmax, 0}, st);
        return launch_channel<LinearOp<0>, int32_t>(x, (int32_t *)q, n, epc, C, scale, offset, {qmin, qmax, 0}, st);
    }
    if (out_bits == 8) return launch_channel<LinearOp<-1>, int8_t>(x, (int8_t *)q, n, epc, C, scale, offset, {qmin, qmax, rounding}, st);
    return launch_channel<LinearOp<-1>, int32_t>(x, (int32_t *)q, n, epc, C, scale, offset, {qmin, qmax, rounding}, st);
}

int ppq_b200_multi_linear_quant_c(const ppq_b200_lc_desc *descs, int count, int64_t max_n, int qmin, int qmax, int rounding, void *stream) {
    if (count <= 0 || count > kMaxMultiTensors || max_n <= 0 || max_n > 0x7fffffffLL || !descs || qmin > qmax) return (int)cudaErrorInvalidValue;
    // upper bound of the work (the true total is summed on the device): one CTA per 8 segments of 512 elements, at most 8 CTAs per SM
    int64_t g = ((int64_t)count * ((max_n + 4 * kSegVec - 1) / (4 * kSegVec)) + 7) / 8;
    if (g > (int64_t)sm_count() * 8) g = (int64_t)sm_count() * 8;
    const size_t smem = (size_t)(count + 1) * sizeof(long long);
    if (rounding == RND_HALF_EVEN) multi_channel_kernel<LinearOp<0>><<<(int)g, kThreads, smem, (cudaStream_t)stream>>>(descs, count, {qmin, qmax, 0});
    else if (rounding == RND_HALF_UP) multi_channel_kernel<LinearOp<RND_HALF_UP>><<<(int)g, kThreads, smem, (cudaStream_t)stream>>>(descs, count, {qmin, qmax, RND_HALF_UP});
    else multi_channel_kernel<LinearOp<-1>><<<(int)g, kThreads, smem, (cudaStream_t)stream>>>(descs, count, {qmin, qmax, rounding});
    return (int)cudaGetLastError();
}

int ppq_b200_multi_linear_quant_t(const ppq_b200_lt_desc *descs, int count, int64_t max_n, int qmin, int qmax, int rounding, void *stream) {
    if (count <= 0 || count > kMaxMultiTensors || max_n <= 0 || max_n > 0x7fffffffLL || !descs || qmin > qmax) return (int)cudaErrorInvalidValue;
    int64_t g = ((int64_t)count * ((max_n + 4 * kSegVec - 1) / (4 * kSegVec)) + 7) / 8;      // upper bound: one CTA per 8 segments, at most 8 CTAs per SM
    if (g > (int64_t)sm_count() * 8) g = (int64_t)sm_count() * 8;
    const size_t smem = (size_t)(count + 1) * sizeof(long long);
    cudaStream_t st = (cudaStream_t)stream;
    PPQB_DISPATCH_MODE(rounding, { multi_tensor_kernel<LinearOp<M_>><<<(int)g, kThreads, smem, st>>>(descs, count, {qmin, qmax, M_}); return (int)cudaGetLastError(); })
    multi_tensor_kernel<LinearOp<-1>><<<(int)g, kThreads, smem, st>>>(descs, count, {qmin, qmax, rounding});
    return (int)cudaGetLastError();
}

int ppq_b200_float_quant_t(const float *x, float *y, int64_t n, const float *scale, const float *offset,
                           int exponent, int mantissa, float clip_min, float clip_max, int rounding, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (!valid_fp_format(exponent, mantissa)) return (int)cudaErrorInvalidValue;
    if (float_fast_path_ok(exponent, mantissa, clip_min, clip_max)) {
        PPQB_DISPATCH_MODE(rounding, return (launch_tensor<FloatOp<M_, true>, float>(x, y, n, scale, offset, {exponent, mantissa, M_, clip_min, clip_max}, st)))
    }
    if (rounding == RND_HALF_EVEN) return launch_tensor<FloatOp<0>, float>(x, y, n, scale, offset, {exponent, mantissa, 0, clip_min, clip_max}, st);
    return launch_tensor<FloatOp<-1>, float>(x, y, n, scale, offset, {exponent, mantissa, rounding, clip_min, clip_max}, st);
}

int ppq_b200_float_quant_c(const float *x, float *y, int64_t n, int64_t epc, int C, const float *scale, const float *offset,
                           int exponent, int mantissa, float clip_min, float clip_max, int rounding, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (!valid_fp_format(exponent, mantissa)) return (int)cudaErrorInvalidValue;
    if (float_fast_path_ok(exponent, mantissa, clip_min, clip_max)) {
        PPQB_DISPATCH_MODE(rounding, return (launch_channel<FloatOp<M_, true>, float>(x, y, n, epc, C, scale, offset, {exponent, mantissa, M_, clip_min, clip_max}, st)))
    }
    if (rounding == RND_HALF_EVEN) return launch_channel<FloatOp<0>, float>(x, y, n, epc, C, scale, offset, {exponent, mantissa, 0, clip_min, clip_max}, st);
    return launch_channel<FloatOp<-1>, float>(x, y, n, epc, C, scale, offset, {exponent, mantissa, rounding, clip_min, clip_max}, st);
}

}  // extern "C"
