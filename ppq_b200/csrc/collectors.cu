// collectors.cu -- sm_90a calibration collectors behind the C ABI of include/ppq_b200.h.
//
//   ppq_b200_minmax_t / _c          fused single-pass min+max; replaces the two torch reductions of
//                                   TorchMinMaxObserver.observe (/root/reference/ppq/quantization/observer/range.py:85-100)
//   ppq_b200_histogram_t            replaces Histogram_T            (ppq/csrc/cuda/sort.cu:75-111)
//   ppq_b200_histogram_asym_t       replaces Histogram_Asymmetric_T (sort.cu:113-165)
//   ppq_b200_histogram_c            replaces Histogram_C            (sort.cu:167-218)
//   ppq_b200_multi_*                one launch over a table of tensors (the calibration arena path, DESIGN.md)
//
// All of them read each element exactly once (4 B/element algorithmic traffic): the single-tensor collectors with 128-bit streaming
// loads, the multi-tensor ones through a cp.async.bulk ring in shared memory (multi_stream_kernel).  Histograms are privatised per
// CTA in shared memory (bins x int32, 16 KB for the KL observer's 4096
// bins) and counted with an unconditional red.shared.add into `bins + 1` slots (the extra one is a trash slot for dropped
// samples; ptxas emits ATOMS.POPC.INC, which aggregates same-address lanes in hardware, so the post-ReLU pile-up in bin 0 is
// not a hot spot); only non-empty bins are flushed to the caller's global histogram with red.global.add.
#include "common.cuh"
#include "half.cuh"
#include "../../include/ppq_b200.h"
#include "variants.h"
#include <cooperative_groups.h>

namespace ppqb {
namespace cg = cooperative_groups;

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

__device__ __forceinline__ float min_nan(float a, float b) { float r; asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float max_nan(float a, float b) { float r; asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }

// NaN-propagating (min, max) of a thread's values -> warp -> CTA; result valid in thread 0.
struct MinMax {
    float lo, hi;
    __device__ __forceinline__ MinMax() { lo = __int_as_float(0x7F800000); hi = __int_as_float(0xFF800000); }
    __device__ __forceinline__ void add(float v) { lo = min_nan(lo, v); hi = max_nan(hi, v); }
    __device__ __forceinline__ void add4(const float4 &v) { add(v.x); add(v.y); add(v.z); add(v.w); }
    __device__ __forceinline__ void warp_reduce() {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo = min_nan(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = max_nan(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
    }
    // publish into accumulating global slots (see common.cuh: raw-bit float atomics, NaN poisons both slots)
    __device__ __forceinline__ void publish(float *gmin, float *gmax) const {
        if (lo != lo || hi != hi) {
            atomic_min_float(gmin, __uint_as_float(0xFFC00000u));
            atomic_max_float(gmax, __uint_as_float(0x7FC00000u));
        } else {
            atomic_min_float(gmin, lo);
            atomic_max_float(gmax, hi);
        }
    }
};

__device__ __forceinline__ void block_reduce_publish(MinMax mm, float *gmin, float *gmax) {
    __shared__ float s_lo[kThreads / 32], s_hi[kThreads / 32];
    mm.warp_reduce();
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { s_lo[w] = mm.lo; s_hi[w] = mm.hi; }
    __syncthreads();
    if (w == 0) {
        MinMax t;
        if (l < kThreads / 32) { t.lo = s_lo[l]; t.hi = s_hi[l]; }
        t.warp_reduce();
        if (l == 0) t.publish(gmin, gmax);
    }
    __syncthreads();
}

// Streams elements [0, n) of x through `f(float)`; float4 path when the base is 16-byte aligned.
// `first`/`stride` are in units of threads over the whole cooperating group (a grid or a sub-grid).
template <class F>
__device__ __forceinline__ void stream_elements(const float *__restrict__ x, int64_t n, int64_t first, int64_t stride, F &&f) {
    if ((reinterpret_cast<uintptr_t>(x) & 15u) == 0) {
        const int64_t n4 = n >> 2;
        const float4 *x4 = reinterpret_cast<const float4 *>(x);
        // warp-contiguous segments of 32 x kUnroll vectors (lane-interleaved): a thread's kUnroll loads in flight fall into one 2 KB
        // span of HBM (same pattern as the fake-quant kernels, where it measured +3..4 points of HBM peak over grid-stride)
        constexpr int64_t kSeg = 32 * kUnroll;
        const int64_t lane = first & 31, warp = first >> 5, warps = stride >> 5;
        const int64_t segs = (n4 + kSeg - 1) / kSeg;
        for (int64_t sg = warp; sg < segs; sg += warps) {
            const int64_t base = sg * kSeg + lane;
            float4 v[kUnroll];
#pragma unroll
            for (int j = 0; j < kUnroll; j++) if (base + j * 32 < n4) v[j] = ld_stream4(x4 + base + j * 32);
#pragma unroll
            for (int j = 0; j < kUnroll; j++) if (base + j * 32 < n4) { f(v[j].x); f(v[j].y); f(v[j].z); f(v[j].w); }
        }
        const int64_t t = (n4 << 2) + first;
        if (t < n) f(x[t]);
    } else {
        for (int64_t i = first; i < n; i += stride) f(ld_stream1(x + i));
    }
}

// The same for fp16 / bf16: 16-byte loads of 8 elements converted to fp32 in registers; the <= 7 elements before the first 16-byte
// boundary and the <= 7 after the last whole vector go one per thread to the first threads of the group.
template <class T, class F, std::enable_if_t<is_half_t<T>::value, int> = 0>
__device__ __forceinline__ void stream_elements(const T *__restrict__ x, int64_t n, int64_t first, int64_t stride, F &&f) {
    const int64_t head = min(n, head_elems(x));
    const int64_t nv = (n - head) >> 3, tail0 = head + (nv << 3);
    const uint4 *x8 = reinterpret_cast<const uint4 *>(x + head);
    constexpr int64_t kSeg = 32 * kUnroll;
    const int64_t lane = first & 31, warp = first >> 5, warps = stride >> 5;
    const int64_t segs = (nv + kSeg - 1) / kSeg;
    for (int64_t sg = warp; sg < segs; sg += warps) {
        const int64_t base = sg * kSeg + lane;
        uint4 v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; j++) if (base + j * 32 < nv) v[j] = ld_stream_u4(x8 + base + j * 32);
#pragma unroll
        for (int j = 0; j < kUnroll; j++) {
            if (base + j * 32 < nv) {
                float4 a, b;
                unpack8<T>(v[j], a, b);
                f(a.x); f(a.y); f(a.z); f(a.w); f(b.x); f(b.y); f(b.z); f(b.w);
            }
        }
    }
    if (first < head) f(ld_stream1_f(x + first));
    else if (first - head < n - tail0) f(ld_stream1_f(x + tail0 + (first - head)));
}

// ---- min / max ------------------------------------------------------------------------------------------------------
__global__ void minmax_init_kernel(float *mins, float *maxs, int64_t count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) {
        if (mins) mins[i] = __int_as_float(0x7F800000);
        if (maxs) maxs[i] = __int_as_float(0xFF800000);
    }
}

template <class T>
__global__ void __launch_bounds__(kThreads)
minmax_t_kernel(const T *__restrict__ x, int64_t n, float *__restrict__ minmax) {
    MinMax mm;
    stream_elements(x, n, (int64_t)blockIdx.x * kThreads + threadIdx.x, (int64_t)gridDim.x * kThreads,
                    [&](float v) { mm.add(v); });
    block_reduce_publish(mm, minmax, minmax + 1);
}

// Per channel: tensor = rows x epc, channel(row) = row % C.  One warp per (row, chunk) work item.
constexpr int kRowChunk = 4096;
template <class T>
__global__ void __launch_bounds__(kThreads)
minmax_c_kernel(const T *__restrict__ x, int64_t rows, int64_t epc, int C, int64_t chunks_per_row,
                FastDiv div_chunks, FastDiv div_C, float *__restrict__ mins, float *__restrict__ maxs) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (kThreads / 32);
    const int64_t items = rows * chunks_per_row;
    for (int64_t item = (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); item < items; item += warps) {
        const int64_t row = (int64_t)div_chunks.quot((uint64_t)item);
        const int64_t chunk = item - row * chunks_per_row;
        const int c = (int)(row - (int64_t)div_C.quot((uint64_t)row) * C);
        const int64_t begin = chunk * kRowChunk;
        const int64_t len = (epc - begin) < kRowChunk ? (epc - begin) : kRowChunk;
        MinMax mm;
        stream_elements(x + row * epc + begin, len, lane, 32, [&](float v) { mm.add(v); });
        mm.warp_reduce();
        if (lane == 0) mm.publish(mins + c, maxs + c);
    }
}

// ---- histograms -------------------------------------------------------------------------------------------------------
// Binning operators map a value to a slot of the CTA-private shared histogram: slots 0..bins-1 are the bins, slot `bins`
// is a trash slot for dropped samples, so that the shared atomic is unconditional (no branch per element; ptxas turns
// `red.shared.add.u32 [a], 1` into ATOMS.POPC.INC, which aggregates same-address lanes of a warp in hardware -- the
// post-ReLU pile-up in bin 0 costs one pass, not 32).
struct BinParams { float a, b; int bins, clip; };   // sym: a = hist_scale;  asym: a = min, b = max
struct SymBin {
    ExactDiv d; unsigned bins; int last; bool clip;
    __device__ __forceinline__ SymBin(float hist_scale, int nbins, bool clip_outliers) : bins(nbins), last(nbins - 1), clip(clip_outliers) { d.init(hist_scale); }
    __device__ __forceinline__ explicit SymBin(const BinParams &p) : SymBin(p.a, p.bins, p.clip != 0) {}
    __device__ __forceinline__ unsigned finish(float t) const {
        const int b = __float2int_rd(t);                              // (int) floor(.), saturating, NaN -> 0; never negative here
        return clip ? min((unsigned)b, bins) : (unsigned)min(b, last);
    }
    __device__ __forceinline__ unsigned operator()(float v) const { return finish(d.div(fabsf(v))); }
    __device__ __forceinline__ uint4 bin4(const float4 &v) const {
        const float4 t = d.div4(make_float4(fabsf(v.x), fabsf(v.y), fabsf(v.z), fabsf(v.w)));
        return make_uint4(finish(t.x), finish(t.y), finish(t.z), finish(t.w));
    }
};
struct AsymBin {
    ExactDiv d; float vmin; unsigned bins; int last; bool clip;
    __device__ __forceinline__ AsymBin(float mn, float mx, int nbins, bool clip_outliers) : vmin(mn), bins(nbins), last(nbins - 1), clip(clip_outliers) {
        d.init(__fdiv_rn(__fsub_rn(mx, mn), (float)nbins));           // hist_scale = (max - min) / bins, in fp32
    }
    __device__ __forceinline__ explicit AsymBin(const BinParams &p) : AsymBin(p.a, p.b, p.bins, p.clip != 0) {}
    __device__ __forceinline__ unsigned finish(float t) const {
        const int b = __float2int_rd(t);
        return clip ? min((unsigned)b, bins) : (unsigned)max(min(b, last), 0);   // negative b wraps above `bins` -> trash
    }
    __device__ __forceinline__ unsigned operator()(float v) const { return finish(d.div(__fsub_rn(v, vmin))); }
    __device__ __forceinline__ uint4 bin4(const float4 &v) const {
        const float4 t = d.div4(make_float4(__fsub_rn(v.x, vmin), __fsub_rn(v.y, vmin), __fsub_rn(v.z, vmin), __fsub_rn(v.w, vmin)));
        return make_uint4(finish(t.x), finish(t.y), finish(t.z), finish(t.w));
    }
};

// Counting into the CTA-private histogram.
//   VARIANT 0 (default): unconditional red.shared.add through a precomputed 32-bit shared-window address.
//   VARIANT 1: the same through generic-pointer atomicAdd;  VARIANT 2: __match_any_sync aggregation in software;
//   VARIANT 3: global atomics straight into `hist` (what the reference does; kept for A/B measurements only).
template <int VARIANT>
struct Counter {
    int *sh; int32_t *gh; uint32_t sh_addr; unsigned trash;
    __device__ __forceinline__ Counter(int *smem_hist, int32_t *global_hist, int bins)
        : sh(smem_hist), gh(global_hist), sh_addr((uint32_t)__cvta_generic_to_shared(smem_hist)), trash(bins) {}
    __device__ __forceinline__ void count(unsigned slot) {
        if constexpr (VARIANT == 0) {
            asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(sh_addr + slot * 4u) : "memory");
        } else if constexpr (VARIANT == 1) {
            atomicAdd(sh + slot, 1);
        } else if constexpr (VARIANT == 2) {
            const unsigned peers = __match_any_sync(0xffffffffu, slot);
            if ((threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(sh + slot, __popc(peers));
        } else {
            if (slot != trash) atomicAdd(gh + slot, 1);
        }
    }
};

template <int VARIANT>
__device__ __forceinline__ void hist_zero(int *sh, int bins) {
    if constexpr (VARIANT != 3) {
        for (int i = threadIdx.x; i <= bins; i += blockDim.x) sh[i] = 0;    // + the trash slot
        __syncthreads();
    }
}
template <int VARIANT>
__device__ __forceinline__ void hist_flush(const int *sh, int bins, int32_t *gh) {
    if constexpr (VARIANT != 3) {
        __syncthreads();
        for (int i = threadIdx.x; i < bins; i += blockDim.x) {
            const int v = sh[i];
            if (v) atomicAdd(gh + i, v);
        }
        __syncthreads();
    }
}

// The ballot in VARIANT 0/2 needs all 32 lanes of a warp to call count() the same number of times: stream_elements
// gives every lane of a warp the same trip count except in the ragged tail, so tails are padded with "drop" (-1).
template <int VARIANT, class Bin, int U = kUnroll>
__device__ __forceinline__ void hist_stream(const float *__restrict__ x, int64_t n, int64_t first, int64_t stride,
                                            const Bin &bin, Counter<VARIANT> &cnt) {
    if ((reinterpret_cast<uintptr_t>(x) & 15u) == 0) {
        const int64_t n4 = n >> 2;
        const float4 *x4 = reinterpret_cast<const float4 *>(x);
        const int64_t warp_first = first - (threadIdx.x & 31);              // lane 0 of this warp
        int64_t i = first;
        // full unrolled rounds: uniform across the warp because lanes are consecutive in i
        for (; warp_first + (i - first) + 31 + (U - 1) * stride < n4; i += U * stride) {
            float4 v[U];
#pragma unroll
            for (int j = 0; j < U; j++) v[j] = ld_stream4(x4 + i + j * stride);
#pragma unroll
            for (int j = 0; j < U; j++) { const uint4 b = bin.bin4(v[j]); cnt.count(b.x); cnt.count(b.y); cnt.count(b.z); cnt.count(b.w); }
        }
        // remaining rounds: warp-uniform loop bound, per-lane predicate
        for (; warp_first + (i - first) < n4; i += stride) {
            const bool ok = i < n4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok) v = ld_stream4(x4 + i);
            const uint4 b = bin.bin4(v);
            cnt.count(ok ? b.x : cnt.trash); cnt.count(ok ? b.y : cnt.trash); cnt.count(ok ? b.z : cnt.trash); cnt.count(ok ? b.w : cnt.trash);
        }
        const int64_t t = (n4 << 2) + first;
        const bool tail_any = (n4 << 2) + warp_first < n;                    // warp-uniform
        if (tail_any) cnt.count(t < n ? bin(x[t]) : cnt.trash);
    } else {
        const int64_t warp_first = first - (threadIdx.x & 31);
        for (int64_t i = first; warp_first + (i - first) < n; i += stride) cnt.count(i < n ? bin(ld_stream1(x + i)) : cnt.trash);
    }
}

// fp16 / bf16: 16-byte loads of 8 elements, same warp-uniform trip counts and trash padding; the <= 7 + 7 unaligned head and tail
// elements go one per thread to the first threads of the group.
template <int VARIANT, class Bin, int U = kUnroll, class T, std::enable_if_t<is_half_t<T>::value, int> = 0>
__device__ __forceinline__ void hist_stream(const T *__restrict__ x, int64_t n, int64_t first, int64_t stride,
                                            const Bin &bin, Counter<VARIANT> &cnt) {
    const int64_t head = min(n, head_elems(x));
    const int64_t nv = (n - head) >> 3, tail0 = head + (nv << 3);
    const uint4 *x8 = reinterpret_cast<const uint4 *>(x + head);
    const int64_t warp_first = first - (threadIdx.x & 31);
    auto count8 = [&](const uint4 &r, bool ok) {
        float4 a, b;
        unpack8<T>(r, a, b);
        const uint4 ba = bin.bin4(a), bb = bin.bin4(b);
        cnt.count(ok ? ba.x : cnt.trash); cnt.count(ok ? ba.y : cnt.trash); cnt.count(ok ? ba.z : cnt.trash); cnt.count(ok ? ba.w : cnt.trash);
        cnt.count(ok ? bb.x : cnt.trash); cnt.count(ok ? bb.y : cnt.trash); cnt.count(ok ? bb.z : cnt.trash); cnt.count(ok ? bb.w : cnt.trash);
    };
    int64_t i = first;
    for (; warp_first + (i - first) + 31 + (U - 1) * stride < nv; i += U * stride) {
        uint4 v[U];
#pragma unroll
        for (int j = 0; j < U; j++) v[j] = ld_stream_u4(x8 + i + j * stride);
#pragma unroll
        for (int j = 0; j < U; j++) count8(v[j], true);
    }
    for (; warp_first + (i - first) < nv; i += stride) {
        const bool ok = i < nv;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (ok) v = ld_stream_u4(x8 + i);
        count8(v, ok);
    }
    const int64_t extra = head + (n - tail0);
    if (warp_first < extra) {                                            // warp-uniform
        const bool ok = first < extra;
        float v = 0.f;
        if (ok) v = ld_stream1_f(first < head ? x + first : x + tail0 + (first - head));
        cnt.count(ok ? bin(v) : cnt.trash);
    }
}

constexpr int kHistThreads = 1024;   // big CTAs: the flush of the private bins (bins global atomics per CTA) is what limits small-CTA
                                     // configurations (measured: 256 thr x 8/SM 59 % -> 1024 thr x 1/SM 82-86 % -> 1024 thr x 2/SM, two
                                     // loads in flight, 87 % of HBM peak: r02_kbench.txt)
template <int VARIANT, class Bin, int U = kUnroll, int TPB = kHistThreads, int MINB = 1, class T = float>
__global__ void __launch_bounds__(TPB, MINB)
histogram_kernel(const T *__restrict__ x, int64_t n, BinParams bp, int32_t *__restrict__ hist) {
    extern __shared__ int sh[];
    const int bins = bp.bins;
    hist_zero<VARIANT>(sh, bins);
    Counter<VARIANT> cnt(sh, hist, bins);
    const Bin bin(bp);
    hist_stream<VARIANT, Bin, U>(x, n, (int64_t)blockIdx.x * TPB + threadIdx.x, (int64_t)gridDim.x * TPB, bin, cnt);
    hist_flush<VARIANT>(sh, bins, hist);
}

// Cluster variant (A/B: variants 7 / 8 = clusters of 2 / 4 CTAs): the CTAs of a thread-block cluster reduce their private bins through
// distributed shared memory before touching global memory -- CTA r sums slice r of all CL private histograms with DSMEM loads and flushes
// only that slice, so a launch issues grid / CL x bins global atomics instead of grid x bins (the flush of 148 x 4096 counters is the fixed
// cost that separates the single-tensor collector from the multi-tensor one, DESIGN.md §5).
template <class Bin, int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(kHistThreads)
histogram_cluster_kernel(const float *__restrict__ x, int64_t n, BinParams bp, int32_t *__restrict__ hist) {
    extern __shared__ int sh[];
    cg::cluster_group cluster = cg::this_cluster();
    const int bins = bp.bins;
    hist_zero<0>(sh, bins);
    Counter<0> cnt(sh, hist, bins);
    const Bin bin(bp);
    hist_stream<0, Bin>(x, n, (int64_t)blockIdx.x * kHistThreads + threadIdx.x, (int64_t)gridDim.x * kHistThreads, bin, cnt);
    cluster.sync();                                                     // every CTA of the cluster has finished counting
    const unsigned r = cluster.block_rank();
    const int *peer[CL];
#pragma unroll
    for (int c = 0; c < CL; c++) peer[c] = cluster.map_shared_rank(sh, c);
    const int slice = (bins + CL - 1) / CL, b0 = (int)r * slice, b1 = min(bins, b0 + slice);
    for (int i = b0 + (int)threadIdx.x; i < b1; i += kHistThreads) {
        int v = 0;
#pragma unroll
        for (int c = 0; c < CL; c++) v += peer[c][i];
        if (v) atomicAdd(hist + i, v);
    }
    cluster.sync();                                                     // nobody exits while a peer still reads its shared memory
}

// hist_scale read from device memory (phase 2 without a host round trip); VARIANT 3 (global atomics) above kMaxSmemBins bins
template <int VARIANT, int TPB = kHistThreads, int MINB = 2, class T = float>
__global__ void __launch_bounds__(TPB, MINB)
histogram_dscale_kernel(const T *__restrict__ x, int64_t n, const float *__restrict__ hist_scale, int clip, int bins,
                        int32_t *__restrict__ hist) {
    extern __shared__ int sh[];
    hist_zero<VARIANT>(sh, bins);
    Counter<VARIANT> cnt(sh, hist, bins);
    const SymBin bin(__ldg(hist_scale), bins, clip != 0);
    hist_stream<VARIANT, SymBin, 2>(x, n, (int64_t)blockIdx.x * TPB + threadIdx.x, (int64_t)gridDim.x * TPB, bin, cnt);
    hist_flush<VARIANT>(sh, bins, hist);
}

// ---- multi-tensor collectors: one streaming engine ------------------------------------------------------------------------
// Each CTA owns one contiguous span of the concatenation of all tensors (cut points inside a tensor rounded up to a multiple of one
// 16-byte vector -- 4 fp32 or 8 fp16 / bf16 elements -- the same way by both neighbours), so per-tensor state is set up and published
// (#CTAs + #tensors) times per launch.  The element type T is one per table: every descriptor's `x` points at elements of that type.
// Warp-specialised CTA: one producer lane walks the CTA's pieces (tensor t, elements [a, b)) and issues 1-D cp.async.bulk copies of
// their 16-byte-aligned bodies into a ring of kRingStages tiles (full / empty mbarriers); the consumer warps walk the same pieces,
// apply Op to every element of each tile from shared memory (half elements are unpacked to fp32 in registers: the ring moves bytes, a
// 16 KB stage is 4096 floats or 8192 halves), and handle the unaligned head / tail elements of a piece (at most 3 + 3 floats, 7 + 7
// halves: a half tensor may start at any 2-byte offset) with plain loads.  Copies keep flowing while the consumers bin, flush or wait
// at a piece boundary.
constexpr int kRingConsumers = 512;                  // 16 consumer warps
constexpr int kRingThreads = kRingConsumers + 32;    // + the producer warp
constexpr int kRingTileVec = 1024;                   // float4 per tile (16 KB): two per consumer thread
constexpr int kRingStages = 4;                       // 64 KB of tiles per CTA
constexpr int kRingBarId = 1;                        // named barrier of the consumer warps (0 is __syncthreads)

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ring_wait(uint64_t *bar, uint32_t parity) {
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n"
                 ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync %0, %1;" ::"n"(kRingBarId), "n"(kRingConsumers) : "memory"); }

// Per-tensor min/max: registers per (CTA, tensor), one publish per visit.
struct MinMaxOp {
    struct Args { float *arena; };
    static size_t smem_bytes(int) { return 2 * 2 * (kRingConsumers / 32) * sizeof(float); }
    Args g; float *s_lo; MinMax mm; int visit;
    __device__ __forceinline__ MinMaxOp(const Args &a, void *smem) : g(a), s_lo(reinterpret_cast<float *>(smem)), visit(0) {}
    __device__ __forceinline__ void begin(const ppq_b200_tensor_desc &) { mm = MinMax(); }
    __device__ __forceinline__ void add(float v) { mm.add(v); }
    __device__ __forceinline__ void add4(const float4 &v) { mm.add4(v); }
    __device__ __forceinline__ void end(const ppq_b200_tensor_desc &d) {
        // two alternating staging buffers: warp 0 has read buffer v before anyone passes the barrier of visit v + 1
        float *lo = s_lo + (visit & 1) * 2 * (kRingConsumers / 32), *hi = lo + kRingConsumers / 32;
        visit++;
        const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
        mm.warp_reduce();
        if (l == 0) { lo[w] = mm.lo; hi[w] = mm.hi; }
        consumers_sync();
        if (w == 0) {
            MinMax t;
            if (l < kRingConsumers / 32) { t.lo = lo[l]; t.hi = hi[l]; }
            t.warp_reduce();
            if (l == 0) t.publish(g.arena + 2 * (int64_t)d.slot, g.arena + 2 * (int64_t)d.slot + 1);
        }
    }
};

// Per-tensor symmetric histogram with device-side hist_scale: CTA-private bins (+ trash slot) in shared memory, non-empty bins flushed
// with red.global.add once per visit.
struct HistOp {
    struct Args { const float *hist_scale_arena; int32_t *hist_arena; int bins, clip; };
    static size_t smem_bytes(int bins) { return (size_t)(bins + 1) * sizeof(int); }
    Args g; int *sh; SymBin bin; Counter<0> cnt;
    __device__ __forceinline__ HistOp(const Args &a, void *smem)
        : g(a), sh(reinterpret_cast<int *>(smem)), bin(1.f, a.bins, a.clip != 0), cnt(sh, nullptr, a.bins) {
        for (int i = threadIdx.x; i <= g.bins; i += kRingConsumers) sh[i] = 0;
        consumers_sync();
    }
    __device__ __forceinline__ void begin(const ppq_b200_tensor_desc &d) { bin = SymBin(__ldg(g.hist_scale_arena + d.slot), g.bins, g.clip != 0); }
    __device__ __forceinline__ void add(float v) { cnt.count(bin(v)); }
    __device__ __forceinline__ void add4(const float4 &v) { const uint4 b = bin.bin4(v); cnt.count(b.x); cnt.count(b.y); cnt.count(b.z); cnt.count(b.w); }
    __device__ __forceinline__ void end(const ppq_b200_tensor_desc &d) {
        consumers_sync();                                              // every count of this visit has landed
        int32_t *gh = g.hist_arena + (int64_t)d.slot * g.bins;
        for (int i = threadIdx.x; i <= g.bins; i += kRingConsumers) {
            const int v = sh[i];
            if (v && i < g.bins) atomicAdd(gh + i, v);
            sh[i] = 0;
        }
        consumers_sync();                                              // zeroed before the next visit counts
    }
};

// Shared memory: [ring kRingStages x 16 KB][full, empty mbarriers][prefix int64 x (count + 1)][Op's own]
__host__ __device__ inline size_t ring_prefix_offset() { return (size_t)kRingStages * kRingTileVec * 16 + 2 * kRingStages * sizeof(uint64_t); }
__host__ __device__ inline size_t ring_op_offset(int count) { return ring_prefix_offset() + (size_t)(count + 1) * sizeof(int64_t); }

template <class Op, class T = float>
__global__ void __launch_bounds__(kRingThreads, 2)
multi_stream_kernel(const ppq_b200_tensor_desc *__restrict__ descs, int count, typename Op::Args args) {
    constexpr int64_t kVecElems = 16 / sizeof(T);                      // elements per 16-byte vector
    constexpr int kVecShift = sizeof(T) == 4 ? 2 : 3;
    extern __shared__ __align__(128) unsigned char smem[];
    float4 *ring = reinterpret_cast<float4 *>(smem);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)kRingStages * kRingTileVec * 16), *empty = full + kRingStages;
    int64_t *prefix = reinterpret_cast<int64_t *>(smem + ring_prefix_offset());
    // parallel prefix of the tensor sizes: every thread loads, warp 0 scans 32 contiguous runs
    for (int t = threadIdx.x; t < count; t += kRingThreads) prefix[t + 1] = descs[t].n;
    if (threadIdx.x == 0) {
        prefix[0] = 0;
        for (int s = 0; s < kRingStages; s++) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(full + s)));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(empty + s)), "r"(kRingConsumers / 32));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int per = (count + 31) / 32, t0 = threadIdx.x * per, t1 = min(count, t0 + per);
        int64_t run = 0;
        for (int t = t0; t < t1; t++) run += prefix[t + 1];
        int64_t incl = run;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int64_t u = __shfl_up_sync(0xffffffffu, incl, o); if ((int)threadIdx.x >= o) incl += u; }
        run = incl - run;
        for (int t = t0; t < t1; t++) { run += prefix[t + 1]; prefix[t + 1] = run; }
    }
    __syncthreads();
    const int64_t total = prefix[count];
    int64_t span = (total + gridDim.x - 1) / gridDim.x;
    span = (span + kVecElems - 1) & ~(kVecElems - 1);
    const int64_t s0 = (int64_t)blockIdx.x * span, s1 = (s0 + span) < total ? (s0 + span) : total;
    if (s0 >= total) return;                                           // uniform per CTA
    int t_first;                                                       // first tensor overlapping [s0, s1): binary search
    { int lo = 0, hi = count - 1; while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (prefix[mid] <= s0) lo = mid; else hi = mid - 1; } t_first = lo; }

    // The pieces of this CTA, walked identically by the producer and the consumers.  body = [ia, ia + kVecElems nv) is 16-byte aligned.
    auto for_each_piece = [&](auto &&f) {
        for (int t = t_first; t < count && prefix[t] < s1; t++) {
            const ppq_b200_tensor_desc d = descs[t];
            int64_t a = s0 - prefix[t]; if (a < 0) a = 0;
            int64_t b = s1 - prefix[t]; if (b > d.n) b = d.n;
            a = (a + kVecElems - 1) & ~(kVecElems - 1); if (a > d.n) a = d.n;
            if (b < d.n) b = (b + kVecElems - 1) & ~(kVecElems - 1); if (b > d.n) b = d.n;
            if (b <= a) continue;
            const T *x = reinterpret_cast<const T *>(d.x);
            int64_t ia;
            if constexpr (sizeof(T) == 4) ia = a + (int64_t)((4u - (uint32_t)((reinterpret_cast<uintptr_t>(x + a) >> 2) & 3u)) & 3u);
            else ia = a + head_elems(x + a);
            if (ia > b) ia = b;
            f(d, x, a, b, ia, (b - ia) >> kVecShift);
        }
    };
    if (threadIdx.x >= kRingConsumers) {
        if (threadIdx.x == kRingConsumers) {                           // producer: one lane
            uint32_t k = 0;
            for_each_piece([&](const ppq_b200_tensor_desc &, const T *x, int64_t, int64_t, int64_t ia, int64_t nv) {
                const float4 *src = reinterpret_cast<const float4 *>(x + ia);
                for (int64_t v0 = 0; v0 < nv; v0 += kRingTileVec, k++) {
                    const uint32_t s = k % kRingStages, bytes = (uint32_t)((nv - v0) < kRingTileVec ? (nv - v0) : kRingTileVec) * 16u;
                    if (k >= kRingStages) ring_wait(empty + s, ((k / kRingStages) - 1) & 1);
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(full + s)), "r"(bytes) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(smem_addr(ring + s * kRingTileVec)), "l"(src + v0), "r"(bytes), "r"(smem_addr(full + s)) : "memory");
                }
            });
        }
        return;
    }
    Op op(args, smem + ring_op_offset(count));
    uint32_t k = 0;
    for_each_piece([&](const ppq_b200_tensor_desc &d, const T *x, int64_t a, int64_t b, int64_t ia, int64_t nv) {
        op.begin(d);
        const int64_t ib = ia + kVecElems * nv;                        // ragged head [a, ia) and tail [ib, b): < kVecElems elements each
        const int i = (int)threadIdx.x, head = (int)(ia - a);
        if (i < head) op.add(ld_stream1_f(x + a + i));
        else if (i < head + (int)(b - ib)) op.add(ld_stream1_f(x + ib + (i - head)));
        for (int64_t v0 = 0; v0 < nv; v0 += kRingTileVec, k++) {
            const uint32_t s = k % kRingStages;
            const int cnt = (int)((nv - v0) < kRingTileVec ? (nv - v0) : kRingTileVec);
            ring_wait(full + s, (k / kRingStages) & 1);
            const float4 *tile = ring + s * kRingTileVec;
#pragma unroll
            for (int j = 0; j < kRingTileVec / kRingConsumers; j++) {
                const int vi = i + j * kRingConsumers;
                if constexpr (sizeof(T) == 4) {
                    if (vi < cnt) op.add4(tile[vi]);
                } else if (vi < cnt) {
                    float4 lo, hi;
                    unpack8<T>(reinterpret_cast<const uint4 *>(tile)[vi], lo, hi);
                    op.add4(lo); op.add4(hi);
                }
            }
            __syncwarp();
            if ((i & 31) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(empty + s)) : "memory");
        }
        op.end(d);
    });
}

// Per-channel histogram: rows x epc, hist[c][bins].  One CTA per (row, chunk); smem holds that row's private bins.
template <int VARIANT>
__global__ void __launch_bounds__(kThreads)
histogram_c_kernel(const float *__restrict__ x, int64_t rows, int64_t epc, int C, int64_t chunk, int64_t chunks_per_row,
                   float hist_scale, int clip, int bins, int32_t *__restrict__ hist) {
    extern __shared__ int sh[];
    const int64_t items = rows * chunks_per_row;
    const SymBin bin(hist_scale, bins, clip != 0);
    for (int64_t item = blockIdx.x; item < items; item += gridDim.x) {
        const int64_t row = item / chunks_per_row;
        const int64_t c0 = item - row * chunks_per_row;
        const int ch = (int)(row % C);
        const int64_t begin = c0 * chunk;
        const int64_t len = (epc - begin) < chunk ? (epc - begin) : chunk;
        int32_t *gh = hist + (int64_t)ch * bins;
        hist_zero<VARIANT>(sh, bins);
        Counter<VARIANT> cnt(sh, gh, bins);
        hist_stream<VARIANT>(x + row * epc + begin, len, threadIdx.x, kThreads, bin, cnt);
        hist_flush<VARIANT>(sh, bins, gh);
    }
}

// ---- launch helpers -------------------------------------------------------------------------------------------------------
constexpr int kMaxSmemBins = 12287;            // (bins + 1) int32 slots within the default 48 KB of dynamic shared memory

// Elements each CTA should own before paying for zeroing + flushing `bins` counters.
static inline int hist_grid(int64_t n, int bins) {
    const int64_t per_cta = (int64_t)bins * 16 > 65536 ? (int64_t)bins * 16 : 65536;
    int64_t g = (n + per_cta - 1) / per_cta;
    const int64_t cap = (int64_t)sm_count();
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

template <class Bin>
static int launch_hist(const float *x, int64_t n, const BinParams &bin, int64_t bins, int32_t *hist, cudaStream_t st) {
    int var = variant_of(kVarHistogram);
    if (bins > kMaxSmemBins) var = 3;
    const int grid = var == 3 ? grid_for(n, kThreads, 16, 8) : hist_grid(n, (int)bins);
    const size_t smem = var == 3 ? 0 : (size_t)(bins + 1) * sizeof(int);
    switch (var) {
    case 1:  histogram_kernel<1, Bin><<<grid, kHistThreads, smem, st>>>(x, n, bin, hist); break;
    case 2:  histogram_kernel<2, Bin><<<grid, kHistThreads, smem, st>>>(x, n, bin, hist); break;
    case 3:  histogram_kernel<3, Bin, kUnroll, kThreads><<<grid, kThreads, smem, st>>>(x, n, bin, hist); break;
    case 4:  histogram_kernel<0, Bin, 8, kThreads><<<grid * 8 > sm_count() * 8 ? sm_count() * 8 : grid * 8, kThreads, smem, st>>>(x, n, bin, hist); break;   // the round-1 small-CTA layout
    // 5 / 6: two 1024-thread CTAs per SM (32 registers per thread), 2 / 4 loads in flight per thread
    case 5:  histogram_kernel<0, Bin><<<grid, kHistThreads, smem, st>>>(x, n, bin, hist); break;          // the round-1 default: one 1024-thread CTA per SM, 4 loads in flight
    case 6:  histogram_kernel<0, Bin, 4, kHistThreads, 2><<<grid * 2 > sm_count() * 2 ? sm_count() * 2 : grid * 2, kHistThreads, smem, st>>>(x, n, bin, hist); break;
    // 7 / 8: thread-block clusters of 2 / 4 CTAs, DSMEM pre-reduction of the private bins (grid rounded down to whole clusters)
    case 7:  if (grid >= 2) { histogram_cluster_kernel<Bin, 2><<<grid & ~1, kHistThreads, smem, st>>>(x, n, bin, hist); break; }
             histogram_kernel<0, Bin><<<grid, kHistThreads, smem, st>>>(x, n, bin, hist); break;
    case 8:  if (grid >= 4) { histogram_cluster_kernel<Bin, 4><<<grid & ~3, kHistThreads, smem, st>>>(x, n, bin, hist); break; }
             histogram_kernel<0, Bin><<<grid, kHistThreads, smem, st>>>(x, n, bin, hist); break;
    // default: two 1024-thread CTAs per SM (32 registers per thread), 2 loads in flight per thread
    default: histogram_kernel<0, Bin, 2, kHistThreads, 2><<<grid * 2 > sm_count() * 2 ? sm_count() * 2 : grid * 2, kHistThreads, smem, st>>>(x, n, bin, hist); break;
    }
    return (int)cudaGetLastError();
}

// fp16 / bf16: the default layout of launch_hist only (two 1024-thread CTAs per SM; global atomics beyond kMaxSmemBins bins)
template <class Bin, class T>
static int launch_hist_half(const T *x, int64_t n, const BinParams &bin, int64_t bins, int32_t *hist, cudaStream_t st) {
    if (bins > kMaxSmemBins) {
        histogram_kernel<3, Bin, kUnroll, kThreads, 1, T><<<grid_for(n, kThreads, 16, 8), kThreads, 0, st>>>(x, n, bin, hist);
        return (int)cudaGetLastError();
    }
    const int grid = hist_grid(n, (int)bins);
    histogram_kernel<0, Bin, 2, kHistThreads, 2, T><<<grid * 2 > sm_count() * 2 ? sm_count() * 2 : grid * 2, kHistThreads,
                                                      (size_t)(bins + 1) * sizeof(int), st>>>(x, n, bin, hist);
    return (int)cudaGetLastError();
}

// Two CTAs per SM when the ring, the prefix and the Op's shared memory allow it; each CTA should own >= 64 Ki elements before it pays
// for its per-tensor set-up and publishes.  Rejects tables whose shared memory exceeds the device's opt-in limit.
template <class Op, class T>
static int launch_multi_stream(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, const typename Op::Args &args, int op_param,
                               cudaStream_t st) {
    const size_t smem = ring_op_offset(count) + Op::smem_bytes(op_param);
    int dev = 0, limit = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return (int)cudaGetLastError();
    if (smem > (size_t)limit) return (int)cudaErrorInvalidValue;
    // the > 48 KB opt-in is per device, not per process: set it on every launch
    if (cudaFuncSetAttribute(multi_stream_kernel<Op, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return (int)cudaGetLastError();
    int resident = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, multi_stream_kernel<Op, T>, kRingThreads, smem) != cudaSuccess)
        return (int)cudaGetLastError();
    if (resident < 1) resident = 1;
    if (resident > 2) resident = 2;
    int64_t g = ((int64_t)count * max_n + 65535) / 65536;
    if (g > (int64_t)sm_count() * resident) g = (int64_t)sm_count() * resident;
    if (g < 1) g = 1;
    multi_stream_kernel<Op, T><<<(int)g, kRingThreads, smem, st>>>(descs, count, args);
    return (int)cudaGetLastError();
}

}  // namespace ppqb

using namespace ppqb;

extern "C" {

int ppq_b200_minmax_init(float *mins, float *maxs, int64_t count, void *stream) {
    if (count <= 0 || (!mins && !maxs)) return (int)cudaErrorInvalidValue;
    minmax_init_kernel<<<(int)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(mins, maxs, count);
    return (int)cudaGetLastError();
}

int ppq_b200_minmax_t_dt(const void *x, int dtype, int64_t n, float *minmax, void *stream) {
    if (!valid_dtype(dtype) || n <= 0 || !x || !minmax) return (int)cudaErrorInvalidValue;
    return with_elem_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        const int grid = grid_for((n + 16 / sizeof(T) - 1) / (16 / sizeof(T)), kThreads, kUnroll * 4, 8);
        minmax_t_kernel<T><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const T *)x, n, minmax);
        return (int)cudaGetLastError();
    });
}

int ppq_b200_minmax_t(const float *x, int64_t n, float *minmax, void *stream) {
    return ppq_b200_minmax_t_dt(x, PPQ_B200_F32, n, minmax, stream);
}

int ppq_b200_minmax_c_dt(const void *x, int dtype, int64_t n, int64_t epc, int C, float *mins, float *maxs, void *stream) {
    if (!valid_dtype(dtype) || n <= 0 || epc <= 0 || C <= 0 || !x || !mins || !maxs || n % epc != 0) return (int)cudaErrorInvalidValue;
    const int64_t rows = n / epc;
    const int64_t chunks = (epc + kRowChunk - 1) / kRowChunk;
    if (chunks > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    const int64_t items = rows * chunks;
    int64_t grid = (items + (kThreads / 32) - 1) / (kThreads / 32);
    if (grid > (int64_t)sm_count() * 8) grid = (int64_t)sm_count() * 8;
    return with_elem_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        minmax_c_kernel<T><<<(int)grid, kThreads, 0, (cudaStream_t)stream>>>((const T *)x, rows, epc, C, chunks, FastDiv((uint32_t)chunks),
                                                                             FastDiv((uint32_t)C), mins, maxs);
        return (int)cudaGetLastError();
    });
}

int ppq_b200_minmax_c(const float *x, int64_t n, int64_t epc, int C, float *mins, float *maxs, void *stream) {
    return ppq_b200_minmax_c_dt(x, PPQ_B200_F32, n, epc, C, mins, maxs, stream);
}

int ppq_b200_histogram_t(const float *x, int64_t n, float hist_scale, int clip_outliers, int32_t *hist, int64_t bins, void *stream) {
    if (n <= 0 || !x || !hist || bins <= 0 || bins > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    return launch_hist<SymBin>(x, n, BinParams{hist_scale, 0.f, (int)bins, clip_outliers}, bins, hist, (cudaStream_t)stream);
}

int ppq_b200_histogram_asym_t_dt(const void *x, int dtype, int64_t n, float vmin, float vmax, int clip_outliers, int32_t *hist, int64_t bins,
                                 void *stream) {
    if (!valid_dtype(dtype) || n <= 0 || !x || !hist || bins <= 0 || bins > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    const BinParams bp{vmin, vmax, (int)bins, clip_outliers};
    if (dtype == PPQ_B200_F32) return launch_hist<AsymBin>((const float *)x, n, bp, bins, hist, (cudaStream_t)stream);
    return with_half_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        return launch_hist_half<AsymBin>((const T *)x, n, bp, bins, hist, (cudaStream_t)stream);
    });
}

int ppq_b200_histogram_asym_t(const float *x, int64_t n, float vmin, float vmax, int clip_outliers, int32_t *hist, int64_t bins,
                              void *stream) {
    return ppq_b200_histogram_asym_t_dt(x, PPQ_B200_F32, n, vmin, vmax, clip_outliers, hist, bins, stream);
}

int ppq_b200_histogram_t_dscale_dt(const void *x, int dtype, int64_t n, const float *hist_scale_dev, int clip_outliers, int32_t *hist,
                                   int64_t bins, void *stream) {
    if (!valid_dtype(dtype) || n <= 0 || !x || !hist || !hist_scale_dev || bins <= 0 || bins > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
    return with_elem_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        if (bins > kMaxSmemBins) {                 // the private bins do not fit: count with global atomics, as launch_hist does for Histogram_T
            histogram_dscale_kernel<3, kThreads, 1, T><<<grid_for(n, kThreads, 16, 8), kThreads, 0, (cudaStream_t)stream>>>(
                (const T *)x, n, hist_scale_dev, clip_outliers, (int)bins, hist);
            return (int)cudaGetLastError();
        }
        const int grid = hist_grid(n, (int)bins) * 2 > sm_count() * 2 ? sm_count() * 2 : hist_grid(n, (int)bins) * 2;
        histogram_dscale_kernel<0, kHistThreads, 2, T><<<grid, kHistThreads, (size_t)(bins + 1) * sizeof(int), (cudaStream_t)stream>>>(
            (const T *)x, n, hist_scale_dev, clip_outliers, (int)bins, hist);
        return (int)cudaGetLastError();
    });
}

int ppq_b200_histogram_t_dscale(const float *x, int64_t n, const float *hist_scale_dev, int clip_outliers, int32_t *hist,
                                int64_t bins, void *stream) {
    return ppq_b200_histogram_t_dscale_dt(x, PPQ_B200_F32, n, hist_scale_dev, clip_outliers, hist, bins, stream);
}

int ppq_b200_histogram_c(const float *x, int64_t n, int64_t epc, int C, float hist_scale, int clip_outliers, int32_t *hist,
                         int64_t bins, void *stream) {
    if (n <= 0 || epc <= 0 || C <= 0 || !x || !hist || bins <= 0 || bins > kMaxSmemBins || n % epc != 0)
        return (int)cudaErrorInvalidValue;
    const int64_t rows = n / epc;
    const int64_t chunk = (int64_t)bins * 8 > 32768 ? (int64_t)bins * 8 : 32768;
    const int64_t chunks = (epc + chunk - 1) / chunk;
    const int64_t items = rows * chunks;
    const int grid = (int)(items < (int64_t)sm_count() * 8 ? items : (int64_t)sm_count() * 8);
    histogram_c_kernel<0><<<grid, kThreads, (size_t)(bins + 1) * sizeof(int), (cudaStream_t)stream>>>(
        x, rows, epc, C, chunk, chunks, hist_scale, clip_outliers, (int)bins, hist);
    return (int)cudaGetLastError();
}

int ppq_b200_multi_minmax_t_dt(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, int dtype, float *minmax_arena, void *stream) {
    if (!valid_dtype(dtype) || count <= 0 || max_n <= 0 || !descs || !minmax_arena) return (int)cudaErrorInvalidValue;
    return with_elem_type(dtype, [&](auto tag) {
        return launch_multi_stream<MinMaxOp, decltype(tag)>(descs, count, max_n, MinMaxOp::Args{minmax_arena}, 0, (cudaStream_t)stream);
    });
}

int ppq_b200_multi_minmax_t(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, float *minmax_arena, void *stream) {
    return ppq_b200_multi_minmax_t_dt(descs, count, max_n, PPQ_B200_F32, minmax_arena, stream);
}

int ppq_b200_multi_histogram_t_dt(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, int dtype, const float *hist_scale_arena,
                                  int clip_outliers, int32_t *hist_arena, int64_t bins, void *stream) {
    if (!valid_dtype(dtype) || count <= 0 || max_n <= 0 || !descs || !hist_scale_arena || !hist_arena || bins <= 0 || bins > kMaxSmemBins)
        return (int)cudaErrorInvalidValue;
    return with_elem_type(dtype, [&](auto tag) {
        return launch_multi_stream<HistOp, decltype(tag)>(descs, count, max_n, HistOp::Args{hist_scale_arena, hist_arena, (int)bins, clip_outliers},
                                                          (int)bins, (cudaStream_t)stream);
    });
}

int ppq_b200_multi_histogram_t(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, const float *hist_scale_arena,
                               int clip_outliers, int32_t *hist_arena, int64_t bins, void *stream) {
    return ppq_b200_multi_histogram_t_dt(descs, count, max_n, PPQ_B200_F32, hist_scale_arena, clip_outliers, hist_arena, bins, stream);
}

}  // extern "C"
