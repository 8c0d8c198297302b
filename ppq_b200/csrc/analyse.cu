// analyse.cu -- the paired-moment kernel behind layerwise_error_analyse (ppq_b200/executor.py).
//
//   ppq_b200_multi_paired_moments[_dt]   for every (prediction, reference) pair of a table and every sample row of it, the four fp64 sums
//                                        {sum (p - r)^2, sum r^2, sum p^2, sum p * r}
//
// Those four sums give the three measures of the reference's analysis (ppq/quantization/measure/norm.py:3-99, measure/cosine.py:6-28):
// snr = sum (p - r)^2 / (sum r^2 + 1e-7), mse = sum (p - r)^2 / D, cosine = sum p r / (|p| |r|).  Every input byte is read once (8 B per
// element pair in fp32, 4 B in fp16 / bf16) with 16-byte streaming loads; the result is O(rows).
//
// Numerics.  p, r are upcast exactly to fp64; p^2, r^2 and p r are exact in fp64 and enter the sums through one fused multiply-add each, so
// the only roundings of those three sums are the additions.  p - r is the fp64 difference of the upcasts (exact unless the exponents of p
// and r are more than 29 apart) and is squared inside the fused multiply-add, so sum (p - r)^2 carries at most two more roundings per term.
// sum (p - r)^2 is accumulated as such, never as sum p^2 - 2 sum p r + sum r^2 (cancellation).
//
// Work split and determinism.  A row is cut into chunks of kChunk element pairs; one CTA reduces one chunk (each thread its own elements in a
// fixed order, then a fixed shuffle tree) into a slot of the workspace, and a second kernel adds a row's chunk slots in chunk order.  The
// assignment of elements to threads depends only on the row's length and the alignment of its two pointers, so a launch is bit-identical from
// run to run and under CUDA-graph replay; nothing depends on the order in which CTAs finish.  The longest addition chain of a launch is at
// most 74 + ceil(row_len / kChunk) additions: 66 per thread (a head element, 64 vector or strided elements, a tail element), 5 + 3
// in the CTA's shuffle trees, then the chunk slots of the row one after another.
#include "common.cuh"
#include "half.cuh"
#include "../../include/ppq_b200.h"

namespace ppqb {

constexpr int kPmThreads = 256;
constexpr int kPmUnroll = 4;
constexpr int64_t kChunk = 16384;                 // element pairs per CTA work item: 128 KB of fp32 input, 64 KB of fp16 / bf16
constexpr int kPmMaxCount = 2048;                 // descriptors per launch: two (count + 1) x int64 prefixes in 32 KB of shared memory

struct Moments {
    double d2, r2, p2, pr;
    __device__ __forceinline__ Moments() : d2(0.0), r2(0.0), p2(0.0), pr(0.0) {}
    __device__ __forceinline__ void add(float p, float r) {
        const double pd = (double)p, rd = (double)r, d = __dsub_rn(pd, rd);
        d2 = __fma_rn(d, d, d2);
        r2 = __fma_rn(rd, rd, r2);
        p2 = __fma_rn(pd, pd, p2);
        pr = __fma_rn(pd, rd, pr);
    }
    __device__ __forceinline__ void add4(const float4 &p, const float4 &r) { add(p.x, r.x); add(p.y, r.y); add(p.z, r.z); add(p.w, r.w); }
    __device__ __forceinline__ void merge(const Moments &o) {
        d2 = __dadd_rn(d2, o.d2); r2 = __dadd_rn(r2, o.r2); p2 = __dadd_rn(p2, o.p2); pr = __dadd_rn(pr, o.pr);
    }
    __device__ __forceinline__ void shfl_merge(int lane_mask) {
        Moments o;
        o.d2 = __shfl_xor_sync(0xffffffffu, d2, lane_mask); o.r2 = __shfl_xor_sync(0xffffffffu, r2, lane_mask);
        o.p2 = __shfl_xor_sync(0xffffffffu, p2, lane_mask); o.pr = __shfl_xor_sync(0xffffffffu, pr, lane_mask);
        merge(o);
    }
};

__device__ __forceinline__ float ld1(const float *p) { return ld_stream1(p); }
template <class T> __device__ __forceinline__ float ld1(const T *p) { return ld_stream1_f(p); }

// One chunk [0, len) of a pair.  16-byte vectors when both pointers share their offset within 16 bytes (the head before the first boundary
// and the ragged tail element by element), element by element otherwise.  Thread t owns a fixed set of elements: head element t, vectors
// t, t + kPmThreads, ... and tail element t.
template <class T>
__device__ __forceinline__ void chunk_moments(const T *__restrict__ p, const T *__restrict__ r, int64_t len, Moments &m) {
    constexpr int kVec = 16 / sizeof(T);
    const int t = threadIdx.x;
    const uintptr_t pa = reinterpret_cast<uintptr_t>(p), ra = reinterpret_cast<uintptr_t>(r);
    if (((pa ^ ra) & 15u) != 0) {
        for (int64_t i = t; i < len; i += kPmThreads) m.add(ld1(p + i), ld1(r + i));
        return;
    }
    int64_t head = (int64_t)(((16u - (uint32_t)(pa & 15u)) & 15u) / sizeof(T));
    if (head > len) head = len;
    if (t < head) m.add(ld1(p + t), ld1(r + t));
    const int64_t nv = (len - head) / kVec;
    const uint4 *pv = reinterpret_cast<const uint4 *>(p + head), *rv = reinterpret_cast<const uint4 *>(r + head);
    int64_t v = t;
    for (; v + (kPmUnroll - 1) * kPmThreads < nv; v += kPmUnroll * kPmThreads) {
        uint4 a[kPmUnroll], b[kPmUnroll];
#pragma unroll
        for (int u = 0; u < kPmUnroll; u++) { a[u] = ld_stream_u4(pv + v + u * kPmThreads); b[u] = ld_stream_u4(rv + v + u * kPmThreads); }
#pragma unroll
        for (int u = 0; u < kPmUnroll; u++) {
            if constexpr (sizeof(T) == 4) {
                m.add4(make_float4(__uint_as_float(a[u].x), __uint_as_float(a[u].y), __uint_as_float(a[u].z), __uint_as_float(a[u].w)),
                       make_float4(__uint_as_float(b[u].x), __uint_as_float(b[u].y), __uint_as_float(b[u].z), __uint_as_float(b[u].w)));
            } else {
                float4 p0, p1, r0, r1;
                unpack8<T>(a[u], p0, p1); unpack8<T>(b[u], r0, r1);
                m.add4(p0, r0); m.add4(p1, r1);
            }
        }
    }
    for (; v < nv; v += kPmThreads) {
        const uint4 a = ld_stream_u4(pv + v), b = ld_stream_u4(rv + v);
        if constexpr (sizeof(T) == 4) {
            m.add4(make_float4(__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(a.w)),
                   make_float4(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(b.w)));
        } else {
            float4 p0, p1, r0, r1;
            unpack8<T>(a, p0, p1); unpack8<T>(b, r0, r1);
            m.add4(p0, r0); m.add4(p1, r1);
        }
    }
    const int64_t tail0 = head + nv * kVec;
    if (tail0 + t < len) m.add(ld1(p + tail0 + t), ld1(r + tail0 + t));
}

__device__ __forceinline__ int64_t chunks_of(int64_t row_len) { return (row_len + kChunk - 1) / kChunk; }

// Both kernels start by reading the table into two exclusive prefixes in shared memory: chunk_pre[i] = work items of descriptors < i,
// row_pre[i] = rows of descriptors < i.  Returns false (for the whole CTA) when the table is malformed: a negative or oversized field, an
// output row range outside [0, total_rows), or more work items than the workspace holds.
__device__ bool read_table(const ppq_b200_pair_desc *__restrict__ descs, int count, int64_t total_rows, int64_t cap, int64_t *chunk_pre,
                           int64_t *row_pre) {
    __shared__ int bad;
    if (threadIdx.x == 0) { bad = 0; chunk_pre[0] = 0; row_pre[0] = 0; }
    __syncthreads();
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
        const int64_t rows = descs[i].rows, len = descs[i].row_len, row0 = descs[i].out_row0;
        const bool ok = rows >= 0 && rows <= (1LL << 31) && len >= 0 && len <= (1LL << 40) && row0 >= 0 && row0 <= total_rows - rows &&
                        (rows == 0 || len == 0 || (descs[i].pred != nullptr && descs[i].real != nullptr));
        if (!ok) bad = 1;
        chunk_pre[i + 1] = ok ? rows * chunks_of(len) : 0;
        row_pre[i + 1] = ok ? rows : 0;
    }
    __syncthreads();
    if (threadIdx.x < 32) {                                           // inclusive scan of entries 1..count, 32 at a time
        const int lane = threadIdx.x;
        int64_t carry_c = 0, carry_r = 0;
        for (int base = 1; base <= count; base += 32) {
            const int i = base + lane;
            int64_t c = i <= count ? chunk_pre[i] : 0, r = i <= count ? row_pre[i] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int64_t cu = __shfl_up_sync(0xffffffffu, c, o), ru = __shfl_up_sync(0xffffffffu, r, o);
                if (lane >= o) { c += cu; r += ru; }
            }
            if (i <= count) { chunk_pre[i] = c + carry_c; row_pre[i] = r + carry_r; }
            carry_c += __shfl_sync(0xffffffffu, c, 31);
            carry_r += __shfl_sync(0xffffffffu, r, 31);
        }
        if (lane == 0 && carry_c > cap) bad = 1;
    }
    __syncthreads();
    return bad == 0;
}

// largest i in [0, count) with pre[i] <= w (descriptors without work share their prefix value with the next one)
__device__ __forceinline__ int find_desc(const int64_t *pre, int count, int64_t w) {
    int lo = 0, hi = count - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (pre[mid] <= w) lo = mid; else hi = mid - 1;
    }
    return lo;
}

template <class T>
__global__ void __launch_bounds__(kPmThreads) paired_moments_chunk_kernel(const ppq_b200_pair_desc *__restrict__ descs, int count,
                                                                          int64_t total_rows, int64_t cap, double *__restrict__ slots) {
    extern __shared__ int64_t pm_smem[];
    int64_t *chunk_pre = pm_smem, *row_pre = pm_smem + count + 1;
    if (!read_table(descs, count, total_rows, cap, chunk_pre, row_pre)) return;
    __shared__ double2 warp_part[kPmThreads / 32][2];
    const int64_t items = chunk_pre[count];
    for (int64_t w = blockIdx.x; w < items; w += gridDim.x) {
        const int d = find_desc(chunk_pre, count, w);
        const int64_t len = descs[d].row_len, cpr = chunks_of(len), local = w - chunk_pre[d];
        const int64_t row = local / cpr, c = local - row * cpr;
        const int64_t first = row * len + c * kChunk;
        const int64_t n = len - c * kChunk < kChunk ? len - c * kChunk : kChunk;
        Moments m;
        chunk_moments<T>(static_cast<const T *>(descs[d].pred) + first, static_cast<const T *>(descs[d].real) + first, n, m);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m.shfl_merge(o);
        const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
        if (lane == 0) { warp_part[wid][0] = make_double2(m.d2, m.r2); warp_part[wid][1] = make_double2(m.p2, m.pr); }
        __syncthreads();
        if (wid == 0) {
            Moments s;
            if (lane < kPmThreads / 32) {
                s.d2 = warp_part[lane][0].x; s.r2 = warp_part[lane][0].y; s.p2 = warp_part[lane][1].x; s.pr = warp_part[lane][1].y;
            }
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) s.shfl_merge(o);
            if (lane == 0) {
                double2 *dst = reinterpret_cast<double2 *>(slots + 4 * w);
                dst[0] = make_double2(s.d2, s.r2);
                dst[1] = make_double2(s.p2, s.pr);
            }
        }
        __syncthreads();
    }
}

// One thread per row: the row's chunk slots added in chunk order.  A malformed table writes NaN into every one of the total_rows rows.
__global__ void __launch_bounds__(kPmThreads) paired_moments_row_kernel(const ppq_b200_pair_desc *__restrict__ descs, int count,
                                                                        int64_t total_rows, int64_t cap, const double *__restrict__ slots,
                                                                        double *__restrict__ out) {
    extern __shared__ int64_t pm_smem[];
    int64_t *chunk_pre = pm_smem, *row_pre = pm_smem + count + 1;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (!read_table(descs, count, total_rows, cap, chunk_pre, row_pre)) {
        const double nan = __longlong_as_double(0x7FF8000000000000LL);
        for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total_rows; g += stride)
            { reinterpret_cast<double2 *>(out)[2 * g] = make_double2(nan, nan); reinterpret_cast<double2 *>(out)[2 * g + 1] = make_double2(nan, nan); }
        return;
    }
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < row_pre[count]; g += stride) {
        const int d = find_desc(row_pre, count, g);
        const int64_t r = g - row_pre[d], cpr = chunks_of(descs[d].row_len);
        const double *s = slots + 4 * (chunk_pre[d] + r * cpr);
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
        for (int64_t c = 0; c < cpr; c++, s += 4) {
            if (c == 0) { a0 = s[0]; a1 = s[1]; a2 = s[2]; a3 = s[3]; }
            else { a0 = __dadd_rn(a0, s[0]); a1 = __dadd_rn(a1, s[1]); a2 = __dadd_rn(a2, s[2]); a3 = __dadd_rn(a3, s[3]); }
        }
        double2 *dst = reinterpret_cast<double2 *>(out) + 2 * (descs[d].out_row0 + r);
        dst[0] = make_double2(a0, a1);
        dst[1] = make_double2(a2, a3);
    }
}

static int64_t workspace_slots(int64_t total_rows, int64_t total_elems) { return total_rows + total_elems / kChunk; }

}  // namespace ppqb

using namespace ppqb;

extern "C" {

int64_t ppq_b200_multi_paired_moments_workspace_bytes(int64_t total_rows, int64_t total_elems) {
    if (total_rows < 0 || total_elems < 0) return 0;
    return workspace_slots(total_rows, total_elems) * 4 * (int64_t)sizeof(double);
}

int ppq_b200_multi_paired_moments_dt(const ppq_b200_pair_desc *descs, int count, int64_t total_rows, int64_t total_elems, int dtype,
                                     double *out, void *workspace, void *stream) {
    if (!valid_dtype(dtype) || count < 0 || count > kPmMaxCount || total_rows < 0 || total_elems < 0) return (int)cudaErrorInvalidValue;
    if (count == 0 || total_rows == 0) return 0;                       // nothing to write
    if (!descs || !out || !workspace) return (int)cudaErrorInvalidValue;
    if (((uintptr_t)out & 15u) != 0 || ((uintptr_t)workspace & 15u) != 0) return (int)cudaErrorInvalidValue;
    const int64_t cap = workspace_slots(total_rows, total_elems);
    const size_t smem = (size_t)2 * (count + 1) * sizeof(int64_t);
    const cudaStream_t st = (cudaStream_t)stream;
    double *slots = static_cast<double *>(workspace);
    const int rc = with_elem_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        int64_t g = cap < (int64_t)sm_count() * 4 ? cap : (int64_t)sm_count() * 4;
        if (g < 1) g = 1;
        paired_moments_chunk_kernel<T><<<(int)g, kPmThreads, smem, st>>>(descs, count, total_rows, cap, slots);
        return (int)cudaGetLastError();
    });
    if (rc != 0) return rc;
    int64_t g2 = (total_rows + kPmThreads - 1) / kPmThreads;
    if (g2 > (int64_t)sm_count() * 8) g2 = (int64_t)sm_count() * 8;
    paired_moments_row_kernel<<<(int)g2, kPmThreads, smem, st>>>(descs, count, total_rows, cap, slots, out);
    return (int)cudaGetLastError();
}

int ppq_b200_multi_paired_moments(const ppq_b200_pair_desc *descs, int count, int64_t total_rows, int64_t total_elems, double *out,
                                  void *workspace, void *stream) {
    return ppq_b200_multi_paired_moments_dt(descs, count, total_rows, total_elems, PPQ_B200_F32, out, workspace, stream);
}

}  // extern "C"
