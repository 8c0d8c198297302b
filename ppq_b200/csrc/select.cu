// select.cu -- exact order statistics without sorting (sm_90a), behind the C ABI of include/ppq_b200.h.
//
//   ppq_b200_quantile_t         replaces Quantile_T (/root/reference/ppq/csrc/cuda/sort.cu:6-20, 42-59): the reference clones the
//                               tensor, thrust::sort's the clone and reads sorted[clip(rn(n*q))] and sorted[clip(rn(n*(1-q)))].
//   ppq_b200_multi_quantile_t   the same for a table of tensors in one launch per pass (the percentile observer of the calibration arena:
//                               TorchPercentileObserver, ppq/quantization/observer/range.py:312-403, is the reference's default observer).
//   ppq_b200_isotone_t          replaces Isotone_T (sort.cu:23-40, 61-73): sorted[n-1], sorted[n-2], sorted[0], sorted[1].
//
// MSD radix *select* on the order-preserving 32-bit key of each float (the order thrust's radix sort uses:
// -NaN < -inf < ... < -0 < +0 < ... < +inf < +NaN, except that thrust gives the two zeros one key, see order_key), digits of 11 + 11 + 10
// bits, both requested ranks resolved together.
//
//   pass 0   streams the tensor once (4 B/element): 2048-bin histogram of the top digit, shared-memory privatised.  The scan that ends the
//            pass knows the population of the bucket each rank fell into.
//   pass 1   streams the tensor a second time and looks only at elements of the one or two selected buckets (a vector whose four elements
//            miss both prefixes costs one AND + three compares per element on the raw bits).  The requested ranks sit in the tails
//            (q = 0.9999), so a bucket normally holds ~1e-4 of the tensor: when it fits the workspace (`cap` keys) its keys are COMPACTED
//            (staged per CTA in shared memory, one global reservation per CTA) instead of histogrammed, and
//   finish   one CTA per rank selects among the few thousand compacted keys (L2-resident, KBs) -- no third pass over the tensor.
//            A bucket too big to compact (post-ReLU tensors: half of the elements are exactly 0) is refined by histogram as before, and
//            the min / max key of the bucket is tracked on the way: when they coincide the bucket is one repeated value and the rank is
//            resolved on the spot.  Only a big bucket with several distinct values needs pass 2 (launched always, returns at once when no
//            rank asks for it).
// Algorithmic traffic (SURVEY 8f-1): 4 B/element; this design moves 8 B/element (two streaming passes), the round-1 version 12.
// No allocation -- the caller provides the workspace.  The result is the identical element, bit for bit, except that a selected zero is
// reported with the sign its key order gives (-0.0 < +0.0), equal as a float to whichever zero the reference's sort left at that index.
#include "common.cuh"
#include "half.cuh"
#include "variants.h"
#include "../../include/ppq_b200.h"

namespace ppqb {

constexpr int kSelThreads = 1024;              // pass 0: two CTAs per SM
constexpr int kFilterThreads = 256;            // passes 1-2: six CTAs per SM
constexpr int kDigits = 2048;                  // 11-bit digits (the last level has 10 bits)
constexpr int kStage = kDigits;                // keys a CTA stages in shared memory per rank before its global reservation
constexpr unsigned kModeHist = 0, kModeCompact = 1, kModeDone = 2;
constexpr int64_t kDefaultCap = 1 << 18;       // single-tensor entry: 256 Ki keys per rank (2 MB of workspace)

struct SelectState {                           // one per tensor, in the caller's workspace
    unsigned long long hist[2][kDigits];       // per rank: digit histogram of the current pass
    unsigned int prefix[2];                    // key bits resolved so far (high bits); the full key once mode == done
    unsigned int mode[2];
    unsigned int shared;                       // both ranks are in the same bucket and mode: rank 1 reads rank 0's histogram / buffer
    unsigned int done;                         // CTAs that have flushed in the current pass (single-tensor path)
    unsigned int ccount[2];                    // keys in the compact buffers
    unsigned int cbuf[2];                      // which buffer holds rank r's candidates
    unsigned int clevel[2];                    // first unresolved level of the compacted keys
    unsigned int compacted[2];
    unsigned int kmin[2], kmax[2];             // min / max key seen in the bucket during a refining pass
    long long rank[2];                         // remaining rank inside the current bucket
    long long count[2];                        // population of the current bucket
    // speculation (table form with a `guess` buffer): candidates beyond last call's thresholds are compacted during pass 0
    unsigned int spec;                         // 1: this call speculates
    unsigned int g[2], k[2], d[2];             // thresholds {hi: key >= g[0], lo: key <= g[1]}, last call's selected keys, threshold margins
    unsigned int eqc[2];                       // candidates equal to k[r] (counted, not stored: post-ReLU tensors select an exact 0 among millions)
    unsigned int veq[2], vkey[2];              // for the finish: `veq` virtual copies of `vkey` belong to the compacted multiset of rank r
    unsigned int pad2_;
};
constexpr int kGuessWords = 8;                 // per slot: {g_hi, k_hi, d_hi, 0, g_lo, k_lo, d_lo, 0}
constexpr unsigned kSpecMarginInit = 1u << 19, kSpecMarginMin = 1u << 12, kSpecMarginMax = 1u << 24;

__host__ __device__ constexpr int level_shift(int level) { return level == 0 ? 21 : (level == 1 ? 10 : 0); }
__host__ __device__ constexpr uint32_t level_dmask(int level) { return level == 2 ? 0x3FFu : 0x7FFu; }
__host__ __device__ constexpr uint32_t level_pmask(int level) { return level == 0 ? 0u : (level == 1 ? 0xFFE00000u : 0xFFFFFC00u); }

// Order-preserving key: flip all bits of negative floats, only the sign bit of the others (an arithmetic shift + one LOP3 -- pass 0 is bound by
// the integer pipe, every instruction per element counts).  Total order: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN.  thrust's radix
// sort treats -0.0 and +0.0 as one key; here -0.0 sorts just below +0.0, so a selected zero may carry either sign -- equal as a float to whichever
// zero the reference's stable sort left at that index (the sign is not recoverable without sorting).
__device__ __forceinline__ uint32_t order_key(float v) {
    const uint32_t b = __float_as_uint(v);
    return b ^ ((uint32_t)((int32_t)b >> 31) | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// index arithmetic of _Quantile_T (sort.cu:13-19): int64 * float -> float, __float2int_rn (half-even, saturating), CLIP<int>(pos, 0, n - 1)
__device__ __forceinline__ long long quantile_rank(int64_t n, float frac) {
    int pos = __float2int_rn((float)n * frac);
    const int last = (int)(n - 1);
    pos = pos > last ? last : pos;
    return pos < 0 ? 0 : pos;
}

// Block-wide search of the bucket that contains rank k in a 2048-bin histogram (TPB threads, kDigits / TPB consecutive bins per thread, warp
// shuffles).  Exactly one (thread, bin) matches because k < total.  Results through shared memory; ends with a barrier.
template <int TPB, class Load>
__device__ __forceinline__ void block_pick(Load &&load, unsigned long long k, unsigned int *digit, unsigned long long *before_out, unsigned long long *cnt_out) {
    constexpr int D = kDigits / TPB;
    __shared__ unsigned long long warp_tot[TPB / 32];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    unsigned long long c[D], mine = 0;
#pragma unroll
    for (int j = 0; j < D; j++) { c[j] = load(D * t + j); mine += c[j]; }
    unsigned long long incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long up = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += up; }
    __syncthreads();                                                   // warp_tot may still be read by a previous call
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    unsigned long long before = incl - mine;
    for (int i = 0; i < w; i++) before += warp_tot[i];
#pragma unroll
    for (int j = 0; j < D; j++) {
        if (k >= before && k < before + c[j]) { *digit = (unsigned int)(D * t + j); *before_out = before; *cnt_out = c[j]; }
        before += c[j];
    }
    __syncthreads();
}

// ---- self-speculation: thresholds from a sample ------------------------------------------------------------------------------------------
// A cold call has no thresholds from a previous batch.  For a big tensor a small grid draws kSampleKeys elements (one per stride window, at a
// hashed offset inside the window so that no channel / row period can alias with the stride), the init CTA selects the j-th largest and j-th smallest sample
// exactly (three 11/11/10-bit rounds in shared memory) and uses them as this call's thresholds: the tail beyond the j-th largest of m samples
// holds Gamma(j) x n / m elements, so with j = max(12, 3 x need x m / n) it contains the `need` wanted elements with overwhelming probability and
// stays far below the compaction buffer.  Copies of the threshold key itself are only counted (k = g), which covers post-ReLU zeros and clipped
// maxima.  A wrong guess costs nothing but the sample: select_scan<0> then falls back to the regular passes.
constexpr int kSampleKeys = 16384;
constexpr int64_t kSampleMinElems = (int64_t)1 << 23;

__host__ __device__ inline long long sample_rank_from_end(long long need, int64_t n) {     // j
    const long long j = (3 * need * kSampleKeys + n - 1) / n;
    return j < 12 ? 12 : j;
}
__host__ __device__ inline bool sample_rank_ok(long long j, int64_t n, int64_t cap) {
    return j <= kSampleKeys / 4 && 3 * j * (n / kSampleKeys) <= 2 * cap;                   // mean tail x 1.5 fits the buffer
}

// both order statistics (ascending ranks rk[0], rk[1]) of the CTA's kSampleKeys keys (PER per thread, 1024 threads), exact
template <int PER>
__device__ __forceinline__ void cta_select_two(const uint32_t (&key)[PER], long long rk0, long long rk1, uint32_t *out0, uint32_t *out1) {
    __shared__ int sh[2][kDigits];
    __shared__ unsigned int s_digit;
    __shared__ unsigned long long s_before, s_cnt;
    uint32_t pre[2] = {0u, 0u};
    unsigned long long rk[2] = {(unsigned long long)rk0, (unsigned long long)rk1};
#pragma unroll
    for (int level = 0; level < 3; level++) {
        const int shift = level_shift(level);
        const uint32_t dmask = level_dmask(level), pmask = level_pmask(level);
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * kDigits; i += blockDim.x) (&sh[0][0])[i] = 0;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < PER; j++) {
            const uint32_t k = key[j];
            const int d = (int)((k >> shift) & dmask);
            if ((k & pmask) == pre[0]) atomicAdd(&sh[0][d], 1);
            if ((k & pmask) == pre[1]) atomicAdd(&sh[1][d], 1);
        }
        __syncthreads();
        for (int r = 0; r < 2; r++) {
            block_pick<1024>([&](int i) { return (unsigned long long)sh[r][i]; }, rk[r], &s_digit, &s_before, &s_cnt);
            pre[r] |= s_digit << shift;
            rk[r] -= s_before;
        }
    }
    *out0 = pre[0]; *out1 = pre[1];
}

// The sample itself is drawn by a grid of small CTAs (16 K scattered 32-byte sectors are ~25 us for one SM's miss queue and ~2 us for 64 SMs).
template <class T>
__global__ void __launch_bounds__(256)
select_sample_kernel(const T *__restrict__ x, int64_t n, uint32_t *__restrict__ keys) {
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    const int64_t stride = n / kSampleKeys;
    const int64_t off = (int64_t)((uint64_t)(i * 0x9E3779B1u) % (uint64_t)stride);
    keys[i] = order_key(to_f(__ldg(x + (int64_t)i * stride + off)));
}

// one CTA per tensor.  q_mode: ranks = {rn(n q), rn(n (1 - q))};  otherwise explicit ranks (isotone).  sample_keys != nullptr (single tensor,
// 1024 threads): thresholds from the sample unless the caller's guess already holds some.
__global__ void __launch_bounds__(1024)
select_init_kernel(SelectState *states, const ppq_b200_tensor_desc *descs, int64_t n_single, float q, int q_mode,
                   long long r0, long long r1, const uint32_t *__restrict__ guess = nullptr, const uint32_t *__restrict__ sample_keys = nullptr, int64_t cap = 0) {
    SelectState *st = states + blockIdx.x;
    for (int i = threadIdx.x; i < 2 * kDigits; i += blockDim.x) (&st->hist[0][0])[i] = 0ull;
    const int64_t n = descs ? descs[blockIdx.x].n : n_single;
    if (q_mode) { r0 = quantile_rank(n, q); r1 = quantile_rank(n, 1.0f - q); }
    const uint32_t *gw = guess ? guess + (descs ? (int64_t)descs[blockIdx.x].slot : 0) * kGuessWords : nullptr;
    uint32_t g_hi = 0xFFFFFFFFu, k_hi = 0xFFFFFFFFu, g_lo = 0u, k_lo = 0u, d_hi = kSpecMarginInit, d_lo = kSpecMarginInit;
    if (gw) { g_hi = gw[0]; k_hi = gw[1]; d_hi = gw[2]; g_lo = gw[4]; k_lo = gw[5]; d_lo = gw[6]; }
    unsigned int spec = guess ? 1u : 0u;
    if (sample_keys && g_hi == 0xFFFFFFFFu && g_lo == 0u) {            // uniform over the CTA: nothing guessed yet
        constexpr int PER = kSampleKeys / 1024;
        uint32_t key[PER];
#pragma unroll
        for (int j = 0; j < PER; j++) key[j] = __ldcg(sample_keys + j * 1024 + threadIdx.x);
        const long long j_hi = sample_rank_from_end(n - r0, n), j_lo = sample_rank_from_end(r1 + 1, n);
        const bool ok_hi = sample_rank_ok(j_hi, n, cap), ok_lo = sample_rank_ok(j_lo, n, cap);
        uint32_t s_hi, s_lo;
        cta_select_two<PER>(key, ok_hi ? kSampleKeys - j_hi : 0, ok_lo ? j_lo - 1 : 0, &s_hi, &s_lo);
        if (ok_hi) g_hi = k_hi = s_hi;
        if (ok_lo) g_lo = k_lo = s_lo;
        spec = 1u;
    }
    if (threadIdx.x == 0) {
        st->prefix[0] = st->prefix[1] = 0u; st->mode[0] = st->mode[1] = kModeHist; st->shared = 1u; st->done = 0u;
        st->ccount[0] = st->ccount[1] = 0u; st->cbuf[0] = 0u; st->cbuf[1] = 1u; st->clevel[0] = st->clevel[1] = 0u;
        st->compacted[0] = st->compacted[1] = 0u; st->kmin[0] = st->kmin[1] = 0xFFFFFFFFu; st->kmax[0] = st->kmax[1] = 0u;
        st->rank[0] = r0; st->rank[1] = r1; st->count[0] = st->count[1] = n;
        st->spec = spec; st->eqc[0] = st->eqc[1] = 0u; st->veq[0] = st->veq[1] = 0u; st->vkey[0] = st->vkey[1] = 0u;
        st->g[0] = g_hi; st->k[0] = k_hi; st->d[0] = d_hi; st->g[1] = g_lo; st->k[1] = k_lo; st->d[1] = d_lo;
    }
}

// Resolve a pass for one tensor: run by the last CTA to finish its part of that tensor (ticket counter), in both the single-tensor and the table form.
template <int LEVEL, int TPB>
__device__ __noinline__ void select_scan(SelectState *st, long long cap) {
    __shared__ unsigned int s_digit;
    __shared__ unsigned long long s_before, s_cnt;
    const int t = threadIdx.x;
    const bool shared_in = st->shared != 0;
    if (LEVEL == 0 && st->spec) {
        // Did the candidates compacted during pass 0 (keys beyond last call's thresholds; copies of last call's key only counted) contain
        // the requested order statistic?  hi: the n - r0 largest elements must all be candidates; lo: the r1 + 1 smallest ones.
        __syncthreads();
        if (t == 0) {
            const long long n = st->count[0];
            for (int r = 0; r < 2; r++) {
                const long long app = (long long)__ldcg(&st->ccount[r]), eq = (long long)__ldcg(&st->eqc[r]), cnt = app + eq;
                const long long need = r == 0 ? n - st->rank[0] : st->rank[1] + 1;
                unsigned int d = st->d[r];
                if (app <= cap && cnt >= need) {
                    st->mode[r] = kModeCompact; st->compacted[r] = 1u; st->clevel[r] = 0u; st->prefix[r] = 0u; st->cbuf[r] = (unsigned)r;
                    st->rank[r] = r == 0 ? cnt - need : st->rank[1];
                    st->veq[r] = (unsigned)eq; st->vkey[r] = st->k[r];
                    if (cnt > 4 * need + 64 && d > kSpecMarginMin) d >>= 1;          // far more candidates than needed: tighten the threshold
                } else {
                    st->ccount[r] = 0u;                                              // the buffer goes back to the regular compaction of pass 1
                    const bool first_call = r == 0 ? st->g[0] == 0xFFFFFFFFu : st->g[1] == 0u;   // nothing was guessed yet: no verdict on the margin
                    if (app > cap) { if (d > kSpecMarginMin) d >>= 1; }
                    else if (!first_call && d < kSpecMarginMax) d <<= 1;             // too few candidates: the distribution moved, widen
                }
                st->d[r] = d;
            }
        }
        __syncthreads();
    }
    for (int r = 0; r < 2; r++) {
        const int src = (r == 1 && shared_in) ? 0 : r;
        const unsigned int mode = st->mode[r];                          // uniform
        if (mode == kModeDone) continue;
        if (mode == kModeCompact) { if (t == 0) st->compacted[r] = 1u; continue; }
        const unsigned int kmin = __ldcg(&st->kmin[src]), kmax = __ldcg(&st->kmax[src]);
        if (LEVEL > 0 && kmin == kmax) {                               // the whole bucket is one repeated value
            __syncthreads();
            if (t == 0) { st->prefix[r] = kmin; st->mode[r] = kModeDone; }
            continue;
        }
        // other CTAs' atomics wrote the histogram: read it at L2
        const unsigned long long *h = st->hist[src];
        block_pick<TPB>([&](int i) { return __ldcg(h + i); }, (unsigned long long)st->rank[r], &s_digit, &s_before, &s_cnt);
        if (t == 0) {
            st->prefix[r] |= s_digit << level_shift(LEVEL);
            st->rank[r] -= (long long)s_before;
            st->count[r] = (long long)s_cnt;
            if (LEVEL == 2) st->mode[r] = kModeDone;
            else if ((long long)s_cnt <= cap) { st->mode[r] = kModeCompact; st->clevel[r] = LEVEL + 1; }
        }
        __syncthreads();
    }
    for (int i = t; i < 2 * kDigits; i += TPB) (&st->hist[0][0])[i] = 0ull;
    if (t == 0) {
        const bool same = st->prefix[0] == st->prefix[1] && st->mode[0] == st->mode[1] && st->mode[0] != kModeDone &&
                          !st->compacted[0] && !st->compacted[1];
        st->shared = same ? 1u : 0u;
        if (st->mode[0] == kModeCompact && !st->compacted[0]) st->cbuf[0] = 0u;
        if (st->mode[1] == kModeCompact && !st->compacted[1]) st->cbuf[1] = same ? 0u : 1u;
        st->kmin[0] = st->kmin[1] = 0xFFFFFFFFu; st->kmax[0] = st->kmax[1] = 0u;
        st->done = 0u;
    }
}

// Streams elements [a, b) of x (a multiple of 4 when x is 16-byte aligned) through `visit4` / `visit1`.
template <int U, bool SEGMENTS, class F4, class F1>
__device__ __forceinline__ void stream_range(const float *__restrict__ x, int64_t a, int64_t b, int64_t first, int64_t stride, F4 &&visit4, F1 &&visit1) {
    const float *p = x + a;
    const int64_t n = b - a;
    if ((reinterpret_cast<uintptr_t>(p) & 15u) == 0) {
        const int64_t n4 = n >> 2;
        const float4 *x4 = reinterpret_cast<const float4 *>(p);
        if (!SEGMENTS) {
            for (int64_t i = first; i < n4; i += U * stride) {
                float4 v[U];
#pragma unroll
                for (int j = 0; j < U; j++) if (i + j * stride < n4) v[j] = ld_stream4(x4 + i + j * stride);
#pragma unroll
                for (int j = 0; j < U; j++) if (i + j * stride < n4) visit4(v[j]);
            }
        } else {                                                       // warp-contiguous segments of 32 lanes x U vectors (2 KB)
            const int64_t lane = first & 31, warps = stride >> 5;
            for (int64_t sg = first >> 5; sg * (32 * U) < n4; sg += warps) {
                const int64_t base = sg * (32 * U) + lane;
                float4 v[U];
#pragma unroll
                for (int j = 0; j < U; j++) if (base + j * 32 < n4) v[j] = ld_stream4(x4 + base + j * 32);
#pragma unroll
                for (int j = 0; j < U; j++) if (base + j * 32 < n4) visit4(v[j]);
            }
        }
        const int64_t t = (n4 << 2) + first;
        if (t < n) visit1(p[t]);
    } else {
        for (int64_t i = first; i < n; i += stride) visit1(ld_stream1(p + i));
    }
}

// fp16 / bf16: 16-byte loads of 8 elements, visited as two float4 of their exact upcasts; the <= 7 + 7 elements before the first 16-byte
// boundary and after the last whole vector go one per thread to the first threads of the group.
template <int U, bool SEGMENTS, class T, class F4, class F1, std::enable_if_t<is_half_t<T>::value, int> = 0>
__device__ __forceinline__ void stream_range(const T *__restrict__ x, int64_t a, int64_t b, int64_t first, int64_t stride, F4 &&visit4, F1 &&visit1) {
    const T *p = x + a;
    const int64_t n = b - a;
    const int64_t head = min(n, head_elems(p));
    const int64_t nv = (n - head) >> 3, tail0 = head + (nv << 3);
    const uint4 *x8 = reinterpret_cast<const uint4 *>(p + head);
    auto visit8 = [&](const uint4 &r) { float4 lo, hi; unpack8<T>(r, lo, hi); visit4(lo); visit4(hi); };
    if (!SEGMENTS) {
        for (int64_t i = first; i < nv; i += U * stride) {
            uint4 v[U];
#pragma unroll
            for (int j = 0; j < U; j++) if (i + j * stride < nv) v[j] = ld_stream_u4(x8 + i + j * stride);
#pragma unroll
            for (int j = 0; j < U; j++) if (i + j * stride < nv) visit8(v[j]);
        }
    } else {
        const int64_t lane = first & 31, warps = stride >> 5;
        for (int64_t sg = first >> 5; sg * (32 * U) < nv; sg += warps) {
            const int64_t base = sg * (32 * U) + lane;
            uint4 v[U];
#pragma unroll
            for (int j = 0; j < U; j++) if (base + j * 32 < nv) v[j] = ld_stream_u4(x8 + base + j * 32);
#pragma unroll
            for (int j = 0; j < U; j++) if (base + j * 32 < nv) visit8(v[j]);
        }
    }
    if (first < head) visit1(ld_stream1_f(p + first));
    else if (first - head < n - tail0) visit1(ld_stream1_f(p + tail0 + (first - head)));
}

// Does this tensor need a streaming pass at LEVEL?  (uniform over the grid: it only reads what the previous scan wrote)
template <int LEVEL>
__device__ __forceinline__ bool level_needed(const SelectState *st) {
    if (LEVEL == 0) return true;
    const unsigned m0 = st->mode[0], m1 = st->mode[1];
    const bool need0 = m0 == kModeHist || (m0 == kModeCompact && !st->compacted[0]);
    const bool need1 = !st->shared && (m1 == kModeHist || (m1 == kModeCompact && !st->compacted[1]));
    return need0 || need1;
}

// One pass over the part [a, b) of a tensor for the CTA (`first`, `stride` in threads of the cooperating group).  Returns false when the
// tensor needs nothing at this level (uniform over the grid).
template <int LEVEL, int TPB, int U = 4, bool SEG = (LEVEL != 0), class T = float>
__device__ __forceinline__ bool select_pass(const T *__restrict__ x, int64_t a, int64_t b, int64_t first, int64_t stride,
                                            SelectState *__restrict__ st, uint32_t *__restrict__ bufs, int64_t cap, int (*sh)[kDigits], unsigned int *sh_cnt) {
    constexpr int shift = level_shift(LEVEL);
    constexpr uint32_t dmask = level_dmask(LEVEL), pmask = level_pmask(LEVEL);
    const uint32_t p0 = st->prefix[0], p1 = st->prefix[1];
    const unsigned m0 = st->mode[0], m1 = st->mode[1];
    const bool same = st->shared != 0;
    const bool need0 = LEVEL == 0 || m0 == kModeHist || (m0 == kModeCompact && !st->compacted[0]);
    const bool need1 = LEVEL > 0 && !same && (m1 == kModeHist || (m1 == kModeCompact && !st->compacted[1]));
    if (!need0 && !need1) return false;
    for (int i = threadIdx.x; i < 2 * kDigits; i += TPB) (&sh[0][0])[i] = 0;
    if (threadIdx.x < 2) sh_cnt[threadIdx.x] = 0u;
    __syncthreads();
    const uint32_t a0 = (uint32_t)__cvta_generic_to_shared(&sh[0][0]), a1 = (uint32_t)__cvta_generic_to_shared(&sh[1][0]);
    uint32_t *buf0 = bufs, *buf1 = bufs + cap;
    uint32_t kmin0 = 0xFFFFFFFFu, kmax0 = 0u, kmin1 = 0xFFFFFFFFu, kmax1 = 0u;
    auto take = [&](uint32_t k, int r, unsigned mode, uint32_t sa, uint32_t *gbuf, uint32_t &kmin, uint32_t &kmax) {
        if (mode == kModeHist) {
            asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(sa + ((k >> shift) & dmask) * 4u) : "memory");
            kmin = min(kmin, k); kmax = max(kmax, k);
        } else {                                                        // compact: stage in shared memory, spill straight to the workspace when full
            const unsigned idx = atomicAdd(&sh_cnt[r], 1u);
            if (idx < (unsigned)kStage) sh[r][idx] = (int)k;
            else { const unsigned g = atomicAdd(&st->ccount[r], 1u); if ((long long)g < cap) gbuf[g] = k; }
        }
    };
    auto count = [&](uint32_t k) {
        if (LEVEL == 0) { asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(a0 + ((k >> shift) & dmask) * 4u) : "memory"); return; }
        const uint32_t hi = k & pmask;
        if (need0 && hi == p0) take(k, 0, m0, a0, buf0, kmin0, kmax0);
        if (need1 && hi == p1) take(k, 1, m1, a1, buf1, kmin1, kmax1);
    };
    // Fast rejection on the RAW bits (levels 1-2): key & pmask == p  <=>  bits & pmask == raw(p), because the key transform only depends on
    // the sign, which the prefix fixes.  One AND + two compares per element.
    auto raw_of = [&](uint32_t p) { return (p & 0x80000000u) ? (p & 0x7FFFFFFFu & pmask) : (~p & pmask); };
    const uint32_t c0 = raw_of(p0), c1 = raw_of(p1);
    auto hit = [&](float f) { const uint32_t t = __float_as_uint(f) & pmask; return (t == c0) | (t == c1); };
    auto visit4 = [&](const float4 &v) {
        if (LEVEL != 0 && !(hit(v.x) | hit(v.y) | hit(v.z) | hit(v.w))) return;
        count(order_key(v.x)); count(order_key(v.y)); count(order_key(v.z)); count(order_key(v.w));
    };
    auto visit1 = [&](float f) { count(order_key(f)); };
    stream_range<U, SEG>(x, a, b, first, stride, visit4, visit1);
    __syncthreads();
    // flush: histograms with global atomics on the non-empty digits, staged keys after one reservation per CTA and rank
    __shared__ unsigned int s_base[2];
    for (int r = 0; r < 2; r++) {
        const bool need = r == 0 ? need0 : need1;
        const unsigned mode = r == 0 ? m0 : m1;
        if (!need) continue;
        if (LEVEL == 0 || mode == kModeHist) {
            for (int i = threadIdx.x; i < kDigits; i += TPB) if (sh[r][i]) atomicAdd(&st->hist[r][i], (unsigned long long)sh[r][i]);
            if (LEVEL > 0) {
                uint32_t lo = r == 0 ? kmin0 : kmin1, hi = r == 0 ? kmax0 : kmax1;
                lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi);
                if ((threadIdx.x & 31) == 0 && lo <= hi) { atomicMin(&st->kmin[r], lo); atomicMax(&st->kmax[r], hi); }
            }
        } else {
            const unsigned m = min(sh_cnt[r], (unsigned)kStage);
            if (threadIdx.x == 0 && m) s_base[r] = atomicAdd(&st->ccount[r], m);
            __syncthreads();
            uint32_t *gbuf = r == 0 ? buf0 : buf1;
            for (unsigned i = threadIdx.x; i < m; i += TPB) if ((long long)(s_base[r] + i) < cap) gbuf[s_base[r] + i] = (uint32_t)sh[r][i];
        }
    }
    return true;
}

template <int TPB> __device__ __forceinline__ void finish_tensor_pass(SelectState *st, unsigned expected, bool *is_last);

// passes 1-2 at six CTAs per SM (40 registers) for fp32; the half unpacking needs a few more registers (five CTAs per SM, no spill)
template <class T> constexpr int kFilterCtas = std::is_same<T, float>::value ? 6 : 5;
// span and piece boundaries of the table kernels fall on whole 16-byte vectors of the table's element type
template <class T> constexpr int64_t kVecElems = 16 / sizeof(T);

// Pass 0 with speculation (table form, `guess` given): the digit histogram of every element as in select_pass<0>, and on the way every key
// beyond the thresholds remembered from the previous call of this slot (the previous batch of the same activation: the tail moves little
// from batch to batch) is compacted -- except copies of the previously selected key, which are only counted.  When the candidates turn out
// to contain the requested order statistics (select_scan<0>), the finish selects among them and the tensor has been read ONCE.
template <int TPB, class T = float>
__device__ __forceinline__ void select_pass0_spec(const T *__restrict__ x, int64_t a, int64_t b, int64_t first, int64_t stride,
                                                  SelectState *__restrict__ st, uint32_t *__restrict__ bufs, int64_t cap, int (*sh)[kDigits], unsigned int *sh_cnt) {
    constexpr int kHalf = kStage / 2;                                     // sh[1] holds both staging lists: hi candidates, then lo candidates
    const uint32_t g_hi = st->g[0], k_hi = st->k[0], g_lo = st->g[1], k_lo = st->k[1];
    for (int i = threadIdx.x; i < 2 * kDigits; i += TPB) (&sh[0][0])[i] = 0;
    if (threadIdx.x < 2) sh_cnt[threadIdx.x] = 0u;
    __syncthreads();
    const uint32_t a0 = (uint32_t)__cvta_generic_to_shared(&sh[0][0]);
    uint32_t *buf[2] = {bufs, bufs + cap};
    unsigned eq_hi = 0, eq_lo = 0;
    auto append = [&](int r, uint32_t k) {
        const unsigned idx = atomicAdd(&sh_cnt[r], 1u);
        if (idx < (unsigned)kHalf) sh[1][r * kHalf + idx] = (int)k;
        else { const unsigned gi = atomicAdd(&st->ccount[r], 1u); if ((long long)gi < cap) buf[r][gi] = k; }
    };
    auto candidate = [&](uint32_t k) {
        if (k >= g_hi) { if (k == k_hi) eq_hi++; else append(0, k); }
        if (k <= g_lo) { if (k == k_lo) eq_lo++; else append(1, k); }
    };
    auto digit = [&](uint32_t k) { asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(a0 + (k >> 21) * 4u) : "memory"); };
    auto visit4 = [&](const float4 &v) {
        const uint32_t k0 = order_key(v.x), k1 = order_key(v.y), k2 = order_key(v.z), k3 = order_key(v.w);
        digit(k0); digit(k1); digit(k2); digit(k3);
        if (max(max(k0, k1), max(k2, k3)) >= g_hi || min(min(k0, k1), min(k2, k3)) <= g_lo) { candidate(k0); candidate(k1); candidate(k2); candidate(k3); }
    };
    auto visit1 = [&](float f) { const uint32_t k = order_key(f); digit(k); candidate(k); };
    stream_range<4, false>(x, a, b, first, stride, visit4, visit1);
    __syncthreads();
    for (int i = threadIdx.x; i < kDigits; i += TPB) if (sh[0][i]) atomicAdd(&st->hist[0][i], (unsigned long long)sh[0][i]);
    eq_hi = __reduce_add_sync(0xffffffffu, eq_hi); eq_lo = __reduce_add_sync(0xffffffffu, eq_lo);
    if ((threadIdx.x & 31) == 0) { if (eq_hi) atomicAdd(&st->eqc[0], eq_hi); if (eq_lo) atomicAdd(&st->eqc[1], eq_lo); }
    __shared__ unsigned int s_base0[2];
    for (int r = 0; r < 2; r++) {
        const unsigned m = min(sh_cnt[r], (unsigned)kHalf);
        if (threadIdx.x == 0 && m) s_base0[r] = atomicAdd(&st->ccount[r], m);
        __syncthreads();
        for (unsigned i = threadIdx.x; i < m; i += TPB) if ((long long)(s_base0[r] + i) < cap) buf[r][s_base0[r] + i] = (uint32_t)sh[1][r * kHalf + i];
    }
}

template <class T>
__global__ void __launch_bounds__(kSelThreads, 1)
select_pass0_spec_kernel(const T *__restrict__ x, int64_t n, SelectState *__restrict__ st, uint32_t *__restrict__ bufs, int64_t cap) {
    __shared__ int sh[2][kDigits];
    __shared__ unsigned int sh_cnt[2];
    __shared__ bool is_last;
    select_pass0_spec<kSelThreads, T>(x, 0, n, (int64_t)blockIdx.x * kSelThreads + threadIdx.x, (int64_t)gridDim.x * kSelThreads, st, bufs, cap, sh, sh_cnt);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(&st->done, 1u) == gridDim.x - 1);
    __syncthreads();
    if (is_last) {
        __threadfence();
        select_scan<0, kSelThreads>(st, cap);
    }
}

template <class T = float>
__global__ void __launch_bounds__(kSelThreads, 1)
multi_select_pass0_spec_kernel(const ppq_b200_tensor_desc *__restrict__ descs, int count, SelectState *__restrict__ states,
                               uint32_t *__restrict__ bufs, int64_t cap) {
    __shared__ int sh[2][kDigits];
    __shared__ unsigned int sh_cnt[2];
    __shared__ bool is_last;
    extern __shared__ long long prefix[];                              // [count + 1]
    if (threadIdx.x == 0) {
        long long run = 0;
        for (int t = 0; t < count; t++) { prefix[t] = run; run += descs[t].n; }
        prefix[count] = run;
    }
    __syncthreads();
    const int64_t total = prefix[count];
    int64_t span = (total + gridDim.x - 1) / gridDim.x;
    span = (span + kVecElems<T> - 1) & ~(kVecElems<T> - 1);
    const int64_t s0 = (int64_t)blockIdx.x * span, s1 = (s0 + span) < total ? (s0 + span) : total;
    if (s0 >= total) return;
    int t = 0;
    { int lo = 0, hi = count - 1; while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (prefix[mid] <= s0) lo = mid; else hi = mid - 1; } t = lo; }
    for (; t < count && prefix[t] < s1; t++) {
        const ppq_b200_tensor_desc d = descs[t];
        if (d.n <= 0) continue;
        int64_t a = s0 - prefix[t]; if (a < 0) a = 0;
        int64_t b = s1 - prefix[t]; if (b > d.n) b = d.n;
        a = (a + kVecElems<T> - 1) & ~(kVecElems<T> - 1); if (a > d.n) a = d.n;
        if (b < d.n) b = (b + kVecElems<T> - 1) & ~(kVecElems<T> - 1); if (b > d.n) b = d.n;
        SelectState *st = states + t;
        if (b > a) select_pass0_spec<kSelThreads, T>(reinterpret_cast<const T *>(d.x), a, b, threadIdx.x, kSelThreads, st, bufs + (int64_t)t * 2 * cap, cap, sh, sh_cnt);
        const unsigned expected = (unsigned)((prefix[t + 1] - 1) / span - prefix[t] / span + 1);
        finish_tensor_pass<kSelThreads>(st, expected, &is_last);
        if (is_last) { __threadfence(); select_scan<0, kSelThreads>(st, cap); }
        __syncthreads();
    }
}

// ---- single tensor: the whole grid interleaves over the tensor, the last CTA to finish resolves the pass ------------------------------
template <int LEVEL, int TPB, int U = 4, bool SEG = (LEVEL != 0), int CTAS = (LEVEL == 0 ? 2 : 6), class T = float>
__global__ void __launch_bounds__(TPB, CTAS)
select_pass_kernel(const T *__restrict__ x, int64_t n, SelectState *__restrict__ st, uint32_t *__restrict__ bufs, int64_t cap) {
    __shared__ int sh[2][kDigits];
    __shared__ unsigned int sh_cnt[2];
    __shared__ bool is_last;
    if (!select_pass<LEVEL, TPB, U, SEG, T>(x, 0, n, (int64_t)blockIdx.x * TPB + threadIdx.x, (int64_t)gridDim.x * TPB, st, bufs, cap, sh, sh_cnt)) return;
    // every CTA's atomics are ordered before its ticket
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(&st->done, 1u) == gridDim.x - 1);
    __syncthreads();
    if (is_last) {
        __threadfence();
        select_scan<LEVEL, TPB>(st, cap);
    }
}

// ---- tables: each CTA owns one contiguous span of the concatenation of all tensors.  The CTAs that overlap a tensor are known from the span
// arithmetic alone, so the last of them to finish resolves that tensor's pass (ticket counter), as in the single-tensor kernel: no extra launch.
template <int TPB>
__device__ __forceinline__ void finish_tensor_pass(SelectState *st, unsigned expected, bool *is_last) {
    __threadfence();                                                   // this CTA's atomics are ordered before its ticket
    __syncthreads();
    if (threadIdx.x == 0) *is_last = (atomicAdd(&st->done, 1u) == expected - 1u);
    __syncthreads();
}

// The table's element type T is one per launch (every descriptor's `x` points at elements of that type).  On top of the single-tensor
// passes a table pass carries the span walk, so the half unpacking does not fit their register budgets without spilling: fp16 / bf16 run
// pass 0 at one 1024-thread CTA per SM (64 registers, like the speculative pass 0) and passes 1-2 at four CTAs per SM.
template <class T> constexpr int kTablePass0Ctas = std::is_same<T, float>::value ? 2 : 1;
template <class T> constexpr int kTableFilterCtas = std::is_same<T, float>::value ? 6 : 4;
template <int LEVEL, int TPB, class T = float>
__global__ void __launch_bounds__(TPB, LEVEL == 0 ? kTablePass0Ctas<T> : kTableFilterCtas<T>)
multi_select_pass_kernel(const ppq_b200_tensor_desc *__restrict__ descs, int count, SelectState *__restrict__ states,
                         uint32_t *__restrict__ bufs, int64_t cap) {
    __shared__ int sh[2][kDigits];
    __shared__ unsigned int sh_cnt[2];
    __shared__ bool is_last;
    extern __shared__ long long prefix[];                              // [count + 1]
    if (threadIdx.x == 0) {
        long long run = 0;
        for (int t = 0; t < count; t++) { prefix[t] = run; run += descs[t].n; }
        prefix[count] = run;
    }
    __syncthreads();
    const int64_t total = prefix[count];
    int64_t span = (total + gridDim.x - 1) / gridDim.x;
    span = (span + kVecElems<T> - 1) & ~(kVecElems<T> - 1);
    const int64_t s0 = (int64_t)blockIdx.x * span, s1 = (s0 + span) < total ? (s0 + span) : total;
    if (s0 >= total) return;
    int t = 0;
    { int lo = 0, hi = count - 1; while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (prefix[mid] <= s0) lo = mid; else hi = mid - 1; } t = lo; }
    for (; t < count && prefix[t] < s1; t++) {
        const ppq_b200_tensor_desc d = descs[t];
        if (d.n <= 0) continue;
        int64_t a = s0 - prefix[t]; if (a < 0) a = 0;
        int64_t b = s1 - prefix[t]; if (b > d.n) b = d.n;
        a = (a + kVecElems<T> - 1) & ~(kVecElems<T> - 1); if (a > d.n) a = d.n;   // both neighbours round the shared boundary the same way
        if (b < d.n) b = (b + kVecElems<T> - 1) & ~(kVecElems<T> - 1); if (b > d.n) b = d.n;
        SelectState *st = states + t;
        bool active;                                                   // uniform over the grid
        if (b > a) active = select_pass<LEVEL, TPB, 4, (LEVEL != 0), T>(reinterpret_cast<const T *>(d.x), a, b, threadIdx.x, TPB, st, bufs + (int64_t)t * 2 * cap, cap, sh, sh_cnt);
        else active = level_needed<LEVEL>(st);                         // overlaps the tensor by less than a vector: no data, but a ticket
        if (active) {
            const unsigned expected = (unsigned)((prefix[t + 1] - 1) / span - prefix[t] / span + 1);
            finish_tensor_pass<TPB>(st, expected, &is_last);
            if (is_last) { __threadfence(); select_scan<LEVEL, TPB>(st, cap); }
        }
        __syncthreads();
    }
}

// ---- finish: one CTA per (tensor, rank) selects among the compacted keys (or just reports a resolved key) -------------------------------
__global__ void __launch_bounds__(kSelThreads)
select_finish_kernel(const SelectState *__restrict__ states, const uint32_t *__restrict__ bufs, int64_t cap,
                     const ppq_b200_tensor_desc *__restrict__ descs, float *__restrict__ out, int64_t out_stride, uint32_t *__restrict__ guess = nullptr) {
    __shared__ int sh[kDigits];
    __shared__ unsigned int s_digit;
    __shared__ unsigned long long s_before, s_cnt;
    const int tensor = blockIdx.x >> 1, r = blockIdx.x & 1;
    const SelectState *st = states + tensor;
    if (descs && descs[tensor].n <= 0) return;                         // an empty table entry has no order statistics: its slot and guess stay as they are
    float *dst = out + (descs ? (int64_t)descs[tensor].slot : 0) * out_stride + r;
    unsigned int key = st->prefix[r];
    if (st->mode[r] == kModeCompact) {
        const uint32_t *keys = bufs + ((int64_t)tensor * 2 + st->cbuf[r]) * cap;
        const unsigned m = st->ccount[st->cbuf[r]];
        unsigned long long k = (unsigned long long)st->rank[r];
        // The first kFinishRegs x 1024 candidates live in registers for all three levels (a cold call that speculated on sampled thresholds
        // brings ~40 K of them: re-reading them from L2 once per level, one dependent load per iteration, cost 15-20 us); the rest is
        // streamed per level with 8 loads in flight.
        constexpr int kFinishRegs = 32;
        uint32_t held[kFinishRegs];
        const unsigned groups = (m + 8u * kSelThreads - 1u) / (8u * kSelThreads);            // CTA-uniform: 8-entry register groups that hold anything
        const unsigned mine = m > threadIdx.x ? (m - threadIdx.x + kSelThreads - 1u) / kSelThreads : 0u;   // entries t, t + 1024, ... < m: entry e is real iff e < mine
#pragma unroll
        for (int g = 0; g < kFinishRegs / 8; g++) {
            if ((unsigned)g < groups) {
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int e = g * 8 + j;
                    held[e] = (unsigned)e < mine ? __ldcg(keys + (unsigned)e * kSelThreads + threadIdx.x) : 0u;
                }
            }
        }
        const uint32_t vkey = st->vkey[r];
        const unsigned veq = st->veq[r];
        for (int level = (int)st->clevel[r]; level <= 2; level++) {
            const int shift = level_shift(level);
            const uint32_t dmask = level_dmask(level), pmask = level_pmask(level), want = key & pmask;
            for (int i = threadIdx.x; i < kDigits; i += kSelThreads) sh[i] = 0;
            __syncthreads();
#pragma unroll
            for (int g = 0; g < kFinishRegs / 8; g++) {
                if ((unsigned)g < groups) {
#pragma unroll
                    for (int j = 0; j < 8; j++) {                          // conditional on purpose: from level 1 on ~95 % of the candidates miss the
                        const int e = g * 8 + j;                           // prefix, and a skipped branch is cheaper than an atomic on a trash slot (measured: 88 vs 94 us)
                        if ((unsigned)e < mine && (held[e] & pmask) == want) atomicAdd(&sh[(held[e] >> shift) & dmask], 1);
                    }
                }
            }
            for (unsigned base = kFinishRegs * kSelThreads; base < m; base += 8 * kSelThreads) {
                uint32_t v[8];
#pragma unroll
                for (int j = 0; j < 8; j++) { const unsigned i = base + (unsigned)j * kSelThreads + threadIdx.x; v[j] = i < m ? __ldcg(keys + i) : 0u; }
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const unsigned i = base + (unsigned)j * kSelThreads + threadIdx.x;
                    if (i < m && (v[j] & pmask) == want) atomicAdd(&sh[(v[j] >> shift) & dmask], 1);
                }
            }
            if (threadIdx.x == 0 && veq && (vkey & pmask) == want)                            // the counted-only copies of the threshold key
                atomicAdd(&sh[(vkey >> shift) & dmask], (int)veq);
            __syncthreads();
            block_pick<kSelThreads>([&](int i) { return (unsigned long long)sh[i]; }, k, &s_digit, &s_before, &s_cnt);
            key |= s_digit << shift;
            k -= s_before;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        *dst = key_to_float(key);
        if (guess) {                                                    // thresholds for the next call of this slot: the selected key -/+ the margin
            uint32_t *gw = guess + (descs ? (int64_t)descs[tensor].slot : 0) * kGuessWords + 4 * r;
            const uint32_t d = st->d[r];
            gw[0] = r == 0 ? (key > d ? key - d : 0u) : (key < 0xFFFFFFFFu - d ? key + d : 0xFFFFFFFFu);
            gw[1] = key; gw[2] = d; gw[3] = 0u;
        }
    }
}

static inline int grid_pass0(int64_t n) {
    int64_t g = (n + (int64_t)kSelThreads * 16 - 1) / ((int64_t)kSelThreads * 16);
    if (g > 2 * sm_count()) g = 2 * sm_count();                                       // pass 0 needs 32 registers per thread: two 1024-thread CTAs fit on an SM
    return (int)(g < 1 ? 1 : g);
}
static inline int grid_filter(int64_t n) {
    int64_t g = (n + (int64_t)kFilterThreads * 16 - 1) / ((int64_t)kFilterThreads * 16);
    if (g > 6 * sm_count()) g = 6 * sm_count();                                       // 40 registers, 16.5 KB of smem: six CTAs per SM, one wave
    return (int)(g < 1 ? 1 : g);
}

template <class T>
static int select_two(const T *x, int64_t n, int q_mode, float q, long long r0, long long r1, float *out, void *workspace, cudaStream_t s,
                      uint32_t *guess = nullptr) {
    SelectState *st = (SelectState *)workspace;
    uint32_t *bufs = (uint32_t *)(st + 1);
    const int64_t cap = kDefaultCap;
    // cold call on a big tensor: thresholds from a sample (select_init_kernel), unless both tails are too heavy for the compaction buffer
    bool sample = false;
    if (q_mode && n >= kSampleMinElems && !(variant_of(kVarSelect) & 64)) {
        auto rank_of = [&](float frac) { long long pos = (long long)nearbyintf((float)n * frac); pos = pos > n - 1 ? n - 1 : pos; return pos < 0 ? 0 : pos; };
        const long long need_hi = n - rank_of(q), need_lo = rank_of(1.0f - q) + 1;
        sample = sample_rank_ok(sample_rank_from_end(need_hi, n), n, cap) || sample_rank_ok(sample_rank_from_end(need_lo, n), n, cap);
    }
    uint32_t *sample_keys = bufs + 2 * cap;
    if (sample) select_sample_kernel<T><<<kSampleKeys / 256, 256, 0, s>>>(x, n, sample_keys);
    select_init_kernel<<<1, 1024, 0, s>>>(st, nullptr, n, q, q_mode, r0, r1, guess, sample ? sample_keys : nullptr, cap);
    if (guess || sample) {
        const int g0 = grid_pass0(n);
        select_pass0_spec_kernel<T><<<g0 > sm_count() ? sm_count() : g0, kSelThreads, 0, s>>>(x, n, st, bufs, cap);
    } else if constexpr (!std::is_same<T, float>::value) {              // the A/B knobs below are fp32 only
        select_pass_kernel<0, kSelThreads, 2, false, 2, T><<<grid_pass0(n), kSelThreads, 0, s>>>(x, n, st, bufs, cap);   // 2 x 16 B in flight: 32 registers, no spill
    } else {
        switch (variant_of(kVarSelect) & 7) {                              // A/B knobs of pass 0 (variants.h)
        case 1: select_pass_kernel<0, kSelThreads, 2><<<grid_pass0(n), kSelThreads, 0, s>>>(x, n, st, bufs, cap); break;
        case 2: select_pass_kernel<0, kSelThreads, 4, true><<<grid_pass0(n), kSelThreads, 0, s>>>(x, n, st, bufs, cap); break;
        case 3: select_pass_kernel<0, kSelThreads, 2, true><<<grid_pass0(n), kSelThreads, 0, s>>>(x, n, st, bufs, cap); break;
        case 4: select_pass_kernel<0, 512, 4, false, 4><<<grid_pass0(n) * 2, 512, 0, s>>>(x, n, st, bufs, cap); break;
        default: select_pass_kernel<0, kSelThreads><<<grid_pass0(n), kSelThreads, 0, s>>>(x, n, st, bufs, cap);
        }
    }
    if constexpr (!std::is_same<T, float>::value) {
        select_pass_kernel<1, kFilterThreads, 4, true, kFilterCtas<T>, T><<<grid_filter(n), kFilterThreads, 0, s>>>(x, n, st, bufs, cap);
    } else {
        switch ((variant_of(kVarSelect) >> 3) & 7) {                             // ... and of pass 1
        case 1: select_pass_kernel<1, kFilterThreads, 2><<<grid_filter(n), kFilterThreads, 0, s>>>(x, n, st, bufs, cap); break;
        case 2: select_pass_kernel<1, 512, 4, true, 3><<<grid_filter(n) > 1 ? grid_filter(n) / 2 : 1, 512, 0, s>>>(x, n, st, bufs, cap); break;
        case 3: select_pass_kernel<1, 1024, 2, true, 2><<<grid_pass0(n), 1024, 0, s>>>(x, n, st, bufs, cap); break;
        case 4: select_pass_kernel<1, kFilterThreads, 4, false><<<grid_filter(n), kFilterThreads, 0, s>>>(x, n, st, bufs, cap); break;
        default: select_pass_kernel<1, kFilterThreads><<<grid_filter(n), kFilterThreads, 0, s>>>(x, n, st, bufs, cap);
        }
    }
    // pass 2 is rarely needed (a bucket too big to compact that holds several distinct values): two CTAs per SM keep its usual early exit cheap
    const int g2 = grid_filter(n) > 2 * sm_count() ? 2 * sm_count() : grid_filter(n);
    select_pass_kernel<2, kFilterThreads, 4, true, kFilterCtas<T>, T><<<g2, kFilterThreads, 0, s>>>(x, n, st, bufs, cap);
    select_finish_kernel<<<2, kSelThreads, 0, s>>>(st, bufs, cap, nullptr, out, 0, guess);
    return (int)cudaGetLastError();
}

}  // namespace ppqb

using namespace ppqb;

extern "C" {

int64_t ppq_b200_quantile_workspace_bytes(void) { return (int64_t)sizeof(SelectState) + (2 * kDefaultCap + kSampleKeys) * (int64_t)sizeof(uint32_t); }

int64_t ppq_b200_quantile_guess_words(void) { return kGuessWords; }

int ppq_b200_quantile_guess_init(uint32_t *guess, int64_t slots, void *stream) {
    if (!guess || slots <= 0) return (int)cudaErrorInvalidValue;
    // thresholds that select nothing (key >= 0xFFFFFFFF / key <= 0), so that the first call takes the regular two-pass route
    static const uint32_t row[kGuessWords] = {0xFFFFFFFFu, 0xFFFFFFFFu, kSpecMarginInit, 0u, 0u, 0u, kSpecMarginInit, 0u};
    for (int64_t i = 0; i < slots; i++)
        if (cudaMemcpyAsync(guess + i * kGuessWords, row, sizeof(row), cudaMemcpyHostToDevice, (cudaStream_t)stream) != cudaSuccess) return (int)cudaGetLastError();
    return 0;
}

int64_t ppq_b200_multi_quantile_workspace_bytes(int count, int64_t cap) {
    if (count <= 0 || cap <= 0) return 0;
    return (int64_t)count * ((int64_t)sizeof(SelectState) + 2 * cap * (int64_t)sizeof(uint32_t));
}

int ppq_b200_quantile_t_dt(const void *x, int dtype, int64_t n, float q, float *out2, void *workspace, uint32_t *guess, void *stream) {
    if (!valid_dtype(dtype) || n <= 0 || !x || !out2 || !workspace) return (int)cudaErrorInvalidValue;
    return with_elem_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        return select_two((const T *)x, n, 1, q, 0, 0, out2, workspace, (cudaStream_t)stream, guess);
    });
}

int ppq_b200_quantile_t(const float *x, int64_t n, float q, float *out2, void *workspace, void *stream) {
    return ppq_b200_quantile_t_dt(x, PPQ_B200_F32, n, q, out2, workspace, nullptr, stream);
}

int ppq_b200_quantile_t_guess(const float *x, int64_t n, float q, float *out2, void *workspace, uint32_t *guess, void *stream) {
    return ppq_b200_quantile_t_dt(x, PPQ_B200_F32, n, q, out2, workspace, guess, stream);
}

int ppq_b200_multi_quantile_t_dt(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, int dtype, float q, float *out, int64_t out_stride,
                                 void *workspace, int64_t cap, uint32_t *guess, void *stream) {
    if (!valid_dtype(dtype) || count <= 0 || max_n <= 0 || !descs || !out || !workspace || cap <= 0 || out_stride < 2) return (int)cudaErrorInvalidValue;
    const size_t smem = (size_t)(count + 1) * sizeof(long long);
    if (smem > 24 * 1024) return (int)cudaErrorInvalidValue;
    cudaStream_t s = (cudaStream_t)stream;
    SelectState *states = (SelectState *)workspace;
    uint32_t *bufs = (uint32_t *)(states + count);
    int64_t work = (int64_t)count * max_n;
    int g0 = grid_pass0(work), g1 = grid_filter(work);
    select_init_kernel<<<count, 1024, 0, s>>>(states, descs, 0, q, 1, 0, 0, guess);
    with_elem_type(dtype, [&](auto tag) {
        using T = decltype(tag);
        if (guess) {                                                    // 64 registers per thread: one 1024-thread CTA per SM
            const int gs = g0 > sm_count() ? sm_count() : g0;
            multi_select_pass0_spec_kernel<T><<<gs, kSelThreads, smem, s>>>(descs, count, states, bufs, cap);
        } else {
            const int resident = kTablePass0Ctas<T> * sm_count();
            multi_select_pass_kernel<0, kSelThreads, T><<<g0 > resident ? resident : g0, kSelThreads, smem, s>>>(descs, count, states, bufs, cap);
        }
        multi_select_pass_kernel<1, kFilterThreads, T><<<g1, kFilterThreads, smem, s>>>(descs, count, states, bufs, cap);
        multi_select_pass_kernel<2, kFilterThreads, T><<<g1 > 2 * sm_count() ? 2 * sm_count() : g1, kFilterThreads, smem, s>>>(descs, count, states, bufs, cap);
        return 0;
    });
    select_finish_kernel<<<2 * count, kSelThreads, 0, s>>>(states, bufs, cap, descs, out, out_stride, guess);
    return (int)cudaGetLastError();
}

int ppq_b200_multi_quantile_t(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, float q, float *out, int64_t out_stride,
                              void *workspace, int64_t cap, uint32_t *guess, void *stream) {
    return ppq_b200_multi_quantile_t_dt(descs, count, max_n, PPQ_B200_F32, q, out, out_stride, workspace, cap, guess, stream);
}

int ppq_b200_isotone_t(const float *x, int64_t n, float *out4, void *workspace, void *stream) {
    if (n <= 0 || !x || !out4 || !workspace) return (int)cudaErrorInvalidValue;
    if (n == 1) {
        int rc = select_two(x, n, 0, 0.f, 0, 0, out4, workspace, (cudaStream_t)stream);
        if (rc) return rc;
        return select_two(x, n, 0, 0.f, 0, 0, out4 + 2, workspace, (cudaStream_t)stream);
    }
    // out = { sorted[n-1], sorted[n-2], sorted[0], sorted[1] }
    int rc = select_two(x, n, 0, 0.f, n - 1, n - 2, out4, workspace, (cudaStream_t)stream);
    if (rc) return rc;
    return select_two(x, n, 0, 0.f, 0, 1, out4 + 2, workspace, (cudaStream_t)stream);
}

}  // extern "C"
