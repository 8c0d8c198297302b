// search.cu -- scale / offset search on the device (sm_90a), behind the C ABI of include/ppq_b200.h.
//
//   ppq_b200_minmax_to_scale_offset   replaces minmax_to_scale_offset   (/root/reference/ppq/quantization/observer/range.py:22-75)
//   ppq_b200_hist_scale_from_minmax   replaces the phase-1 render of TorchHistObserver (range.py:291-301)
//   ppq_b200_kl_search                replaces TorchHistObserver.hist_to_scale_offset (range.py:190-282) +
//                                     torch_KL_divergence (ppq/quantization/measure/statistic.py:3-12)
//   ppq_b200_mse_search               replaces TorchMSEObserver.hist_to_scale_offset (range.py:456-520) driving
//                                     compute_mse_loss (ppq/csrc/cpu/hist_mse.cc:3-28)
//
// These are tiny (O(tensors x bins)) but they keep the render phase of the calibration on the device: no .item() per
// tensor, no per-channel Python loop, and the histogram arena never has to leave HBM before the all-reduce.
// Arithmetic follows the Python originals: fp64 for the scale/offset algebra (Python floats), fp32 histograms and fp64
// log10 for the KL divergence.
#include "common.cuh"
#include "../../include/ppq_b200.h"
#include "variants.h"

namespace ppqb {

// ppq_numerical_round(v, ROUND_HALF_EVEN) on a double (utils/round.py:78: Decimal.quantize half-even == rint).
__device__ __forceinline__ double round_half_even(double v) { return rint(v); }

// ppq_round_to_power_of_2 (utils/round.py:115-135): 2^round(log2(x)); ROUND_UP = ceil, ROUND_HALF_UP on the exponent.
// Exact powers of two are recognised from the binary exponent (math.log2 is exact on them); everything else follows the Python formula
// on the double log2, so a value a few ulps above a power of two rounds the way math.log2 + ceil() does.  The result is built with ldexp.
// Ties of the HALF_UP policy: Decimal ROUND_HALF_UP for value > 0 (2.5 -> 3) and ROUND_HALF_DOWN for value <= 0 (-9.5 -> -9,
// utils/round.py:80-82) -- both send an exact .5 to floor + 1.
__device__ __forceinline__ double pow2_round(double v, bool half_up) {
    if (v == 0.0) return 0.0;
    const double sign = v >= 0.0 ? 1.0 : -1.0;
    int e2;
    const double m = frexp(sign * v, &e2);                             // |v| = m * 2^e2, m in [0.5, 1)
    int e;
    if (m == 0.5) e = e2 - 1;                                           // exact power of two
    else {
        const double l = log2(sign * v);
        if (!half_up) e = (int)ceil(l);
        else { const double f = floor(l); e = (l - f >= 0.5) ? (int)f + 1 : (int)f; }
    }
    return sign * ldexp(1.0, e);
}

struct ScaleOffset { double scale, offset; };
__device__ __forceinline__ ScaleOffset minmax_to_scale_offset_dev(double mn, double mx, int qmin, int qmax, bool sym, bool pow2,
                                                                  double min_scale) {
    if (mn > 0.0) mn = 0.0;
    if (mx < 0.0) mx = 0.0;
    ScaleOffset r;
    const double levels = (double)(qmax - qmin);
    if (sym) {
        const double range = 2.0 * fmax(fabs(mx), fabs(mn));
        r.scale = fmax(range / levels, min_scale);
        r.offset = 0.0;
    } else {
        const double range = mx - mn;
        r.scale = fmax(range / levels, min_scale);
        r.offset = round_half_even(-mn / r.scale);
    }
    if (pow2) r.scale = pow2_round(r.scale, false);
    return r;
}

__global__ void minmax_to_scale_offset_kernel(const float *__restrict__ mins, const float *__restrict__ maxs, int64_t count,
                                              int64_t stride, int qmin, int qmax, int sym, int pow2, double min_scale,
                                              float *__restrict__ scale, float *__restrict__ offset) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const ScaleOffset r = minmax_to_scale_offset_dev((double)mins[i * stride], (double)maxs[i * stride], qmin, qmax, sym != 0,
                                                     pow2 != 0, min_scale);
    scale[i] = (float)r.scale;
    offset[i] = (float)r.offset;
}

__global__ void hist_scale_kernel(const float *__restrict__ minmax, int64_t count, int sym, int64_t bins, float *__restrict__ hs) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const double mn = (double)minmax[2 * i], mx = (double)minmax[2 * i + 1];
    const double range = sym ? fmax(fabs(mx), fabs(mn)) : (mx - mn);
    hs[i] = (float)(range / (double)bins);
}

// ---- KL search: one CTA per histogram ---------------------------------------------------------------------------------------
constexpr int kKlThreads = 512;
constexpr int kKlMemoBins = 8192;             // up to here the memoised logarithms fit next to the histogram and its prefix sums

__device__ __forceinline__ double block_sum(double v, double *scratch) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) scratch[w] = v;
    __syncthreads();
    double t = 0.0;
    for (int i = 0; i < kKlThreads / 32; i++) t += scratch[i];
    return t;
}

__global__ void __launch_bounds__(kKlThreads)
kl_search_kernel(const int32_t *__restrict__ hist_arena, int bins, const float *__restrict__ hist_scale_arena,
                 const float *__restrict__ minmax_arena, int num_of_bits, int pow2, double min_scale, float *__restrict__ scale_out, int32_t *__restrict__ best_out) {
    extern __shared__ unsigned char kl_smem[];
    float *h = reinterpret_cast<float *>(kl_smem);                    // [bins]   the edited histogram as fp32
    const int pre_len = max(bins + 1, kKlThreads);                    // the prefix array doubles as scratch for the per-thread totals of the scan
    double *pre = reinterpret_cast<double *>(kl_smem + (((size_t)bins * 4 + 7) & ~(size_t)7));   // [bins + 1] exclusive prefix sums
    float *gval = reinterpret_cast<float *>(pre + pre_len);           // [quant_bins] per-group spread value, then q of the group
    // memo (bins <= kKlMemoBins): log10(p + 1e-30) of every bin is the same for all 32 candidates (only the bin that absorbs the tail
    // differs), and log10(q + 1e-30) is shared by the bins of a group -> 4096 + 32 x 128 fp64 logarithms instead of 2 x 67 584.
    // The doubles that enter the sum are the same ones, in the same order, so the losses are bit-identical to the direct evaluation.
    const bool memo = bins <= kKlMemoBins;
    double *glogq = reinterpret_cast<double *>(kl_smem + ((((size_t)bins * 4 + 7) & ~(size_t)7) + (size_t)pre_len * 8 +
                                                          (((size_t)(1 << (num_of_bits - 1)) * 4 + 7) & ~(size_t)7)));   // [quant_bins]
    double *logp = glogq + (1 << (num_of_bits - 1));                                                                    // [bins]
    __shared__ double scratch[kKlThreads / 32];
    __shared__ double s_best_loss; __shared__ int s_best;

    const int32_t *hist = hist_arena + (int64_t)blockIdx.x * bins;
    const int quant_bins = 1 << (num_of_bits - 1);
    const int dead = (int)((double)bins * .002);                      // int(hist_bins * .002)
    for (int i = threadIdx.x; i < bins; i += kKlThreads) {
        float v = (float)hist[i];
        if (i < dead) v = 0.f;
        if (i == dead) v = 1.f;
        h[i] = v;
    }
    __syncthreads();
    // exclusive prefix sums (integer-valued counts: exact in fp64); serial per 64-bin segment, then segment offsets
    {
        const int seg = (bins + kKlThreads - 1) / kKlThreads;
        const int b0 = threadIdx.x * seg, b1 = min(bins, b0 + seg);
        double s = 0.0;
        for (int i = b0; i < b1; i++) s += (double)h[i];
        // inclusive scan of the per-thread totals through shared memory
        double *tot = pre;                                            // reuse: pre[0..kKlThreads) temporarily
        __syncthreads();
        tot[threadIdx.x] = s;
        __syncthreads();
        double base = 0.0;
        for (int t = 0; t < (int)threadIdx.x; t++) base += tot[t];
        __syncthreads();
        double run = base;
        for (int i = b0; i < b1; i++) { const double v = (double)h[i]; pre[i] = run; run += v; }
        if (b1 == bins && b0 < bins) pre[bins] = run;
        if (bins == 0 && threadIdx.x == 0) pre[0] = 0.0;
        __syncthreads();
    }
    const float total = (float)pre[bins];                            // torch.sum(histogram) (fp32 tensor)
    if (threadIdx.x == 0) { s_best_loss = 0.0; s_best = -1; }
    if (memo) for (int i = threadIdx.x; i < bins; i += kKlThreads) logp[i] = log10((double)__fdiv_rn(h[i], total) + 1e-30);

    for (int br = quant_bins; br < bins + quant_bins - 1; br += quant_bins) {
        if (br > bins) break;                                         // range() upstream never exceeds bins for bins % quant_bins == 0
        const int ratio = br / quant_bins;
        // group statistics: spread value = (sum of the group) / (number of non-empty bins), fp32 like torch.div
        for (int g = threadIdx.x; g < quant_bins; g += kKlThreads) {
            const int a = g * ratio;
            int cnt = 0;
            for (int i = a; i < a + ratio; i++) cnt += h[i] > 0.f;
            const float gsum = (float)(pre[a + ratio] - pre[a]);
            gval[g] = __fdiv_rn(gsum, (float)(cnt == 0 ? 1 : cnt));
        }
        __syncthreads();
        // normaliser of q: sum over non-empty bins of their group's spread value
        double qs = 0.0;
        for (int i = threadIdx.x; i < br; i += kKlThreads) if (h[i] > 0.f) qs += (double)gval[i / ratio];
        const float qsum = (float)block_sum(qs, scratch);
        const float tail = (float)(pre[bins] - pre[br]);              // torch.sum(histogram[bin_range:])
        // q = (spread value * non-empty mask) / sum: when every bin of the candidate is empty this is 0/0 = NaN upstream
        // and the candidate's loss is NaN (python's sorted() then keeps that first candidate in front) -- keep that.
        const float q_empty = __fdiv_rn(0.f, qsum);
        if (memo) {
            for (int g = threadIdx.x; g < quant_bins; g += kKlThreads) {
                const float q = __fdiv_rn(gval[g], qsum);
                gval[g] = q;                                          // every thread is past its last read of the spread values (block_sum)
                glogq[g] = log10((double)q + 1e-30);
            }
            __syncthreads();
        }
        double kl = 0.0;
        for (int i = threadIdx.x; i < br; i += kKlThreads) {
            float pv = h[i];
            const bool nonempty = pv > 0.f, last = (i == br - 1);
            if (last) pv = __fadd_rn(pv, tail);
            const float p = __fdiv_rn(pv, total);
            const float q = nonempty ? (memo ? gval[i / ratio] : __fdiv_rn(gval[i / ratio], qsum)) : q_empty;
            if (p == 0.f && q == q) continue;                         // 0 * (finite) contributes exactly 0
            const double lp = (memo && !last) ? logp[i] : log10((double)p + 1e-30);
            const double lq = (memo && nonempty) ? glogq[i / ratio] : log10((double)q + 1e-30);
            kl += (double)p * (lp - lq);
        }
        kl = block_sum(kl, scratch);
        if (threadIdx.x == 0 && (s_best < 0 || kl < s_best_loss)) { s_best = br; s_best_loss = kl; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double hs;
        if (minmax_arena) {
            const double mn = (double)minmax_arena[2 * blockIdx.x], mx = (double)minmax_arena[2 * blockIdx.x + 1];
            hs = fmax(fabs(mx), fabs(mn)) / (double)bins;            // the Python double of range.py:294-300
        } else hs = (double)hist_scale_arena[blockIdx.x];
        double scale = ((double)s_best / (double)bins) * hs * ((double)bins / (double)quant_bins);
        scale = fmax(scale, min_scale);
        if (pow2) scale = pow2_round(scale, true);
        scale_out[blockIdx.x] = (float)scale;
        if (best_out) best_out[blockIdx.x] = s_best;
    }
}

// ---- KL search, one WARP per candidate (default for bins <= 8192) ------------------------------------------------------------------------------
// The candidates are independent given the edited histogram, its prefix sums and the memoised log10(p): the kernel above walks them one
// after the other with four block-wide barriers each (160-196 us for 106 histograms, and the same latency for a single one -- what the
// drop-in flow pays per rendered tensor).  Here the 32 warps of a 1024-thread CTA take one candidate each (round-robin when there are more,
// e.g. 512 for 4-bit configs) with warp-level reductions only; the first minimum in candidate order wins, as with python's stable sort.
// The fp64 sums associate differently from the serial kernel (lane-strided partial sums + shuffle tree), which can only matter when two
// candidates' divergences agree to ~1e-15 relative (DESIGN.md, documented deviation 2).
constexpr int kKlwThreads = 1024;
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(kKlwThreads)
kl_search_warp_kernel(const int32_t *__restrict__ hist_arena, int bins, const float *__restrict__ hist_scale_arena,
                      const float *__restrict__ minmax_arena, int num_of_bits, int pow2, double min_scale, float *__restrict__ scale_out, int32_t *__restrict__ best_out) {
    extern __shared__ unsigned char kl_smem[];
    const int quant_bins = 1 << (num_of_bits - 1);
    const int ncand = bins / quant_bins;                              // range(quant_bins, bins + quant_bins - 1, quant_bins), capped at bins
    const int pre_len = max(bins + 1, kKlwThreads);
    float *h = reinterpret_cast<float *>(kl_smem);                    // [bins]
    double *pre = reinterpret_cast<double *>(kl_smem + (((size_t)bins * 4 + 7) & ~(size_t)7));      // [bins + 1]
    double *logp = pre + pre_len;                                     // [bins]
    double *loss = logp + bins;                                       // [ncand]
    float *gval_all = reinterpret_cast<float *>(loss + ((ncand + 1) & ~1));      // [32 warps][quant_bins]: a warp's per-group spread values
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float *gval = gval_all + (size_t)w * quant_bins;

    const int32_t *hist = hist_arena + (int64_t)blockIdx.x * bins;
    const int dead = (int)((double)bins * .002);
    for (int i = threadIdx.x; i < bins; i += kKlwThreads) {
        float v = (float)hist[i];
        if (i < dead) v = 0.f;
        if (i == dead) v = 1.f;
        h[i] = v;
    }
    __syncthreads();
    {   // exclusive prefix sums (integer-valued counts: exact in fp64)
        const int seg = (bins + kKlwThreads - 1) / kKlwThreads;
        const int b0 = threadIdx.x * seg, b1 = min(bins, b0 + seg);
        double s_ = 0.0;
        for (int i = b0; i < b1; i++) s_ += (double)h[i];
        double *tot = pre;
        tot[threadIdx.x] = s_;
        __syncthreads();
        double base = 0.0;
        for (int t = 0; t < (int)threadIdx.x; t++) base += tot[t];
        __syncthreads();
        double run = base;
        for (int i = b0; i < b1; i++) { const double v = (double)h[i]; pre[i] = run; run += v; }
        if (b1 == bins && b0 < bins) pre[bins] = run;
        __syncthreads();
    }
    const float total = (float)pre[bins];
    for (int i = threadIdx.x; i < bins; i += kKlwThreads) logp[i] = log10((double)__fdiv_rn(h[i], total) + 1e-30);
    __syncthreads();

    for (int c = w; c < ncand; c += kKlwThreads / 32) {
        // candidate bin_range = (c + 1) * quant_bins: every group spans `ratio` = c + 1 bins.  A lane owns whole groups (lane, lane + 32, ...),
        // so nothing in the loops divides an index by the ratio and a group's q and log10(q) stay in registers.
        const int br = (c + 1) * quant_bins, ratio = c + 1;
        double qs = 0.0;
        for (int g = lane; g < quant_bins; g += 32) {
            const int a = g * ratio;
            int cnt = 0;
            for (int i = a; i < a + ratio; i++) cnt += h[i] > 0.f;
            const float spread = __fdiv_rn((float)(pre[a + ratio] - pre[a]), (float)(cnt == 0 ? 1 : cnt));
            gval[g] = spread;
            qs += (double)spread * (double)cnt;                          // the sum over the group's non-empty bins of their spread value
        }
        const float qsum = (float)warp_sum(qs);
        const float tail = (float)(pre[bins] - pre[br]);
        const float q_empty = __fdiv_rn(0.f, qsum);                      // 0/0 = NaN when every bin of the candidate is empty, as upstream
        const double lq_empty = log10((double)q_empty + 1e-30);
        double kl = 0.0;
        for (int g = lane; g < quant_bins; g += 32) {
            const int a = g * ratio;
            const float q = __fdiv_rn(gval[g], qsum);
            const double lq = log10((double)q + 1e-30);
            for (int i = a; i < a + ratio; i++) {
                float pv = h[i];
                const bool nonempty = pv > 0.f, last = (i == br - 1);
                if (last) pv = __fadd_rn(pv, tail);
                const float p = __fdiv_rn(pv, total);
                const float qq = nonempty ? q : q_empty;
                if (p == 0.f && qq == qq) continue;                      // 0 * (finite) contributes exactly 0
                const double lp = last ? log10((double)p + 1e-30) : logp[i];
                kl += (double)p * (lp - (nonempty ? lq : lq_empty));
            }
        }
        kl = warp_sum(kl);
        if (lane == 0) loss[c] = kl;
        __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int best = -1; double best_loss = 0.0;
        for (int c = 0; c < ncand; c++) if (best < 0 || loss[c] < best_loss) { best = c; best_loss = loss[c]; }
        const int s_best = (best + 1) * quant_bins;
        double hs;
        if (minmax_arena) {
            const double mn = (double)minmax_arena[2 * blockIdx.x], mx = (double)minmax_arena[2 * blockIdx.x + 1];
            hs = fmax(fabs(mx), fabs(mn)) / (double)bins;
        } else hs = (double)hist_scale_arena[blockIdx.x];
        double scale = ((double)s_best / (double)bins) * hs * ((double)bins / (double)quant_bins);
        scale = fmax(scale, min_scale);
        if (pow2) scale = pow2_round(scale, true);
        scale_out[blockIdx.x] = (float)scale;
        if (best_out) best_out[blockIdx.x] = s_best;
    }
}

// ---- MSE search: one CTA per histogram, one thread per candidate grid ----------------------------------------------------------
// TorchMSEObserver.hist_to_scale_offset (range.py:456-520) drives compute_mse_loss (hist_mse.cc:3-28) over candidate (start, step)
// grids.  The loss of a candidate is a SERIAL fp32 accumulation over the bins; each thread reproduces that order exactly, so every
// candidate's loss is bit-identical to the host function and the first minimum in enumeration order wins, as with python's stable sort.
constexpr int kMseThreads = 1024;

__device__ __forceinline__ float mse_loss_of(const float *__restrict__ h, int bins, float ftotal, int start, int step, int end) {
    float loss = 0.f;
    for (int idx = 0; idx < bins; idx++) {
        float err;
        if (idx < start) err = (float)((double)(start - idx - 1) + 0.5);
        else if (idx > end) err = (float)((double)(idx - end) + 0.5);
        else {
            const int l = (idx - start) % step, r = step - l - 1;
            if (l == r) err = (float)((double)l + 0.25);
            else { const float le = (float)((double)l + 0.5), re = (float)((double)r + 0.5); err = le < re ? le : re; }
        }
        loss = __fadd_rn(loss, __fdiv_rn(__fmul_rn(__fmul_rn(h[idx], err), err), ftotal));
    }
    return loss;
}

__global__ void __launch_bounds__(kMseThreads)
mse_search_kernel(const int32_t *__restrict__ hist_arena, int bins, const float *__restrict__ minmax_arena, int qmin, int qmax, int sym,
                  int pow2, double min_scale, int interval, float *__restrict__ scale_out, float *__restrict__ offset_out) {
    extern __shared__ float mh[];                                      // [bins] counts as fp32 (int64 -> float upstream; same value)
    __shared__ long long s_total;
    __shared__ float best_loss[kMseThreads / 32];
    __shared__ int best_idx[kMseThreads / 32];
    const int32_t *hist = hist_arena + (int64_t)blockIdx.x * bins;
    if (threadIdx.x == 0) { long long t = 0; for (int i = 0; i < bins; i++) t += hist[i]; s_total = t; }
    for (int i = threadIdx.x; i < bins; i += kMseThreads) mh[i] = (float)hist[i];
    __syncthreads();
    const float ftotal = (float)s_total;
    const double vmin = (double)minmax_arena[2 * blockIdx.x], vmax = (double)minmax_arena[2 * blockIdx.x + 1];
    const double hs = (sym ? fmax(fabs(vmax), fabs(vmin)) : (vmax - vmin)) / (double)bins;      // python doubles, range.py:294-300
    const int levels = (qmax - qmin) + 1;
    const int S = bins / levels;                                       // steps 1..S
    // candidate enumeration, in the reference's order: 0 = the min-max fallback (start 0, step S+1); then (start_i, step) row-major
    int nstarts = 1;
    if (!sym) { nstarts = 0; for (int st = 0; st < bins; st += interval) { if ((double)st * hs + vmin > 0.0) break; nstarts++; } }
    const int ncand = 1 + nstarts * S;
    float my_loss = __int_as_float(0x7F800000); int my_idx = 0x7fffffff;
    for (int c = threadIdx.x; c < ncand; c += kMseThreads) {
        int start, step, end; bool valid = true;
        if (c == 0) { start = 0; step = S + 1; end = levels * step; }
        else {
            const int si = (c - 1) / S; step = (c - 1) % S + 1; start = sym ? 0 : si * interval; end = start + levels * step;
            if (end > bins + levels) valid = false;                    // the reference `break`s the step loop here: larger steps are invalid too
        }
        if (!valid) continue;
        const float loss = mse_loss_of(mh, bins, ftotal, start, step, end);
        if (loss < my_loss || (loss == my_loss && c < my_idx)) { my_loss = loss; my_idx = c; }
    }
    // block arg-min, ties to the lowest candidate index
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ol = __shfl_xor_sync(0xffffffffu, my_loss, o); const int oi = __shfl_xor_sync(0xffffffffu, my_idx, o);
        if (ol < my_loss || (ol == my_loss && oi < my_idx)) { my_loss = ol; my_idx = oi; }
    }
    if ((threadIdx.x & 31) == 0) { best_loss[threadIdx.x >> 5] = my_loss; best_idx[threadIdx.x >> 5] = my_idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float bl = best_loss[0]; int bi = best_idx[0];
        for (int w = 1; w < kMseThreads / 32; w++) if (best_loss[w] < bl || (best_loss[w] == bl && best_idx[w] < bi)) { bl = best_loss[w]; bi = best_idx[w]; }
        int start, step;
        if (bi == 0) { start = 0; step = S + 1; } else { start = sym ? 0 : ((bi - 1) / S) * interval; step = (bi - 1) % S + 1; }
        const int end = start + levels * step;
        const double lo = sym ? -((double)end * hs) : (double)start * hs + vmin;
        const double hi = sym ? ((double)end * hs) : (double)end * hs + vmin;
        const ScaleOffset r = minmax_to_scale_offset_dev(lo, hi, qmin, qmax, sym != 0, pow2 != 0, min_scale);
        scale_out[blockIdx.x] = (float)r.scale;
        offset_out[blockIdx.x] = (float)r.offset;
    }
}

}  // namespace ppqb

using namespace ppqb;

extern "C" {

int ppq_b200_minmax_to_scale_offset(const float *mins, const float *maxs, int64_t count, int64_t stride, int qmin, int qmax,
                                    int symmetrical, int power_of_2, double min_scale, float *scale, float *offset, void *stream) {
    if (count <= 0 || stride <= 0 || !mins || !maxs || !scale || !offset || qmax <= qmin) return (int)cudaErrorInvalidValue;
    minmax_to_scale_offset_kernel<<<(int)((count + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        mins, maxs, count, stride, qmin, qmax, symmetrical, power_of_2, min_scale, scale, offset);
    return (int)cudaGetLastError();
}

int ppq_b200_hist_scale_from_minmax(const float *minmax_arena, int64_t count, int symmetrical, int64_t bins, float *hist_scale_arena,
                                    void *stream) {
    if (count <= 0 || bins <= 0 || !minmax_arena || !hist_scale_arena) return (int)cudaErrorInvalidValue;
    hist_scale_kernel<<<(int)((count + 127) / 128), 128, 0, (cudaStream_t)stream>>>(minmax_arena, count, symmetrical, bins, hist_scale_arena);
    return (int)cudaGetLastError();
}

int ppq_b200_kl_search(const int32_t *hist_arena, int64_t count, int64_t bins, const float *hist_scale_arena,
                       const float *minmax_arena, int num_of_bits, int power_of_2, double min_scale, float *scale_out, int32_t *best_bin_range_out, void *stream) {
    if (count <= 0 || count > 0x7fffffffLL || !hist_arena || (!hist_scale_arena && !minmax_arena) || !scale_out)
        return (int)cudaErrorInvalidValue;
    if (num_of_bits < 2 || num_of_bits > 16) return (int)cudaErrorInvalidValue;
    const int64_t qb = 1ll << (num_of_bits - 1);
    if (bins < qb || bins > 16384) return (int)cudaErrorInvalidValue;  // OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE: any multiple of the quant bins works
    if (bins <= kKlMemoBins && bins % qb == 0 && variant_of(kVarKlSearch) == 0) {        // one warp per candidate
        const size_t ncand = (size_t)(bins / qb);
        const size_t plen = (size_t)(bins + 1 > kKlwThreads ? bins + 1 : kKlwThreads);
        const size_t smem_w = (((size_t)bins * 4 + 7) & ~(size_t)7) + plen * 8 + (size_t)bins * 8 + ((ncand + 1) & ~(size_t)1) * 8 +
                              (size_t)(kKlwThreads / 32) * (size_t)qb * 4;
        if (smem_w <= 220 * 1024) {
            if (smem_w > 48 * 1024 && cudaFuncSetAttribute(kl_search_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024) != cudaSuccess)
                return (int)cudaGetLastError();
            kl_search_warp_kernel<<<(int)count, kKlwThreads, smem_w, (cudaStream_t)stream>>>(hist_arena, (int)bins, hist_scale_arena, minmax_arena,
                                                                                               num_of_bits, power_of_2, min_scale, scale_out, best_bin_range_out);
            return (int)cudaGetLastError();
        }
    }
    const size_t pre_len = (size_t)(bins + 1 > kKlThreads ? bins + 1 : kKlThreads);
    size_t smem = (((size_t)bins * 4 + 7) & ~(size_t)7) + pre_len * 8 + (((size_t)qb * 4 + 7) & ~(size_t)7);
    if (bins <= kKlMemoBins) smem += (size_t)(qb + bins) * 8;          // memoised logarithms (see the kernel)
    // > 48 KB of dynamic shared memory is an opt-in PER DEVICE: set it on every launch (a process-wide flag would leave the second GPU of a
    // process without it; the call is a few hundred nanoseconds against a kernel of >= 100 us)
    if (smem > 48 * 1024 && cudaFuncSetAttribute(kl_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024) != cudaSuccess)
        return (int)cudaGetLastError();
    kl_search_kernel<<<(int)count, kKlThreads, smem, (cudaStream_t)stream>>>(hist_arena, (int)bins, hist_scale_arena, minmax_arena,
                                                                               num_of_bits, power_of_2, min_scale, scale_out, best_bin_range_out);
    return (int)cudaGetLastError();
}

int ppq_b200_mse_search(const int32_t *hist_arena, int64_t count, int64_t bins, const float *minmax_arena, int qmin, int qmax,
                        int symmetrical, int power_of_2, double min_scale, int interval, float *scale_out, float *offset_out, void *stream) {
    if (count <= 0 || count > 0x7fffffffLL || !hist_arena || !minmax_arena || !scale_out || !offset_out || qmax <= qmin || interval <= 0)
        return (int)cudaErrorInvalidValue;
    const int64_t levels = (int64_t)qmax - qmin + 1;
    if (bins < levels || bins > 11264) return (int)cudaErrorInvalidValue;       // at least one step; fp32 copy of the bins within 44 KB of smem
    mse_search_kernel<<<(int)count, kMseThreads, (size_t)bins * sizeof(float), (cudaStream_t)stream>>>(
        hist_arena, (int)bins, minmax_arena, qmin, qmax, symmetrical, power_of_2, min_scale, interval, scale_out, offset_out);
    return (int)cudaGetLastError();
}

}  // extern "C"
