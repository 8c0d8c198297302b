/*
 * ppq_b200.h -- C ABI of libppq_b200.so: H100 (sm_90a) kernels for the PPQ quantization-simulation hot path.
 *
 * This is the drop-in boundary.  Every entry point replaces one function of the reference's native extension
 * `PPQ_Cuda_Impls` (pybind table: /root/reference/ppq/csrc/export.cc:8-34, bound by ppq/core/ffi.py:56-350);
 * the reference file:line each one replaces is cited on the declaration.  The torch/pybind layer on top
 * (ppq_b200/csrc/torch_binding.cc) re-creates the reference's tensor checks, allocation and exception text and
 * exports the same 20 names with the same positional signatures; INTEGRATION.md shows how a PPQ maintainer
 * installs it (CUDA_COMPLIER.__CUDA_EXTENTION__ = ppq_b200.extension()).
 *
 * Conventions (all functions unless stated otherwise)
 *   - plain pointers and sizes, no torch types; all tensors fp32 (the `_dt` entries also take fp16 / bf16 values),
 *     flat, contiguous, DEVICE memory;
 *   - `scale` / `offset` are DEVICE pointers (1 element per-tensor, C elements per-channel), exactly what the
 *     reference passes (scale/offset tensors live on the executor device);
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - asynchronous: kernels are enqueued on `stream`, nothing synchronises, nothing allocates;
 *   - return value: 0 on success, otherwise a cudaError_t code (invalid arguments -> cudaErrorInvalidValue = 1);
 *     ppq_b200_error_string() turns it into text;
 *   - `rounding` ids follow ppq/csrc/cuda/common.cuh:17-24: 0 HALF_EVEN, 1 HALF_UP, 2 HALF_DOWN,
 *     3 HALF_TOWARDS_ZERO, 4 HALF_FAR_FROM_ZERO, 5 TO_NEAR_INT, 6 UP, 7 DOWN;
 *   - per-channel layout: the tensor is [outer, C, epc] row-major, channel of flat index i is (i / epc) % C
 *     (epc = product of the dims after channel_axis: floating.cu:118-122, linear.cu:213).
 */
#ifndef PPQ_B200_H_
#define PPQ_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PPQ_B200_API __attribute__((visibility("default")))
#else
#define PPQ_B200_API
#endif

/* ---- element types ------------------------------------------------------------------------------ */
/* The `_dt` entries take `const void *x` plus one of these codes.  For fp16 / bf16 every statistic equals the fp32 one on the exact
 * upcast x.float(); a fake-quantised output has the input's type and holds the fp32 result rounded once to nearest even.
 * Scales, offsets and statistics stay fp32.  Any other code returns cudaErrorInvalidValue before a launch. */
#define PPQ_B200_F32  0
#define PPQ_B200_F16  1
#define PPQ_B200_BF16 2

/* ---- library ----------------------------------------------------------------------------------- */
PPQ_B200_API int         ppq_b200_abi_version(void);              /* bumps when a signature changes */
PPQ_B200_API const char *ppq_b200_error_string(int status);
PPQ_B200_API const char *ppq_b200_build_info(void);               /* "sm_90a nvcc 12.9 ..." */
/* Runtime tuning knob used by bench/profiling to select a kernel variant (0 = default). */
PPQ_B200_API int         ppq_b200_set_variant(const char *kernel, int variant);
PPQ_B200_API int         ppq_b200_get_variant(const char *kernel);

/* ---- integer fake-quant: y = float(clip(round(x / s) + o, qmin, qmax) - o) * s ------------------ */
/* replaces QuantizeTensor_LT, ppq/csrc/cuda/linear.cu:38-130 (ffi.py:78-90 CUDA.LinearQuantize_T). */
PPQ_B200_API int ppq_b200_linear_quant_t(const float *x, float *y, int64_t n,
                                         const float *scale, const float *offset,
                                         int qmin, int qmax, int rounding, void *stream);
/* replaces QuantizeTensor_LC, ppq/csrc/cuda/linear.cu:132-233 (ffi.py:92-103 CUDA.LinearQuantize_C). */
PPQ_B200_API int ppq_b200_linear_quant_c(const float *x, float *y, int64_t n, int64_t epc, int C,
                                         const float *scale, const float *offset,
                                         int qmin, int qmax, int rounding, void *stream);
/* Integer-emitting variants (no dequantise): device twin of PPQLinearQuant_toInt,
 * ppq/quantization/qfunction/linear.py:218-238 (torch-only upstream; SURVEY §8f-4).
 * out_bits: 8 -> int8 (or uint8 when qmin >= 0 and qmax > 127), 32 -> int32. */
PPQ_B200_API int ppq_b200_linear_quant_t_toint(const float *x, void *q, int out_bits, int64_t n,
                                               const float *scale, const float *offset,
                                               int qmin, int qmax, int rounding, void *stream);
PPQ_B200_API int ppq_b200_linear_quant_c_toint(const float *x, void *q, int out_bits, int64_t n, int64_t epc, int C,
                                               const float *scale, const float *offset,
                                               int qmin, int qmax, int rounding, void *stream);
/* The four entries above for an input of element type `dtype` (PPQ_B200_F32 / _F16 / _BF16); `y` has the input's type. */
PPQ_B200_API int ppq_b200_linear_quant_t_dt(const void *x, int dtype, void *y, int64_t n,
                                            const float *scale, const float *offset,
                                            int qmin, int qmax, int rounding, void *stream);
PPQ_B200_API int ppq_b200_linear_quant_c_dt(const void *x, int dtype, void *y, int64_t n, int64_t epc, int C,
                                            const float *scale, const float *offset,
                                            int qmin, int qmax, int rounding, void *stream);
PPQ_B200_API int ppq_b200_linear_quant_t_toint_dt(const void *x, int dtype, void *q, int out_bits, int64_t n,
                                                  const float *scale, const float *offset,
                                                  int qmin, int qmax, int rounding, void *stream);
PPQ_B200_API int ppq_b200_linear_quant_c_toint_dt(const void *x, int dtype, void *q, int out_bits, int64_t n, int64_t epc, int C,
                                                  const float *scale, const float *offset,
                                                  int qmin, int qmax, int rounding, void *stream);

/* Every per-channel weight of a network in ONE launch (the executor re-quantises all Conv/Gemm weights on every forward until
 * they are baked: ppq/executor/torch.py:516-518; ParameterBakingPass, optim/baking.py:34-47).  Descriptors in DEVICE memory. */
typedef struct {
    const float *x;        /* weight (fp32; the table's type in the `_dt` entry) */
    float       *y;        /* fake-quantised output (!= x), same type as x */
    const float *scale;    /* [C] */
    const float *offset;   /* [C] */
    int64_t      n;        /* elements                        */
    int64_t      epc;      /* elements per channel            */
    int32_t      C;        /* channels                        */
    int32_t      pad_;
} ppq_b200_lc_desc;
/* count <= 4096 tensors per call, every n <= 2^31 - 1; max_n = the largest n of the table (sizes the grid). */
PPQ_B200_API int ppq_b200_multi_linear_quant_c(const ppq_b200_lc_desc *descs, int count, int64_t max_n,
                                               int qmin, int qmax, int rounding, void *stream);
/* The same for a table whose weights all have element type `dtype`: `x` and `y` of every descriptor point at elements of that type
 * (the struct keeps its layout; the element type is one per table, not per descriptor), `y` holds the fp32 result on x.float()
 * rounded once to nearest even -- what ppq_b200_linear_quant_c_dt writes for that weight.  scale / offset stay fp32. */
PPQ_B200_API int ppq_b200_multi_linear_quant_c_dt(const ppq_b200_lc_desc *descs, int count, int64_t max_n, int dtype,
                                                  int qmin, int qmax, int rounding, void *stream);

/* QuantizeTensor_LT (linear.cu:88-130) for a table of tensors in ONE launch, each with its own (scale, offset): the per-tensor
 * activation configs of a quantised graph (executor/torch.py:516-518, 541-543 call the op ~100x per forward on tensors of a few hundred KB,
 * where a launch costs more than the kernel).  One descriptor per tensor, in DEVICE memory. */
typedef struct {
    const float *x;        /* input  (borrowed) */
    float       *y;        /* output (caller-allocated, may not alias x) */
    const float *scale;    /* [1] */
    const float *offset;   /* [1] */
    int64_t      n;        /* elements */
} ppq_b200_lt_desc;
PPQ_B200_API int ppq_b200_multi_linear_quant_t(const ppq_b200_lt_desc *descs, int count, int64_t max_n,
                                               int qmin, int qmax, int rounding, void *stream);

/* ---- low-precision float fake-quant (FP8 E4M3 default; E in 1..5 and 2^(E-1)+M-2 in 0..30: E4M3, E5M2, E5M10 ...) --------------- */
/* replaces QuantizeTensor_FT, ppq/csrc/cuda/floating.cu:36-75 with QuantizeScalarFloating,
 * common.cuh:154-226 (ffi.py:272-288 CUDA.FloatingQuantize_T).  Reference tie rule kept (ties toward zero in the
 * normal range), so this is NOT cvt.rn.satfinite.e4m3x2. */
PPQ_B200_API int ppq_b200_float_quant_t(const float *x, float *y, int64_t n,
                                        const float *scale, const float *offset,
                                        int exponent, int mantissa, float clip_min, float clip_max,
                                        int rounding, void *stream);
/* replaces QuantizeTensor_FC, ppq/csrc/cuda/floating.cu:77-131 (ffi.py:290-306 CUDA.FloatingQuantize_C). */
PPQ_B200_API int ppq_b200_float_quant_c(const float *x, float *y, int64_t n, int64_t epc, int C,
                                        const float *scale, const float *offset,
                                        int exponent, int mantissa, float clip_min, float clip_max,
                                        int rounding, void *stream);
/* The two entries above for an input of element type `dtype`; `y` has the input's type. */
PPQ_B200_API int ppq_b200_float_quant_t_dt(const void *x, int dtype, void *y, int64_t n,
                                           const float *scale, const float *offset,
                                           int exponent, int mantissa, float clip_min, float clip_max,
                                           int rounding, void *stream);
PPQ_B200_API int ppq_b200_float_quant_c_dt(const void *x, int dtype, void *y, int64_t n, int64_t epc, int C,
                                           const float *scale, const float *offset,
                                           int exponent, int mantissa, float clip_min, float clip_max,
                                           int rounding, void *stream);

/* ---- calibration collectors ---------------------------------------------------------------------- */
/* Fused single-pass min+max.  Replaces the two torch reductions of TorchMinMaxObserver.observe,
 * ppq/quantization/observer/range.py:85-100 (value.min(), value.max(); per-channel :93-98).
 * `minmax` is DEVICE float[2] = {min, max} that is ACCUMULATED into (initialise with
 * ppq_b200_minmax_init -> {+inf, -inf}); NaN inputs poison both, as torch.min/max do. */
PPQ_B200_API int ppq_b200_minmax_init(float *mins, float *maxs, int64_t count, void *stream);
PPQ_B200_API int ppq_b200_minmax_t(const float *x, int64_t n, float *minmax, void *stream);
/* per channel: mins[C], maxs[C] accumulated. */
PPQ_B200_API int ppq_b200_minmax_c(const float *x, int64_t n, int64_t epc, int C,
                                   float *mins, float *maxs, void *stream);

/* replaces Histogram_T, ppq/csrc/cuda/sort.cu:75-111 (ffi.py:136-145): hist[floor(|x| / hist_scale)] += 1,
 * bins beyond the last are dropped (clip_outliers) or clamped.  `hist` is DEVICE int32[bins], accumulated in place. */
PPQ_B200_API int ppq_b200_histogram_t(const float *x, int64_t n, float hist_scale, int clip_outliers,
                                      int32_t *hist, int64_t bins, void *stream);
/* replaces Histogram_Asymmetric_T, sort.cu:113-165 (ffi.py:147-157): hist_scale = (max - min) / bins in fp32,
 * b = floor((x - min) / hist_scale), both tails dropped or clamped. */
PPQ_B200_API int ppq_b200_histogram_asym_t(const float *x, int64_t n, float vmin, float vmax, int clip_outliers,
                                           int32_t *hist, int64_t bins, void *stream);
/* replaces Histogram_C, sort.cu:167-218 (ffi.py:159-169): per-channel symmetric histogram, hist[C][bins]. */
PPQ_B200_API int ppq_b200_histogram_c(const float *x, int64_t n, int64_t epc, int C, float hist_scale,
                                      int clip_outliers, int32_t *hist, int64_t bins, void *stream);
/* Same as ppq_b200_histogram_t but hist_scale is read from DEVICE memory (written by
 * ppq_b200_hist_scale_from_minmax), so phase 2 of the calibration needs no host round-trip. */
PPQ_B200_API int ppq_b200_histogram_t_dscale(const float *x, int64_t n, const float *hist_scale_dev, int clip_outliers,
                                             int32_t *hist, int64_t bins, void *stream);
/* min/max and the two histograms above for an input of element type `dtype`: the same statistics as on the fp32 upcast. */
PPQ_B200_API int ppq_b200_minmax_t_dt(const void *x, int dtype, int64_t n, float *minmax, void *stream);
PPQ_B200_API int ppq_b200_minmax_c_dt(const void *x, int dtype, int64_t n, int64_t epc, int C,
                                      float *mins, float *maxs, void *stream);
PPQ_B200_API int ppq_b200_histogram_asym_t_dt(const void *x, int dtype, int64_t n, float vmin, float vmax, int clip_outliers,
                                              int32_t *hist, int64_t bins, void *stream);
PPQ_B200_API int ppq_b200_histogram_t_dscale_dt(const void *x, int dtype, int64_t n, const float *hist_scale_dev, int clip_outliers,
                                                int32_t *hist, int64_t bins, void *stream);

/* replaces Quantile_T, sort.cu:6-20, 42-59 (ffi.py:171-176): out[0] = sorted[clip(rn(n*q))], out[1] = sorted[clip(rn(n*(1-q)))],
 * found by an exact radix select on the order-preserving key (no clone, no full sort; same element bit for bit): two streaming passes
 * over the tensor (top-digit histogram, then compaction of the two selected buckets) and a finish over the compacted keys; a third
 * pass only when a selected bucket does not fit the workspace and holds more than one distinct value.  Tensors of >= 8 Mi elements
 * first try to get away with ONE pass: thresholds derived from 16 Ki sampled elements decide which keys are compacted during the
 * first pass; if they turn out not to contain the wanted order statistics, the regular passes follow (the result is exact either way).
 * `workspace` is DEVICE scratch of ppq_b200_quantile_workspace_bytes() bytes. */
PPQ_B200_API int64_t ppq_b200_quantile_workspace_bytes(void);
PPQ_B200_API int ppq_b200_quantile_t(const float *x, int64_t n, float q, float *out2, void *workspace, void *stream);
/* the same with a one-slot `guess` buffer (see ppq_b200_multi_quantile_t): consecutive calls on batches of one activation -- what
 * TorchPercentileObserver.observe does (range.py:338-349) -- read the tensor once when the previous call's thresholds still hold. */
PPQ_B200_API int ppq_b200_quantile_t_guess(const float *x, int64_t n, float q, float *out2, void *workspace, uint32_t *guess, void *stream);
/* both of the above for an input of element type `dtype` (guess may be NULL): the selected values are the exact fp32 upcasts. */
PPQ_B200_API int ppq_b200_quantile_t_dt(const void *x, int dtype, int64_t n, float q, float *out2, void *workspace, uint32_t *guess,
                                        void *stream);
/* replaces Isotone_T, sort.cu:23-40, 61-73: out4 = {sorted[n-1], sorted[n-2], sorted[0], sorted[1]} (same workspace). */
PPQ_B200_API int ppq_b200_isotone_t(const float *x, int64_t n, float *out4, void *workspace, void *stream);

/* ---- multi-tensor collectors (one launch over a table of tensors; the H100-native calibration path) ---------
 * A descriptor lives in DEVICE memory.  `slot` selects the statistics slot in the arena:
 *   minmax arena: float[2 * slots]  ({min, max} per slot);   hist arena: int32[slots * bins];
 *   hist_scale arena: float[slots].
 * Both keep a prefix of the table's sizes in shared memory ((count + 1) x 8 bytes next to a 64 KB staging ring and, for the histogram,
 * (bins + 1) x 4 bytes of private counters); a table that does not fit the device's shared memory per block is rejected.
 * The `_dt` entries take a table whose tensors all have element type `dtype` (one per table, not per descriptor: `x` of every
 * descriptor points at elements of that type, which may start at any element-aligned address); every statistic equals, bit for bit,
 * what the fp32 entry writes for the same table over the upcasts x.float().  A mixed set of tensors is served by one call per type. */
typedef struct {
    const float *x;      /* device pointer to the tensor (elements of the table's type in the `_dt` entries) */
    int64_t      n;      /* elements */
    int32_t      slot;   /* statistics slot */
    int32_t      pad_;
} ppq_b200_tensor_desc;

PPQ_B200_API int ppq_b200_multi_minmax_t(const ppq_b200_tensor_desc *descs, int count, int64_t max_n,
                                         float *minmax_arena, void *stream);
PPQ_B200_API int ppq_b200_multi_histogram_t(const ppq_b200_tensor_desc *descs, int count, int64_t max_n,
                                            const float *hist_scale_arena, int clip_outliers,
                                            int32_t *hist_arena, int64_t bins, void *stream);
PPQ_B200_API int ppq_b200_multi_minmax_t_dt(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, int dtype,
                                            float *minmax_arena, void *stream);
PPQ_B200_API int ppq_b200_multi_histogram_t_dt(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, int dtype,
                                               const float *hist_scale_arena, int clip_outliers,
                                               int32_t *hist_arena, int64_t bins, void *stream);
/* Quantile_T (sort.cu:6-20, 42-59) for a table of tensors, one launch per pass: what TorchPercentileObserver.observe
 * (ppq/quantization/observer/range.py:338-349) asks for once per observed tensor and batch.  Tensor i writes
 * out[slot_i * out_stride + {0, 1}] = {sorted[clip(rn(n q))], sorted[clip(rn(n (1 - q)))]}.  `cap` = keys of a selected bucket the
 * workspace can hold per rank (bigger buckets are refined by a further streaming pass instead);
 * `workspace` is DEVICE scratch of ppq_b200_multi_quantile_workspace_bytes(count, cap) bytes.
 * `guess` (optional, DEVICE, ppq_b200_quantile_guess_words() uint32 per statistics slot, initialised once by ppq_b200_quantile_guess_init and
 * then owned by this function) makes consecutive calls on the same slots speculative: keys beyond the thresholds remembered from the
 * previous call are compacted during the first pass, and when they contain the requested order statistics (the usual case for consecutive
 * calibration batches of one activation) the tensor is read ONCE.  A wrong guess only costs the regular second pass; results are always
 * the exact order statistics.  An entry with n = 0 has no order statistics: its two output values and its guess words are left as they are. */
PPQ_B200_API int64_t ppq_b200_multi_quantile_workspace_bytes(int count, int64_t cap);
PPQ_B200_API int64_t ppq_b200_quantile_guess_words(void);
PPQ_B200_API int ppq_b200_quantile_guess_init(uint32_t *guess, int64_t slots, void *stream);
PPQ_B200_API int ppq_b200_multi_quantile_t(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, float q,
                                           float *out, int64_t out_stride, void *workspace, int64_t cap, uint32_t *guess, void *stream);
/* the same for a table of element type `dtype`: workspace size, `cap` and the guess words are those of the fp32 entry. */
PPQ_B200_API int ppq_b200_multi_quantile_t_dt(const ppq_b200_tensor_desc *descs, int count, int64_t max_n, int dtype, float q,
                                              float *out, int64_t out_stride, void *workspace, int64_t cap, uint32_t *guess, void *stream);

/* ---- quantisation error analysis ----------------------------------------------------------------------------- */
/* One (prediction, reference) pair of a paired-moment table: `rows` sample rows of `row_len` elements each, contiguous one after the other
 * from `pred` and from `real` (a sample is the outermost dimension, or the whole tensor of a 1-d pair: ppq/quantization/measure/norm.py:36-38).
 * Row i of the pair writes out row out_row0 + i.  Lives in DEVICE memory; pred and real may alias. */
typedef struct {
    const void *pred;      /* elements of the table's type */
    const void *real;
    int64_t     rows;
    int64_t     row_len;
    int64_t     out_row0;
} ppq_b200_pair_desc;
/* For every row of every pair, out[row] = {sum (p - r)^2, sum r^2, sum p^2, sum p * r} in fp64 (out: DEVICE double[total_rows][4], 16-byte
 * aligned, rows no pair covers are left as they are; the row ranges of the pairs must not overlap).  The products are exact in fp64 and the
 * only roundings are the additions (sum (p - r)^2 also rounds p - r when the exponents of p and r are more than 29 apart); the result is
 * bit-identical from run to run and under CUDA-graph replay.  The longest chain of additions a term goes through is 74 + ceil(row_len / 16384).
 * NaN and +-inf propagate as IEEE fp64 arithmetic gives them.  Every byte is read once.
 * total_elems >= the sum of rows * row_len over the table; `workspace`: DEVICE scratch of
 * ppq_b200_multi_paired_moments_workspace_bytes(total_rows, total_elems) bytes, 16-byte aligned.  count <= 2048; count == 0 or
 * total_rows == 0 writes nothing.  A table the arguments do not describe (negative fields, an out row range outside [0, total_rows), more
 * elements than total_elems) writes NaN into all total_rows rows. */
PPQ_B200_API int64_t ppq_b200_multi_paired_moments_workspace_bytes(int64_t total_rows, int64_t total_elems);
PPQ_B200_API int ppq_b200_multi_paired_moments(const ppq_b200_pair_desc *descs, int count, int64_t total_rows, int64_t total_elems,
                                               double *out, void *workspace, void *stream);
/* the same for a table whose pairs all have element type `dtype` (p and r alike): the moments of the exact upcasts. */
PPQ_B200_API int ppq_b200_multi_paired_moments_dt(const ppq_b200_pair_desc *descs, int count, int64_t total_rows, int64_t total_elems,
                                                  int dtype, double *out, void *workspace, void *stream);

/* ---- scale / offset search on the device ---------------------------------------------------------------------- */
/* replaces minmax_to_scale_offset, ppq/quantization/observer/range.py:22-75, vectorised over `count` ranges
 * (tensors or channels); arithmetic in fp64 like the Python original, results stored as fp32. */
PPQ_B200_API int ppq_b200_minmax_to_scale_offset(const float *mins, const float *maxs, int64_t count, int64_t stride,
                                                 int qmin, int qmax, int symmetrical, int power_of_2, double min_scale,
                                                 float *scale, float *offset, void *stream);
/* TorchHistObserver.render_quantization_config phase 1, range.py:291-301: hist_scale = range / bins (fp64 -> fp32). */
PPQ_B200_API int ppq_b200_hist_scale_from_minmax(const float *minmax_arena, int64_t count, int symmetrical, int64_t bins,
                                                 float *hist_scale_arena, void *stream);
/* replaces TorchHistObserver.hist_to_scale_offset (KL search), range.py:190-282 + measure/statistic.py:3-12,
 * for `count` histograms of `bins` bins in one launch.  scale_out[i] (fp32); offset is always 0 (symmetric only). */
PPQ_B200_API int ppq_b200_kl_search(const int32_t *hist_arena, int64_t count, int64_t bins, const float *hist_scale_arena,
                                    const float *minmax_arena /* nullable: when given, hist_scale is re-derived in fp64
                                    from {min,max} exactly like the Python original (range.py:294-300) */,
                                    int num_of_bits, int power_of_2, double min_scale,
                                    float *scale_out, int32_t *best_bin_range_out, void *stream);
/* replaces compute_mse_loss, ppq/csrc/cpu/hist_mse.cc:3-28 (ffi.py:263-270).  HOST function on HOST memory, exactly
 * like the reference's (it is a serial fp32 accumulation over <= 2048 bins). */
PPQ_B200_API float ppq_b200_compute_mse_loss(const int64_t *hist, int64_t nbins, int start, int step, int end);
/* Device MSE grid search: TorchMSEObserver.hist_to_scale_offset (range.py:456-520) over `count` histograms in one launch; each
 * candidate's loss is the bit-exact serial fp32 accumulation of compute_mse_loss.  minmax_arena: {min,max} per histogram. */
PPQ_B200_API int ppq_b200_mse_search(const int32_t *hist_arena, int64_t count, int64_t bins, const float *minmax_arena,
                                     int qmin, int qmax, int symmetrical, int power_of_2, double min_scale, int interval,
                                     float *scale_out, float *offset_out, void *stream);

/* ---- training-pass helpers that share the scalar quantizer ("next" rows, SURVEY §8f) ---------------------------- */
/* replaces QuantizeTensor_LT_B, linear.cu:235-324: grad_x (STE with clip mask) and grad_s (1 float; zeroed here). */
PPQ_B200_API int ppq_b200_linear_quant_t_backward(const float *x, const float *dy, int64_t n,
                                                  const float *scale, const float *offset, int qmin, int qmax, int rounding,
                                                  float *grad_x, float *grad_s, void *stream);
/* replaces QuantizeTensor_LC_B, linear.cu:326-433: grad_s has C floats. */
PPQ_B200_API int ppq_b200_linear_quant_c_backward(const float *x, const float *dy, int64_t n, int64_t epc, int C,
                                                  const float *scale, const float *offset, int qmin, int qmax, int rounding,
                                                  float *grad_x, float *grad_s, void *stream);
/* replace QuantizeTensor_FT_B / _FC_B, floating.cu:133-331. */
PPQ_B200_API int ppq_b200_float_quant_t_backward(const float *x, const float *dy, int64_t n, const float *scale, const float *offset,
                                                 int exponent, int mantissa, float clip_min, float clip_max, int rounding,
                                                 float *grad_x, float *grad_s, void *stream);
PPQ_B200_API int ppq_b200_float_quant_c_backward(const float *x, const float *dy, int64_t n, int64_t epc, int C,
                                                 const float *scale, const float *offset,
                                                 int exponent, int mantissa, float clip_min, float clip_max, int rounding,
                                                 float *grad_x, float *grad_s, void *stream);
/* replace TensorClip_T / _C, train.cu:34-113: out = CLIP(value, reference - limit[c], reference + limit[c]). */
PPQ_B200_API int ppq_b200_tensor_clip_t(const float *value, const float *reference, const float *limit, int64_t n, float *out, void *stream);
PPQ_B200_API int ppq_b200_tensor_clip_c(const float *value, const float *reference, const float *limit, int64_t n, int64_t epc, int C,
                                        float *out, void *stream);
/* replace RoundingLoss_LT / _LC (per_channel = 0 / 1), train.cu:115-176, 224-283, and their _B, :178-222, 285-338. */
PPQ_B200_API int ppq_b200_rounding_loss(const float *x, int64_t n, int64_t epc, int C, int per_channel,
                                        const float *scale, const float *offset, int qmin, int qmax, int rounding,
                                        float *loss, void *stream);
PPQ_B200_API int ppq_b200_rounding_loss_backward(const float *x, const float *dy, int64_t n, int64_t epc, int C, int per_channel,
                                                 const float *scale, const float *offset, int qmin, int qmax, int rounding,
                                                 float *grad_x, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PPQ_B200_H_ */
