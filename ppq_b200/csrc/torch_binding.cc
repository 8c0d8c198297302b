// torch_binding.cc -- the torch / pybind11 face of libppq_b200: a drop-in for the reference's native extension
// `PPQ_Cuda_Impls` (/root/reference/ppq/csrc/export.cc:8-34).
//
// Same 20 exported names, same positional signatures, same tensor checks and exception texts
// (CheckTensor, ppq/csrc/cuda/common.cuh:78-86), same ownership rules (inputs borrowed, outputs freshly allocated with
// at::empty_like, `hist` accumulated in place).  Everything heavy is forwarded to the C ABI in include/ppq_b200.h with the
// tensor's raw pointers and the current CUDA stream; this file contains no kernels.
// Differences from the reference, on purpose: a CUDAGuard on the value's device (the reference assumes device 0),
// epc computed from the trailing sizes instead of stride(channel_axis) (safe for size-1 dims), and a loud error
// for CPU tensors instead of a crash.
//
// Extra names (not in the reference table) expose the H100-native calibration path: fused min/max, device-resident
// hist_scale, multi-tensor collectors and the on-device scale search.  ppq_b200/ffi.py wraps both sets.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <stdexcept>
#include <string>
#include <vector>

#include "ppq_b200.h"

using at::Tensor;

namespace {

struct KernelFailure : public std::runtime_error { using std::runtime_error::runtime_error; };

void CheckTensor(const Tensor &t, c10::ScalarType type, const char *name) {         // (const char*: no std::string is built on the success path)
    if (at::typeMetaToScalarType(t.dtype()) != type) throw KernelFailure(std::string("Kernel Failure, Invalid dtype of Input tensor: ") + name);
    if (t.numel() == 0) throw KernelFailure(std::string("Kernel Failure, Tensor is empty: ") + name);
    if (!t.is_cuda()) throw KernelFailure(std::string("Kernel Failure, Tensor is not on a CUDA device: ") + name);
}
// A value tensor of fp32, fp16 or bf16 (half_only: fp16 or bf16); returns its element-type code in the C ABI.
int CheckValue(const Tensor &t, bool half_only) {
    const auto st = at::typeMetaToScalarType(t.dtype());
    const int code = st == at::kHalf ? PPQ_B200_F16 : st == at::kBFloat16 ? PPQ_B200_BF16 : (st == at::kFloat && !half_only) ? PPQ_B200_F32 : -1;
    if (code < 0)
        throw KernelFailure(std::string("Kernel Failure, Invalid dtype of Input tensor: ") +
                            (half_only ? "Value(Expect to be FP16 or BF16)" : "Value(Expect to be FP32, FP16 or BF16)"));
    if (t.numel() == 0) throw KernelFailure("Kernel Failure, Tensor is empty: Value");
    if (!t.is_cuda()) throw KernelFailure("Kernel Failure, Tensor is not on a CUDA device: Value");
    return code;
}
void CheckStatus(int status, const char *what) {
    if (status != 0) throw KernelFailure(std::string("Kernel Failure, ") + what + ": " + ppq_b200_error_string(status));
}
void CheckSize(const Tensor &t) {
    if (t.numel() > 0x7fffffffLL) throw KernelFailure("There are too many element in your tensor(more than 2*10^9)");
}
void *Stream() { return (void *)at::cuda::getCurrentCUDAStream().stream(); }
// Per-TENSOR operators are order-independent (element-wise maps, reductions, histograms, order statistics): any dense layout (e.g. a
// channels_last activation) is processed in storage order, without the NCHW copy `.contiguous()` would make; at::empty_like keeps the strides.
Tensor Dense(const Tensor &t) { return t.is_non_overlapping_and_dense() ? t : t.contiguous(); }
// Operators that RETURN a tensor keep the reference's layout contract (output = empty_like of the contiguous value, linear.cu:106-112) except for
// the channels_last memory formats, where -- like torch's own element-wise operators -- the format is preserved instead of copying to NCHW.
Tensor DenseFormat(const Tensor &t) {
    if (t.is_contiguous()) return t;
    if ((t.dim() == 4 && t.is_contiguous(at::MemoryFormat::ChannelsLast)) || (t.dim() == 5 && t.is_contiguous(at::MemoryFormat::ChannelsLast3d))) return t;
    return t.contiguous();
}
const float *F(const Tensor &t) { return t.data_ptr<float>(); }

struct Geometry { int64_t epc; int C; };
Geometry ChannelGeometry(const Tensor &v, int64_t axis) {
    const int64_t nd = v.dim();
    if (axis < 0) axis += nd;
    if (axis < 0 || axis >= nd) throw KernelFailure("Kernel Failure, channel_axis is out of range.");
    int64_t epc = 1;
    for (int64_t a = nd - 1; a > axis; a--) epc *= v.size(a);
    return {epc, (int)v.size(axis)};
}
void CheckChannelParams(const Tensor &scale, const Tensor &offset, int C) {
    if (scale.numel() != C || offset.numel() != C)
        throw KernelFailure("Kernel Failure, scale / offset must hold one value per channel.");
}

// ---------------------------------------------------------------- integer fake-quant (linear.h:3-10)
Tensor QuantizeTensor_LT(const Tensor &value, const Tensor &scale, const Tensor &offset, const int clip_min, const int clip_max,
                         const int rounding) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = DenseFormat(value);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_linear_quant_t(F(v), out.data_ptr<float>(), v.numel(), F(scale), F(offset), clip_min, clip_max, rounding,
                                        Stream()), "QuantizeTensor_LT");
    return out;
}

Tensor QuantizeTensor_LC(const Tensor &value, const Tensor &scale, const Tensor &offset, const int clip_min, const int clip_max,
                         const int channel_axis, const int rounding) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    auto s = scale.contiguous(), o = offset.contiguous();
    const Geometry g = ChannelGeometry(v, channel_axis);
    CheckChannelParams(s, o, g.C);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_linear_quant_c(F(v), out.data_ptr<float>(), v.numel(), g.epc, g.C, F(s), F(o), clip_min, clip_max, rounding,
                                        Stream()), "QuantizeTensor_LC");
    return out;
}

// device twin of PPQLinearQuant_toInt (ppq/quantization/qfunction/linear.py:218-238); channel_axis < -100 means per-tensor
Tensor QuantizeTensor_toInt(const Tensor &value, const Tensor &scale, const Tensor &offset, const int clip_min, const int clip_max,
                            const int channel_axis, const int rounding, const int out_bits) {
    const int dt = CheckValue(value, false);
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    auto s = scale.contiguous(), o = offset.contiguous();
    const auto dtype = out_bits == 32 ? at::kInt : ((clip_min >= 0 && clip_max > 127) ? at::kByte : at::kChar);
    Tensor out = at::empty(v.sizes(), v.options().dtype(dtype));
    if (channel_axis < -100) {
        CheckStatus(ppq_b200_linear_quant_t_toint_dt(v.data_ptr(), dt, out.data_ptr(), out_bits, v.numel(), F(s), F(o), clip_min, clip_max,
                                                     rounding, Stream()), "QuantizeTensor_toInt");
    } else {
        const Geometry g = ChannelGeometry(v, channel_axis);
        CheckChannelParams(s, o, g.C);
        CheckStatus(ppq_b200_linear_quant_c_toint_dt(v.data_ptr(), dt, out.data_ptr(), out_bits, v.numel(), g.epc, g.C, F(s), F(o), clip_min,
                                                     clip_max, rounding, Stream()), "QuantizeTensor_toInt");
    }
    return out;
}

// ---------------------------------------------------------------- float fake-quant (floating.h:3-12)
Tensor QuantizeTensor_FT(const Tensor &value, const Tensor &scale, const Tensor &offset, const int exponent, const int mantissa,
                         const float clip_min, const float clip_max, const int rounding) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = DenseFormat(value);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_float_quant_t(F(v), out.data_ptr<float>(), v.numel(), F(scale), F(offset), exponent, mantissa, clip_min,
                                       clip_max, rounding, Stream()), "QuantizeTensor_FT");
    return out;
}

Tensor QuantizeTensor_FC(const Tensor &value, const Tensor &scale, const Tensor &offset, const int exponent, const int mantissa,
                         const float clip_min, const float clip_max, const int channel_axis, const int rounding) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    auto s = scale.contiguous(), o = offset.contiguous();
    const Geometry g = ChannelGeometry(v, channel_axis);
    CheckChannelParams(s, o, g.C);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_float_quant_c(F(v), out.data_ptr<float>(), v.numel(), g.epc, g.C, F(s), F(o), exponent, mantissa, clip_min,
                                       clip_max, rounding, Stream()), "QuantizeTensor_FC");
    return out;
}

// ---------------------------------------------------------------- fp16 / bf16 siblings of the fake-quant names
// Same positional signatures; the value is fp16 or bf16 and so is the output (the fp32 result on the exact upcast, rounded once to nearest
// even).  Scale and offset stay fp32.  The reference names above keep their fp32-only checks.
Tensor QuantizeTensor_LT_Half(const Tensor &value, const Tensor &scale, const Tensor &offset, const int clip_min, const int clip_max,
                              const int rounding) {
    const int dt = CheckValue(value, true);
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = DenseFormat(value);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_linear_quant_t_dt(v.data_ptr(), dt, out.data_ptr(), v.numel(), F(scale), F(offset), clip_min, clip_max, rounding,
                                           Stream()), "QuantizeTensor_LT_Half");
    return out;
}

Tensor QuantizeTensor_LC_Half(const Tensor &value, const Tensor &scale, const Tensor &offset, const int clip_min, const int clip_max,
                              const int channel_axis, const int rounding) {
    const int dt = CheckValue(value, true);
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    auto s = scale.contiguous(), o = offset.contiguous();
    const Geometry g = ChannelGeometry(v, channel_axis);
    CheckChannelParams(s, o, g.C);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_linear_quant_c_dt(v.data_ptr(), dt, out.data_ptr(), v.numel(), g.epc, g.C, F(s), F(o), clip_min, clip_max, rounding,
                                           Stream()), "QuantizeTensor_LC_Half");
    return out;
}

Tensor QuantizeTensor_FT_Half(const Tensor &value, const Tensor &scale, const Tensor &offset, const int exponent, const int mantissa,
                              const float clip_min, const float clip_max, const int rounding) {
    const int dt = CheckValue(value, true);
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = DenseFormat(value);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_float_quant_t_dt(v.data_ptr(), dt, out.data_ptr(), v.numel(), F(scale), F(offset), exponent, mantissa, clip_min,
                                          clip_max, rounding, Stream()), "QuantizeTensor_FT_Half");
    return out;
}

Tensor QuantizeTensor_FC_Half(const Tensor &value, const Tensor &scale, const Tensor &offset, const int exponent, const int mantissa,
                              const float clip_min, const float clip_max, const int channel_axis, const int rounding) {
    const int dt = CheckValue(value, true);
    CheckTensor(scale, at::kFloat, "Scale(Expect to be FP32)");
    CheckTensor(offset, at::kFloat, "Offset(Expect to be FP32)");
    CheckSize(value);
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    auto s = scale.contiguous(), o = offset.contiguous();
    const Geometry g = ChannelGeometry(v, channel_axis);
    CheckChannelParams(s, o, g.C);
    Tensor out = at::empty_like(v);
    CheckStatus(ppq_b200_float_quant_c_dt(v.data_ptr(), dt, out.data_ptr(), v.numel(), g.epc, g.C, F(s), F(o), exponent, mantissa, clip_min,
                                          clip_max, rounding, Stream()), "QuantizeTensor_FC_Half");
    return out;
}

void Histogram_Asymmetric_T_Half(const float min, const float max, const Tensor &value, const bool clip_outliers, Tensor &hist) {
    const int dt = CheckValue(value, true);
    CheckTensor(hist, at::kInt, "Histogram(Expect to be INT32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = Dense(value);
    CheckStatus(ppq_b200_histogram_asym_t_dt(v.data_ptr(), dt, v.numel(), min, max, clip_outliers, hist.data_ptr<int>(), hist.numel(), Stream()),
                "Histogram_Asymmetric_T_Half");
}

// ---------------------------------------------------------------- histograms (sort.h:5-23)
void Histogram_T(const Tensor &value, const float hist_scale, const bool clip_outliers, Tensor &hist) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(hist, at::kInt, "Histogram(Expect to be INT32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = Dense(value);
    CheckStatus(ppq_b200_histogram_t(F(v), v.numel(), hist_scale, clip_outliers, hist.data_ptr<int>(), hist.numel(), Stream()),
                "Histogram_T");
}

void Histogram_Asymmetric_T(const float min, const float max, const Tensor &value, const bool clip_outliers, Tensor &hist) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(hist, at::kInt, "Histogram(Expect to be INT32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = Dense(value);
    CheckStatus(ppq_b200_histogram_asym_t(F(v), v.numel(), min, max, clip_outliers, hist.data_ptr<int>(), hist.numel(), Stream()),
                "Histogram_Asymmetric_T");
}

void Histogram_C(const Tensor &value, const int channel_axis, const float hist_scale, const bool clip_outliers, Tensor &hist) {
    CheckTensor(value, at::kFloat, "Value(Expect to be FP32)");
    CheckTensor(hist, at::kInt, "Histogram(Expect to be INT32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    const Geometry g = ChannelGeometry(v, channel_axis);
    if (hist.numel() % g.C != 0) throw KernelFailure("Kernel Failure, Histogram shape is invalid.");
    CheckStatus(ppq_b200_histogram_c(F(v), v.numel(), g.epc, g.C, hist_scale, clip_outliers, hist.data_ptr<int>(),
                                     hist.numel() / g.C, Stream()), "Histogram_C");
}

float compute_mse_loss(const std::vector<int64_t> &hist, const int start, const int step, const int end) {
    return ppq_b200_compute_mse_loss(hist.data(), (int64_t)hist.size(), start, step, end);
}

// ---------------------------------------------------------------- H100-native extras (not in the reference table)
void MinMax_Init(Tensor &mins, Tensor &maxs) {
    CheckTensor(mins, at::kFloat, "Min(Expect to be FP32)");
    CheckTensor(maxs, at::kFloat, "Max(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(mins.device());
    CheckStatus(ppq_b200_minmax_init(mins.data_ptr<float>(), maxs.data_ptr<float>(), mins.numel(), Stream()), "MinMax_Init");
}
// minmax: float[2] = {min, max}, accumulated
void MinMax_T(const Tensor &value, Tensor &minmax) {
    const int dt = CheckValue(value, false);
    CheckTensor(minmax, at::kFloat, "MinMax(Expect to be FP32)");
    if (minmax.numel() != 2) throw KernelFailure("Kernel Failure, MinMax buffer must hold 2 floats.");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = Dense(value);
    CheckStatus(ppq_b200_minmax_t_dt(v.data_ptr(), dt, v.numel(), minmax.data_ptr<float>(), Stream()), "MinMax_T");
}
void MinMax_C(const Tensor &value, const int channel_axis, Tensor &mins, Tensor &maxs) {
    const int dt = CheckValue(value, false);
    CheckTensor(mins, at::kFloat, "Min(Expect to be FP32)");
    CheckTensor(maxs, at::kFloat, "Max(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = value.contiguous();
    const Geometry g = ChannelGeometry(v, channel_axis);
    if (mins.numel() != g.C || maxs.numel() != g.C) throw KernelFailure("Kernel Failure, min / max must hold one value per channel.");
    CheckStatus(ppq_b200_minmax_c_dt(v.data_ptr(), dt, v.numel(), g.epc, g.C, mins.data_ptr<float>(), maxs.data_ptr<float>(), Stream()), "MinMax_C");
}
void Histogram_T_DeviceScale(const Tensor &value, const Tensor &hist_scale, const bool clip_outliers, Tensor &hist) {
    const int dt = CheckValue(value, false);
    CheckTensor(hist_scale, at::kFloat, "HistScale(Expect to be FP32)");
    CheckTensor(hist, at::kInt, "Histogram(Expect to be INT32)");
    const c10::cuda::CUDAGuard guard(value.device());
    auto v = Dense(value);
    CheckStatus(ppq_b200_histogram_t_dscale_dt(v.data_ptr(), dt, v.numel(), F(hist_scale), clip_outliers, hist.data_ptr<int>(), hist.numel(), Stream()),
                "Histogram_T_DeviceScale");
}
// descs: int64 tensor [count, 3] on the device = (data_ptr, numel, slot) -- bit-compatible with ppq_b200_tensor_desc
// (pointer, int64, {int32 slot, int32 pad}) on a little-endian machine.
void Multi_MinMax_T(const Tensor &descs, const int64_t max_numel, Tensor &minmax_arena) {
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    CheckTensor(minmax_arena, at::kFloat, "MinMaxArena(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_minmax_t(reinterpret_cast<const ppq_b200_tensor_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0),
                                        max_numel, minmax_arena.data_ptr<float>(), Stream()), "Multi_MinMax_T");
}
void Multi_Histogram_T(const Tensor &descs, const int64_t max_numel, const Tensor &hist_scale_arena, const bool clip_outliers,
                       Tensor &hist_arena, const int64_t bins) {
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    CheckTensor(hist_scale_arena, at::kFloat, "HistScaleArena(Expect to be FP32)");
    CheckTensor(hist_arena, at::kInt, "HistArena(Expect to be INT32)");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_histogram_t(reinterpret_cast<const ppq_b200_tensor_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0),
                                           max_numel, F(hist_scale_arena), clip_outliers, hist_arena.data_ptr<int>(), bins, Stream()),
                "Multi_Histogram_T");
}
// out: float tensor, tensor i writes out.flat[slot_i * out_stride + {0, 1}] = {upper, lower} quantile; workspace: uint8 scratch
// guess: optional int32 tensor [slots, Quantile_Guess_Words()] made by Quantile_Guess_Init -- consecutive calls on the same slots become one-pass
void Multi_Quantile_T(const Tensor &descs, const int64_t max_numel, const float q, Tensor &out, const int64_t out_stride, Tensor &workspace,
                      const int64_t cap, const c10::optional<Tensor> &guess) {
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    CheckTensor(out, at::kFloat, "Quantiles(Expect to be FP32)");
    if (descs.dim() != 2 || descs.size(1) != 3 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 3] int64.");
    const int count = (int)descs.size(0);
    if (workspace.scalar_type() != at::kByte || workspace.numel() < ppq_b200_multi_quantile_workspace_bytes(count, cap))
        throw KernelFailure("Kernel Failure, quantile workspace is too small (see Multi_Quantile_Workspace_Bytes).");
    const c10::cuda::CUDAGuard guard(descs.device());
    uint32_t *gp = nullptr;
    if (guess.has_value()) {
        CheckTensor(*guess, at::kInt, "Guess(Expect to be INT32)");
        if (!guess->is_contiguous() || guess->numel() % ppq_b200_quantile_guess_words() != 0) throw KernelFailure("Kernel Failure, quantile guess buffer has a wrong shape.");
        gp = reinterpret_cast<uint32_t *>(guess->data_ptr<int>());
    }
    CheckStatus(ppq_b200_multi_quantile_t(reinterpret_cast<const ppq_b200_tensor_desc *>(descs.data_ptr<int64_t>()), count, max_numel, q,
                                          out.data_ptr<float>(), out_stride, workspace.data_ptr(), cap, gp, Stream()), "Multi_Quantile_T");
}
// ---------------------------------------------------------------- fp16 / bf16 siblings of the table names
// The positional signatures of the fp32 names with the table's element type after max_numel: a raw pointer table cannot tell it.
int HalfTableType(const py::object &dtype) {
    const auto st = torch::python::detail::py_object_to_dtype(dtype);
    if (st == at::kHalf) return PPQ_B200_F16;
    if (st == at::kBFloat16) return PPQ_B200_BF16;
    throw KernelFailure("Kernel Failure, Invalid dtype of Input tensor: Value(Expect to be FP16 or BF16)");
}
void Multi_MinMax_T_Half(const Tensor &descs, const int64_t max_numel, const py::object &dtype, Tensor &minmax_arena) {
    const int dt = HalfTableType(dtype);
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    CheckTensor(minmax_arena, at::kFloat, "MinMaxArena(Expect to be FP32)");
    if (descs.dim() != 2 || descs.size(1) != 3 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 3] int64.");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_minmax_t_dt(reinterpret_cast<const ppq_b200_tensor_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0),
                                           max_numel, dt, minmax_arena.data_ptr<float>(), Stream()), "Multi_MinMax_T_Half");
}
void Multi_Histogram_T_Half(const Tensor &descs, const int64_t max_numel, const py::object &dtype, const Tensor &hist_scale_arena,
                            const bool clip_outliers, Tensor &hist_arena, const int64_t bins) {
    const int dt = HalfTableType(dtype);
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    CheckTensor(hist_scale_arena, at::kFloat, "HistScaleArena(Expect to be FP32)");
    CheckTensor(hist_arena, at::kInt, "HistArena(Expect to be INT32)");
    if (descs.dim() != 2 || descs.size(1) != 3 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 3] int64.");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_histogram_t_dt(reinterpret_cast<const ppq_b200_tensor_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0),
                                              max_numel, dt, F(hist_scale_arena), clip_outliers, hist_arena.data_ptr<int>(), bins, Stream()),
                "Multi_Histogram_T_Half");
}
void Multi_Quantile_T_Half(const Tensor &descs, const int64_t max_numel, const py::object &dtype, const float q, Tensor &out,
                           const int64_t out_stride, Tensor &workspace, const int64_t cap, const c10::optional<Tensor> &guess) {
    const int dt = HalfTableType(dtype);
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    CheckTensor(out, at::kFloat, "Quantiles(Expect to be FP32)");
    if (descs.dim() != 2 || descs.size(1) != 3 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 3] int64.");
    const int count = (int)descs.size(0);
    if (workspace.scalar_type() != at::kByte || workspace.numel() < ppq_b200_multi_quantile_workspace_bytes(count, cap))
        throw KernelFailure("Kernel Failure, quantile workspace is too small (see Multi_Quantile_Workspace_Bytes).");
    const c10::cuda::CUDAGuard guard(descs.device());
    uint32_t *gp = nullptr;
    if (guess.has_value()) {
        CheckTensor(*guess, at::kInt, "Guess(Expect to be INT32)");
        if (!guess->is_contiguous() || guess->numel() % ppq_b200_quantile_guess_words() != 0) throw KernelFailure("Kernel Failure, quantile guess buffer has a wrong shape.");
        gp = reinterpret_cast<uint32_t *>(guess->data_ptr<int>());
    }
    CheckStatus(ppq_b200_multi_quantile_t_dt(reinterpret_cast<const ppq_b200_tensor_desc *>(descs.data_ptr<int64_t>()), count, max_numel, dt, q,
                                             out.data_ptr<float>(), out_stride, workspace.data_ptr(), cap, gp, Stream()), "Multi_Quantile_T_Half");
}
// descs as for Multi_QuantizeTensor_LC; x and y of every row point at elements of `dtype`
void Multi_QuantizeTensor_LC_Half(const Tensor &descs, const int64_t max_numel, const py::object &dtype, const int clip_min, const int clip_max,
                                  const int rounding) {
    const int dt = HalfTableType(dtype);
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    if (descs.dim() != 2 || descs.size(1) != 7 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 7] int64.");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_linear_quant_c_dt(reinterpret_cast<const ppq_b200_lc_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0), max_numel,
                                                 dt, clip_min, clip_max, rounding, Stream()), "Multi_QuantizeTensor_LC_Half");
}
Tensor Quantile_Guess_Init(const int64_t slots, const Tensor &like) {
    const c10::cuda::CUDAGuard guard(like.device());
    Tensor g = at::empty({slots, ppq_b200_quantile_guess_words()}, like.options().dtype(at::kInt));
    CheckStatus(ppq_b200_quantile_guess_init(reinterpret_cast<uint32_t *>(g.data_ptr<int>()), slots, Stream()), "Quantile_Guess_Init");
    return g;
}
int64_t Multi_Quantile_Workspace_Bytes(const int count, const int64_t cap) { return ppq_b200_multi_quantile_workspace_bytes(count, cap); }
std::vector<Tensor> MinMax_To_Scale_Offset(const Tensor &mins, const Tensor &maxs, const int64_t stride, const int quant_min,
                                           const int quant_max, const bool symmetrical, const bool power_of_2, const double min_scale) {
    CheckTensor(mins, at::kFloat, "Min(Expect to be FP32)");
    CheckTensor(maxs, at::kFloat, "Max(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(mins.device());
    const int64_t count = (mins.numel() + stride - 1) / stride;
    Tensor scale = at::empty({count}, mins.options()), offset = at::empty({count}, mins.options());
    CheckStatus(ppq_b200_minmax_to_scale_offset(F(mins), F(maxs), count, stride, quant_min, quant_max, symmetrical, power_of_2, min_scale,
                                                scale.data_ptr<float>(), offset.data_ptr<float>(), Stream()), "MinMax_To_Scale_Offset");
    return {scale, offset};
}
Tensor Hist_Scale_From_MinMax(const Tensor &minmax_arena, const bool symmetrical, const int64_t bins) {
    CheckTensor(minmax_arena, at::kFloat, "MinMaxArena(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(minmax_arena.device());
    const int64_t count = minmax_arena.numel() / 2;
    Tensor hs = at::empty({count}, minmax_arena.options());
    CheckStatus(ppq_b200_hist_scale_from_minmax(F(minmax_arena), count, symmetrical, bins, hs.data_ptr<float>(), Stream()),
                "Hist_Scale_From_MinMax");
    return hs;
}
std::vector<Tensor> KL_Search(const Tensor &hist_arena, const int64_t bins, const Tensor &hist_scale_arena,
                              const c10::optional<Tensor> &minmax_arena, const int num_of_bits,
                              const bool power_of_2, const double min_scale) {
    CheckTensor(hist_arena, at::kInt, "HistArena(Expect to be INT32)");
    CheckTensor(hist_scale_arena, at::kFloat, "HistScaleArena(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(hist_arena.device());
    const int64_t count = hist_arena.numel() / bins;
    Tensor scale = at::empty({count}, hist_scale_arena.options());
    Tensor best = at::empty({count}, hist_arena.options());
    const float *mm = nullptr;
    if (minmax_arena.has_value()) { CheckTensor(*minmax_arena, at::kFloat, "MinMaxArena(Expect to be FP32)"); mm = F(*minmax_arena); }
    CheckStatus(ppq_b200_kl_search(hist_arena.data_ptr<int>(), count, bins, F(hist_scale_arena), mm, num_of_bits, power_of_2, min_scale,
                                   scale.data_ptr<float>(), best.data_ptr<int>(), Stream()), "KL_Search");
    return {scale, best};
}
// descs: int64 tensor [count, 7] on the device = (x, y, scale, offset, numel, epc, C) -- bit-compatible with ppq_b200_lc_desc
void Multi_QuantizeTensor_LC(const Tensor &descs, const int64_t max_numel, const int clip_min, const int clip_max, const int rounding) {
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    if (descs.dim() != 2 || descs.size(1) != 7 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 7] int64.");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_linear_quant_c(reinterpret_cast<const ppq_b200_lc_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0), max_numel,
                                              clip_min, clip_max, rounding, Stream()), "Multi_QuantizeTensor_LC");
}
// descs: int64 tensor [count, 5] on the device = (x, y, scale, offset, numel) -- bit-compatible with ppq_b200_lt_desc
void Multi_QuantizeTensor_LT(const Tensor &descs, const int64_t max_numel, const int clip_min, const int clip_max, const int rounding) {
    CheckTensor(descs, at::kLong, "Descriptors(Expect to be INT64)");
    if (descs.dim() != 2 || descs.size(1) != 5 || !descs.is_contiguous()) throw KernelFailure("Kernel Failure, descriptor table must be [count, 5] int64.");
    const c10::cuda::CUDAGuard guard(descs.device());
    CheckStatus(ppq_b200_multi_linear_quant_t(reinterpret_cast<const ppq_b200_lt_desc *>(descs.data_ptr<int64_t>()), (int)descs.size(0), max_numel,
                                              clip_min, clip_max, rounding, Stream()), "Multi_QuantizeTensor_LT");
}
std::vector<Tensor> MSE_Search(const Tensor &hist_arena, const int64_t bins, const Tensor &minmax_arena, const int quant_min, const int quant_max,
                               const bool symmetrical, const bool power_of_2, const double min_scale, const int interval) {
    CheckTensor(hist_arena, at::kInt, "HistArena(Expect to be INT32)");
    CheckTensor(minmax_arena, at::kFloat, "MinMaxArena(Expect to be FP32)");
    const c10::cuda::CUDAGuard guard(hist_arena.device());
    const int64_t count = hist_arena.numel() / bins;
    Tensor scale = at::empty({count}, minmax_arena.options()), offset = at::empty({count}, minmax_arena.options());
    CheckStatus(ppq_b200_mse_search(hist_arena.data_ptr<int>(), count, bins, F(minmax_arena), quant_min, quant_max, symmetrical, power_of_2,
                                    min_scale, interval, scale.data_ptr<float>(), offset.data_ptr<float>(), Stream()), "MSE_Search");
    return {scale, offset};
}
int set_variant(const std::string &kernel, int variant) { return ppq_b200_set_variant(kernel.c_str(), variant); }
int get_variant(const std::string &kernel) { return ppq_b200_get_variant(kernel.c_str()); }

}  // namespace

#include "torch_binding_more.inc"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.doc() = "ppq_b200: H100-native drop-in for PPQ_Cuda_Impls";
    // the reference table, ppq/csrc/export.cc:9-33
    m.def("Histogram_T", Histogram_T, "Histogram_T");
    m.def("Histogram_Asymmetric_T", Histogram_Asymmetric_T, "Histogram_Asymmetric_T");
    m.def("Histogram_C", Histogram_C, "Histogram_C");
    m.def("QuantizeTensor_LT", QuantizeTensor_LT, "QuantizeTensor_LT");
    m.def("QuantizeTensor_LC", QuantizeTensor_LC, "QuantizeTensor_LC");
    m.def("QuantizeTensor_FT", QuantizeTensor_FT, "QuantizeTensor_FT");
    m.def("QuantizeTensor_FC", QuantizeTensor_FC, "QuantizeTensor_FC");
    m.def("compute_mse_loss", compute_mse_loss, "compute_mse_loss");
    register_more(m);
    // H100-native extras
    m.def("QuantizeTensor_toInt", QuantizeTensor_toInt, "QuantizeTensor_toInt");
    m.def("QuantizeTensor_LT_Half", QuantizeTensor_LT_Half, "QuantizeTensor_LT_Half");
    m.def("QuantizeTensor_LC_Half", QuantizeTensor_LC_Half, "QuantizeTensor_LC_Half");
    m.def("QuantizeTensor_FT_Half", QuantizeTensor_FT_Half, "QuantizeTensor_FT_Half");
    m.def("QuantizeTensor_FC_Half", QuantizeTensor_FC_Half, "QuantizeTensor_FC_Half");
    m.def("Histogram_Asymmetric_T_Half", Histogram_Asymmetric_T_Half, "Histogram_Asymmetric_T_Half");
    m.def("Multi_QuantizeTensor_LC", Multi_QuantizeTensor_LC, "Multi_QuantizeTensor_LC");
    m.def("Multi_QuantizeTensor_LT", Multi_QuantizeTensor_LT, "Multi_QuantizeTensor_LT");
    m.def("MinMax_Init", MinMax_Init, "MinMax_Init");
    m.def("MinMax_T", MinMax_T, "MinMax_T");
    m.def("MinMax_C", MinMax_C, "MinMax_C");
    m.def("Histogram_T_DeviceScale", Histogram_T_DeviceScale, "Histogram_T_DeviceScale");
    m.def("Multi_MinMax_T", Multi_MinMax_T, "Multi_MinMax_T");
    m.def("Multi_Histogram_T", Multi_Histogram_T, "Multi_Histogram_T");
    m.def("Multi_Quantile_T", Multi_Quantile_T, "Multi_Quantile_T");
    m.def("Multi_MinMax_T_Half", Multi_MinMax_T_Half, "Multi_MinMax_T_Half");
    m.def("Multi_Histogram_T_Half", Multi_Histogram_T_Half, "Multi_Histogram_T_Half");
    m.def("Multi_Quantile_T_Half", Multi_Quantile_T_Half, "Multi_Quantile_T_Half");
    m.def("Multi_QuantizeTensor_LC_Half", Multi_QuantizeTensor_LC_Half, "Multi_QuantizeTensor_LC_Half");
    m.def("Quantile_Guess_Init", Quantile_Guess_Init, "Quantile_Guess_Init");
    m.def("Multi_Quantile_Workspace_Bytes", Multi_Quantile_Workspace_Bytes, "Multi_Quantile_Workspace_Bytes");
    m.def("MinMax_To_Scale_Offset", MinMax_To_Scale_Offset, "MinMax_To_Scale_Offset");
    m.def("Hist_Scale_From_MinMax", Hist_Scale_From_MinMax, "Hist_Scale_From_MinMax");
    m.def("KL_Search", KL_Search, "KL_Search");
    m.def("MSE_Search", MSE_Search, "MSE_Search");
    m.def("set_variant", set_variant, "set_variant");
    m.def("get_variant", get_variant, "get_variant");
    m.def("abi_version", ppq_b200_abi_version, "abi_version");
    m.def("build_info", []() { return std::string(ppq_b200_build_info()); }, "build_info");
}
