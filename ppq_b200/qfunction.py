"""Quantization functions: the mirror of ppq/quantization/qfunction (/root/reference/ppq/quantization/qfunction/
__init__.py:10-61, linear.py:8-238, floating.py:7-120), CUDA branch only.

Same names, same state / policy checks, same straight-through backward; the forward of every autograd Function calls the
sm_90a kernels through ppq_b200.ffi.CUDA.  There is deliberately no torch fallback: CPU tensors raise.
"""
import torch
from torch.autograd import Function

from .core import QuantizationProperty, QuantizationStates, RoundingPolicy, TensorQuantizationConfig
from .ffi import CUDA, CUDA_COMPLIER


def _rounding_value(rounding) -> int:
    return rounding.value if hasattr(rounding, 'value') else int(rounding)


def _require_cuda(tensor: torch.Tensor):
    if not tensor.is_cuda:
        raise PermissionError('ppq_b200 quantization functions require CUDA tensors (no CPU fallback exists in this package).')


class TensorwiseLinearQuantImpl(Function):
    """linear.py:8-50 (CUDA branch :34-46)."""
    @staticmethod
    def forward(ctx, tensor, scales, offsets, quant_min: int, quant_max: int, rounding) -> torch.Tensor:
        _require_cuda(tensor)
        scales, offsets = scales.to(tensor.device), offsets.to(tensor.device)
        return CUDA.LinearQuantize_T(tensor=tensor, scales=scales, offsets=offsets, minimum=quant_min, maximum=quant_max,
                                     rounding=_rounding_value(rounding))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        return dy, None, None, None, None, None


class ChannelwiseLinearQuantImpl(Function):
    """linear.py:53-96 (CUDA branch :82-92)."""
    @staticmethod
    def forward(ctx, tensor, scales, offsets, channel_axis: int, quant_min: int, quant_max: int, rounding) -> torch.Tensor:
        _require_cuda(tensor)
        scales, offsets = scales.to(tensor.device), offsets.to(tensor.device)
        return CUDA.LinearQuantize_C(tensor=tensor, scales=scales, offsets=offsets, channel_axis=channel_axis,
                                     minimum=quant_min, maximum=quant_max, rounding=_rounding_value(rounding))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        return dy, None, None, None, None, None, None


class TensorwiseFloatingQuantImpl(Function):
    """floating.py:7-50."""
    @staticmethod
    def forward(ctx, tensor, scales, offsets, exponet_bits: int, mantissa_bits: int, quant_min: float, quant_max: float,
                rounding) -> torch.Tensor:
        _require_cuda(tensor)
        scales, offsets = scales.to(tensor.device), offsets.to(tensor.device)
        return CUDA.FloatingQuantize_T(tensor=tensor, scales=scales, offsets=offsets, exponent=exponet_bits,
                                       mantissa=mantissa_bits, minimum=quant_min, maximum=quant_max,
                                       rounding=_rounding_value(rounding))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        return dy, None, None, None, None, None, None, None


class ChannelwiseFloatingQuantImpl(Function):
    """floating.py:53-92."""
    @staticmethod
    def forward(ctx, tensor, scales, offsets, channel_axis: int, exponet_bits: int, mantissa_bits: int, quant_min: float,
                quant_max: float, rounding) -> torch.Tensor:
        _require_cuda(tensor)
        scales, offsets = scales.to(tensor.device), offsets.to(tensor.device)
        return CUDA.FloatingQuantize_C(tensor=tensor, scales=scales, offsets=offsets, channel_axis=channel_axis,
                                       exponent=exponet_bits, mantissa=mantissa_bits, minimum=quant_min, maximum=quant_max,
                                       rounding=_rounding_value(rounding))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        return dy, None, None, None, None, None, None, None, None


def PPQLinearQuantFunction(tensor: torch.Tensor, config: TensorQuantizationConfig) -> torch.Tensor:
    """linear.py:200-216."""
    if not QuantizationStates.is_activated(config.state): return tensor
    if not config.policy.has_property(QuantizationProperty.LINEAR):
        raise ValueError('Critical Quantization Error! Non-linear config detected.')
    if config.policy.has_property(QuantizationProperty.DYNAMIC):
        raise ValueError('Unexpected Dynamic Flag in Quantization Policy. Use PPQDyamicQuantFunction Instead.')
    if config.policy.has_property(QuantizationProperty.PER_CHANNEL):
        return ChannelwiseLinearQuantImpl.apply(tensor, config.scale, config.offset, config.channel_axis,
                                                config.quant_min, config.quant_max, config.rounding)
    elif config.policy.has_property(QuantizationProperty.PER_TENSOR):
        return TensorwiseLinearQuantImpl.apply(tensor, config.scale, config.offset, config.quant_min, config.quant_max,
                                               config.rounding)


def PPQDyamicLinearQuantFunction(tensor: torch.Tensor, config: TensorQuantizationConfig) -> torch.Tensor:
    """linear.py:99-198: min/max -> scale/offset -> quantize, here as three device launches with no host round trip
    (the reference calls .item() / .tolist() and loops over channels in Python)."""
    if not QuantizationStates.is_activated(config.state): return tensor
    if not config.policy.has_property(QuantizationProperty.LINEAR):
        raise ValueError('Critical Quantization Error! Non-linear config detected.')
    if not config.policy.has_property(QuantizationProperty.DYNAMIC):
        raise ValueError('Quantization Policy Do Not Have Dynamic Flag!')
    _require_cuda(tensor)
    ext = CUDA_COMPLIER.CUDA_EXTENSION
    sym = config.policy.has_property(QuantizationProperty.SYMMETRICAL)
    pow2 = config.policy.has_property(QuantizationProperty.POWER_OF_2)
    from .core import OBSERVER_MIN_SCALE, OBSERVER_MIN_SCALE_MANUL_OVERRIDE
    min_scale = config.detail.get(OBSERVER_MIN_SCALE_MANUL_OVERRIDE, OBSERVER_MIN_SCALE)
    rounding = _rounding_value(config.rounding)
    if config.policy.has_property(QuantizationProperty.PER_CHANNEL):
        C = tensor.shape[config.channel_axis]
        mins = torch.empty(C, dtype=torch.float32, device=tensor.device); maxs = torch.empty_like(mins)
        ext.MinMax_Init(mins, maxs)
        ext.MinMax_C(tensor, config.channel_axis, mins, maxs)
        scales, offsets = ext.MinMax_To_Scale_Offset(mins, maxs, 1, config.quant_min, config.quant_max, sym, pow2, min_scale)
        return CUDA.LinearQuantize_C(tensor, scales, offsets, config.channel_axis, config.quant_min, config.quant_max, rounding)
    mm = torch.empty(2, dtype=torch.float32, device=tensor.device)
    ext.MinMax_Init(mm[0:1], mm[1:2])
    ext.MinMax_T(tensor, mm)
    scales, offsets = ext.MinMax_To_Scale_Offset(mm[0:1], mm[1:2], 1, config.quant_min, config.quant_max, sym, pow2, min_scale)
    return CUDA.LinearQuantize_T(tensor, scales, offsets, config.quant_min, config.quant_max, rounding)


def PPQFloatingQuantFunction(tensor: torch.Tensor, config: TensorQuantizationConfig) -> torch.Tensor:
    """floating.py:95-120."""
    if not tensor.is_cuda:
        raise PermissionError('PPQ Floating Quant Function requires tensor device to be cuda, '
                              'CPU floating quantization is not implemented yet.')
    if not QuantizationStates.is_activated(config.state): return tensor
    if not config.policy.has_property(QuantizationProperty.FLOATING):
        raise ValueError('Critical Quantization Error! Unexpected policy detected. '
                         'PPQFloatingQuantFunction except a Floating Quantization Config.')
    if config.policy.has_property(QuantizationProperty.DYNAMIC):
        raise ValueError('Unexpected Dynamic Flag in Quantization Policy.')
    if config.policy.has_property(QuantizationProperty.PER_CHANNEL):
        return ChannelwiseFloatingQuantImpl.apply(tensor, config.scale, config.offset, config.channel_axis,
                                                  config.exponent_bits, config.mantissa_bits, config.quant_min,
                                                  config.quant_max, config.rounding)
    elif config.policy.has_property(QuantizationProperty.PER_TENSOR):
        return TensorwiseFloatingQuantImpl.apply(tensor, config.scale, config.offset, config.exponent_bits,
                                                 config.mantissa_bits, config.quant_min, config.quant_max, config.rounding)


def PPQuantFunction(tensor: torch.Tensor, config: TensorQuantizationConfig) -> torch.Tensor:
    """qfunction/__init__.py:10-44."""
    if tensor is None: raise ValueError('Tensor is empty.')
    if config.policy.has_property(QuantizationProperty.LINEAR):
        if not config.policy.has_property(QuantizationProperty.DYNAMIC):
            return PPQLinearQuantFunction(tensor, config)
        return PPQDyamicLinearQuantFunction(tensor, config)
    if config.policy.has_property(QuantizationProperty.FLOATING):
        return PPQFloatingQuantFunction(tensor, config)
    raise ValueError('Unexpected Quantization Property Found in PPQuantFunction. '
                     'Do not konw how to quantize your config yet.')


def PPQLinearQuant_toInt(tensor: torch.Tensor, config: TensorQuantizationConfig) -> torch.Tensor:
    """linear.py:218-238, on the device: quantise without dequantising -> int8 / uint8 / int32 tensor."""
    if not config.policy.has_property(QuantizationProperty.LINEAR):
        raise ValueError('Critical Quantization Error! Non-linear config detected.')
    _require_cuda(tensor)
    if config.num_of_bits == 8: bits = 8
    elif config.num_of_bits > 8: bits = 32
    else: raise Exception('Do not konw how to convert value into int. num of bits is unexpected.')
    axis = config.channel_axis if config.policy.has_property(QuantizationProperty.PER_CHANNEL) else None
    out = CUDA.LinearQuantize_toInt(tensor, config.scale.to(tensor.device), config.offset.to(tensor.device), axis,
                                    config.quant_min, config.quant_max, _rounding_value(config.rounding), bits)
    if bits == 8:
        # the reference picks the dtype from the policy, not from the clip range (linear.py:231-235)
        want = torch.int8 if config.policy.has_property(QuantizationProperty.SYMMETRICAL) else torch.uint8
        if out.dtype != want: out = out.view(want)
    return out


def PPQuantFunction_toInt(tensor: torch.Tensor, config: TensorQuantizationConfig) -> torch.Tensor:
    """qfunction/__init__.py:47-61."""
    if config.policy.has_property(QuantizationProperty.LINEAR):
        if not config.policy.has_property(QuantizationProperty.DYNAMIC):
            return PPQLinearQuant_toInt(tensor, config)
    raise ValueError('Unexpected Quantization Property Found in PPQuantFunction_toInt. '
                     'Do not konw how to quantize your config yet.')


class CuLSQ_LT(Function):
    """ppq/quantization/algorithm/training.py:17-52: learned-step-size quantisation, per tensor.  Forward = the fake-quant kernel,
    backward = QuantizeTensor_LT_B (grad_x with the clip mask, grad_scale reduced on the device)."""
    @staticmethod
    def forward(ctx, tensor, scales, offsets, quant_min: int, quant_max: int, rounding) -> torch.Tensor:
        _require_cuda(tensor)
        r = _rounding_value(rounding)
        quantized = CUDA.LinearQuantize_T(tensor=tensor, scales=scales, offsets=offsets, minimum=quant_min, maximum=quant_max, rounding=r)
        ctx.save_for_backward(tensor, scales, offsets)
        ctx._quant_params = [quant_min, quant_max, r]
        return quantized

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        tensor, scales, offsets = ctx.saved_tensors
        quant_min, quant_max, rounding = ctx._quant_params
        dx, ds = CUDA.LinearQuantize_T_B(tensor, scales, offsets, dy.contiguous(), quant_min, quant_max, rounding)
        return dx, ds, None, None, None, None


class CuLSQ_LC(Function):
    """training.py:55-90: per-channel variant (QuantizeTensor_LC_B)."""
    @staticmethod
    def forward(ctx, tensor, scales, offsets, channel_axis: int, quant_min: int, quant_max: int, rounding) -> torch.Tensor:
        _require_cuda(tensor)
        r = _rounding_value(rounding)
        quantized = CUDA.LinearQuantize_C(tensor=tensor, scales=scales, offsets=offsets, channel_axis=channel_axis,
                                          minimum=quant_min, maximum=quant_max, rounding=r)
        ctx.save_for_backward(tensor, scales, offsets)
        ctx._quant_params = [quant_min, quant_max, channel_axis, r]
        return quantized

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        tensor, scales, offsets = ctx.saved_tensors
        quant_min, quant_max, channel_axis, rounding = ctx._quant_params
        dx, ds = CUDA.LinearQuantize_C_B(tensor, scales, offsets, dy.contiguous(), quant_min, quant_max, channel_axis, rounding)
        return dx, ds, None, None, None, None, None
