"""Foreign-function layer: the mirror of ppq/core/ffi.py (/root/reference/ppq/core/ffi.py:16-350).

`CUDA_COMPLIER.CUDA_EXTENSION` is the in-tree torch extension ppq_b200/_C.so (built by `python -m ppq_b200.build`, never JIT)
and `class CUDA` has the reference's static methods with the reference's argument orders -- including the re-orderings the
reference does between Python and C++ (LinearQuantize_C, Histogram_T ...; SURVEY.md §8b "argument-order traps").

There is no CPU fallback anywhere in this package: if the extension is missing or the tensors are not on a CUDA device the
call fails loudly.
"""
import importlib.util
import os
from typing import List

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_EXT_PATH = os.path.join(_HERE, '_C.so')


class ComplieHelper:
    """Same surface as ppq.core.ffi.ComplieHelper (ffi.py:16-49) -- `complie()` loads the prebuilt in-tree extension."""

    def __init__(self) -> None:
        self.__CUDA_EXTENTION__ = None

    def complie(self):
        if self.__CUDA_EXTENTION__ is not None:
            return self.__CUDA_EXTENTION__
        if not os.path.exists(_EXT_PATH):
            raise ImportError(
                f'ppq_b200 native extension not found at {_EXT_PATH}. Build it in-tree first: `python -m ppq_b200.build` '
                '(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback.')
        spec = importlib.util.spec_from_file_location('ppq_b200._C', _EXT_PATH)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        self.__CUDA_EXTENTION__ = mod
        return mod

    @property
    def CUDA_EXTENSION(self):
        if self.__CUDA_EXTENTION__ is None:
            self.complie()
        return self.__CUDA_EXTENTION__


CUDA_COMPLIER = ComplieHelper()


def extension():
    """The module object to assign into the real PPQ: ppq.core.ffi.CUDA_COMPLIER.__CUDA_EXTENTION__ = extension()."""
    return CUDA_COMPLIER.CUDA_EXTENSION


def _dense(t: torch.Tensor) -> torch.Tensor:
    """The reference wrappers make their operands contiguous before the call (ffi.py:199-306); same here."""
    return t if t.is_contiguous() else t.contiguous()


def _ext():
    return CUDA_COMPLIER.CUDA_EXTENSION


class CUDA:
    """Static wrappers with the reference's names and argument orders (ffi.py:56-350).  The only logic in them is what the reference's
    wrappers do themselves: argument re-ordering between Python and C++, `contiguous()`, and the exponent check of the float formats."""

    @staticmethod
    def LinearQuantize_T(tensor: torch.Tensor, scales: torch.Tensor, offsets: torch.Tensor, minimum: int = -128,
                         maximum: int = 127, rounding: int = 0) -> torch.Tensor:
        return _ext().QuantizeTensor_LT(tensor, scales, offsets, minimum, maximum, rounding)

    @staticmethod
    def LinearQuantize_C(tensor: torch.Tensor, scales: torch.Tensor, offsets: torch.Tensor, channel_axis: int,
                         minimum: int = -128, maximum: int = 127, rounding: int = 0) -> torch.Tensor:
        return _ext().QuantizeTensor_LC(tensor, scales, offsets, minimum, maximum, channel_axis, rounding)

    @staticmethod
    def LinearQuantize_T_B(tensor, scales, offsets, dy, minimum: int, maximum: int, rounding: int) -> List[torch.Tensor]:
        return _ext().QuantizeTensor_LT_B(tensor, scales, offsets, dy, minimum, maximum, rounding)

    @staticmethod
    def LinearQuantize_C_B(tensor, scales, offsets, dy, minimum: int, maximum: int, channel_axis: int,
                           rounding: int) -> List[torch.Tensor]:
        return _ext().QuantizeTensor_LC_B(tensor, scales, offsets, dy, minimum, maximum, rounding, channel_axis)

    @staticmethod
    def Histogram_T(tensor: torch.Tensor, histogram: torch.Tensor, scale: float, clip_outliers: bool = True) -> torch.Tensor:
        _ext().Histogram_T(tensor, scale, clip_outliers, histogram)
        return histogram

    @staticmethod
    def Histogram_Asymmetric_T(min_value: float, max_value: float, tensor: torch.Tensor, histogram: torch.Tensor,
                               clip_outliers: bool = True) -> torch.Tensor:
        _ext().Histogram_Asymmetric_T(min_value, max_value, tensor, clip_outliers, histogram)
        return histogram

    @staticmethod
    def Histogram_C(tensor: torch.Tensor, channel_axis: int, histogram: torch.Tensor, scale: float,
                    clip_outliers: bool = True) -> torch.Tensor:
        _ext().Histogram_C(tensor, channel_axis, scale, clip_outliers, histogram)
        return histogram

    @staticmethod
    def Quantile(tensor: torch.Tensor, q: float) -> torch.Tensor:
        return _ext().Quantile_T(tensor, q)

    @staticmethod
    def TensorClip_T(tensor: torch.Tensor, reference: torch.Tensor, limit: torch.Tensor) -> torch.Tensor:
        tensor = _dense(tensor)
        reference = _dense(reference)
        return _ext().TensorClip_T(tensor, reference, limit)

    @staticmethod
    def TensorClip_C(tensor: torch.Tensor, reference: torch.Tensor, limit: torch.Tensor, channel_axis: int) -> torch.Tensor:
        tensor = _dense(tensor)
        reference = _dense(reference)
        return _ext().TensorClip_C(tensor, reference, limit, channel_axis)

    @staticmethod
    def RoundingLoss_LT(tensor, scales, offsets, minimum: int = -128, maximum: int = 127, rounding: int = 0) -> torch.Tensor:
        tensor = _dense(tensor)
        return _ext().RoundingLoss_LT(tensor, scales, offsets, minimum, maximum, rounding)

    @staticmethod
    def RoundingLoss_LT_B(tensor, dy, scales, offsets, minimum: int = -128, maximum: int = 127, rounding: int = 0) -> torch.Tensor:
        tensor = _dense(tensor)
        return _ext().RoundingLoss_LT_B(tensor, dy, scales, offsets, minimum, maximum, rounding)

    @staticmethod
    def RoundingLoss_LC(tensor, scales, offsets, channel_axis: int, minimum: int = -128, maximum: int = 127,
                        rounding: int = 0) -> torch.Tensor:
        tensor = _dense(tensor)
        return _ext().RoundingLoss_LC(tensor, scales, offsets, minimum, maximum, channel_axis, rounding)

    @staticmethod
    def RoundingLoss_LC_B(tensor, dy, scales, offsets, channel_axis: int, minimum: int = -128, maximum: int = 127,
                          rounding: int = 0) -> torch.Tensor:
        tensor = _dense(tensor)
        return _ext().RoundingLoss_LC_B(tensor, dy, scales, offsets, minimum, maximum, channel_axis, rounding)

    @staticmethod
    def compute_mse_loss(histogram: list, start: int, step: int, end: int) -> float:
        return _ext().compute_mse_loss(histogram, start, step, end)

    @staticmethod
    def FloatingQuantize_T(tensor, scales, offsets, exponent: int = 4, mantissa: int = 3, minimum: float = -448,
                           maximum: float = +448, rounding: int = 0) -> torch.Tensor:
        if exponent <= 0: raise ValueError('Floating Quantization requires exponent > 0')
        tensor = _dense(tensor)
        return _ext().QuantizeTensor_FT(tensor, scales, offsets, exponent, mantissa, minimum, maximum, rounding)

    @staticmethod
    def FloatingQuantize_C(tensor, scales, offsets, channel_axis: int, exponent: int = 4, mantissa: int = 3,
                           minimum: float = -448, maximum: float = +448, rounding: int = 0) -> torch.Tensor:
        if exponent <= 0: raise ValueError('Floating Quantization requires exponent > 0')
        tensor = _dense(tensor)
        return _ext().QuantizeTensor_FC(tensor, scales, offsets, exponent, mantissa, minimum, maximum, channel_axis, rounding)

    @staticmethod
    def FloatingQuantize_T_B(tensor, scales, offsets, dy, exponent: int, mantissa: int, minimum: float, maximum: float,
                             rounding: int) -> List[torch.Tensor]:
        tensor = _dense(tensor)
        return _ext().QuantizeTensor_FT_B(tensor, scales, offsets, dy, exponent, mantissa, minimum, maximum, rounding)

    @staticmethod
    def FloatingQuantize_C_B(tensor, scales, offsets, dy, exponent: int, mantissa: int, minimum: float, maximum: float,
                             channel_axis: int, rounding: int) -> List[torch.Tensor]:
        tensor = _dense(tensor)
        return _ext().QuantizeTensor_FC_B(tensor, scales, offsets, dy, exponent, mantissa, minimum, maximum, rounding, channel_axis)

    @staticmethod
    def Sync():
        torch.cuda.synchronize()

    # ---- H100-native additions (no counterpart in the reference table) -------------------------------------------
    @staticmethod
    def LinearQuantize_toInt(tensor, scales, offsets, channel_axis=None, minimum: int = -128, maximum: int = 127,
                             rounding: int = 0, out_bits: int = 8) -> torch.Tensor:
        axis = -1000 if channel_axis is None else channel_axis
        return _ext().QuantizeTensor_toInt(tensor, scales, offsets, minimum, maximum, axis, rounding, out_bits)

    @staticmethod
    def MinMax_T(tensor: torch.Tensor, minmax: torch.Tensor) -> torch.Tensor:
        _ext().MinMax_T(tensor, minmax)
        return minmax

    @staticmethod
    def MinMax_C(tensor: torch.Tensor, channel_axis: int, mins: torch.Tensor, maxs: torch.Tensor):
        _ext().MinMax_C(tensor, channel_axis, mins, maxs)
        return mins, maxs
