"""ppq_b200 -- H100-native (sm_90a) implementation of the PPQ quantization-simulation hot path.

    csrc/        hand-written CUDA kernels + C ABI (include/ppq_b200.h) + torch binding with the reference's 20 names
    ffi          mirror of ppq.core.ffi  (CUDA_COMPLIER, class CUDA)
    core         TensorQuantizationConfig / policies / states / constants consumed by the path
    qfunction    PPQuantFunction & friends (CUDA branch only -- there is no CPU fallback in this package)
    observer     min-max / KL / MSE / percentile / FP8 observers over a device-resident statistics arena
    calibration  sample-sharded RuntimeCalibrationPass with one all-reduce per phase
    install      plug into the real `ppq` package without touching its sources

Importing this package does not load the native extension; the first use of ffi.CUDA / extension() does, and raises
ImportError if it has not been built (python -m ppq_b200.build).
"""
from .core import (FloatingQuantizationConfig, LinearQuantizationConfig, QuantizationPolicy, QuantizationProperty,
                   QuantizationStates, RoundingPolicy, TensorQuantizationConfig)

__version__ = '0.1.0'


def extension():
    from .ffi import extension as _e
    return _e()
