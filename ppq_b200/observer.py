"""Calibration observers: the mirror of ppq/quantization/observer (/root/reference/ppq/quantization/observer/
__init__.py:15-124, range.py:22-520, floating.py:11-144) on top of the sm_90a collectors.

What changed versus the reference (results are the same, the data flow is H100-first):
  * observe() never appends to Python lists: every observer owns a slice of a device-resident *statistics arena*
    ({min, max} floats, int32 histogram bins) that the kernels accumulate into with atomics;
  * min and max are one fused pass (MinMax_T / MinMax_C), not value.min() + value.max();
  * render() computes scale/offset on the device (MinMax_To_Scale_Offset, KL_Search): no .item() per tensor, no Python
    loop per channel; the arena is what the multi-GPU calibration all-reduces (ppq_b200/calibration.py).
Class and table names follow the reference so that `OBSERVER_TABLE[...]` replacement in the real PPQ is one assignment
(INTEGRATION.md).
"""
from typing import Dict, List, Optional

import torch

from .core import (OBSERVER_FLOATING_MSE_FETCHES, OBSERVER_KL_HIST_BINS, OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE,
                   OBSERVER_MIN_SCALE, OBSERVER_MIN_SCALE_MANUL_OVERRIDE, OBSERVER_MSE_COMPUTE_INTERVAL,
                   OBSERVER_MSE_HIST_BINS, OBSERVER_PERCENTILE, OBSERVER_PERCENTILE_MANUL_OVERRIDE, QuantizationProperty,
                   QuantizationStates, TensorQuantizationConfig, set_state, state_is)
from .ffi import CUDA, CUDA_COMPLIER


def _ext():
    return CUDA_COMPLIER.CUDA_EXTENSION


def _min_scale(cfg) -> float:
    return cfg.detail.get(OBSERVER_MIN_SCALE_MANUL_OVERRIDE, OBSERVER_MIN_SCALE)


class StatSlot:
    """One observer's slice of the statistics arena (or a private allocation when used stand-alone)."""

    def __init__(self, device, channels: Optional[int] = None, bins: int = 0, arena: 'StatArena' = None, index: int = -1):
        self.arena, self.index = arena, index
        if arena is not None:
            self.minmax = arena.minmax[index]                    # float[2] view
            self.hist = arena.hist[index] if bins else None      # int32[bins] view
            self.hist_scale = arena.hist_scale[index:index + 1]
        else:
            self.minmax = torch.empty(2, dtype=torch.float32, device=device)
            _ext().MinMax_Init(self.minmax[0:1], self.minmax[1:2])
            self.hist = torch.zeros(bins, dtype=torch.int32, device=device) if bins else None
            self.hist_scale = torch.zeros(1, dtype=torch.float32, device=device)
        self.cmins = self.cmaxs = None
        if channels is not None:
            self.cmins = torch.empty(channels, dtype=torch.float32, device=device)
            self.cmaxs = torch.empty(channels, dtype=torch.float32, device=device)
            _ext().MinMax_Init(self.cmins, self.cmaxs)


class StatArena:
    """Contiguous device buffers for T per-tensor observers: minmax [T,2] fp32, hist [T,bins] int32, hist_scale [T] fp32.
    One all-reduce per calibration phase runs over `minmax` (max on {-min, max}) and `hist` (sum)."""

    def __init__(self, slots: int, bins: int, device):
        self.slots, self.bins, self.device = slots, bins, device
        self.minmax = torch.empty(slots, 2, dtype=torch.float32, device=device)
        self.reset_minmax()
        self.hist = torch.zeros(slots, max(bins, 1), dtype=torch.int32, device=device)
        self.hist_scale = torch.zeros(slots, dtype=torch.float32, device=device)

    def reset_minmax(self):
        self.minmax[:, 0] = float('inf')
        self.minmax[:, 1] = float('-inf')


class BaseTensorObserver:
    """observer/base.py:9-33."""

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig):
        self._watch_on = watch_on
        self._quant_cfg = quant_cfg

    def observe(self, value):
        raise NotImplementedError('Implement this function first.')

    def render_quantization_config(self):
        raise NotImplementedError('Implement this function first.')

    def report(self):
        return None


class TorchMinMaxObserver(BaseTensorObserver):
    """range.py:78-137, fused single pass on the device."""

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig, slot: StatSlot = None, bins: int = 0):
        super().__init__(watch_on, quant_cfg)
        self._slot = slot
        self._bins = bins
        self._observed = 0

    def _ensure_slot(self, value: torch.Tensor):
        per_channel = self._quant_cfg.policy.has_property(QuantizationProperty.PER_CHANNEL)
        if self._slot is None:
            self._slot = StatSlot(value.device, channels=value.shape[self._quant_cfg.channel_axis] if per_channel else None,
                                  bins=self._bins)
        elif per_channel and self._slot.cmins is None:
            C = value.shape[self._quant_cfg.channel_axis]
            self._slot.cmins = torch.empty(C, dtype=torch.float32, device=value.device)
            self._slot.cmaxs = torch.empty(C, dtype=torch.float32, device=value.device)
            _ext().MinMax_Init(self._slot.cmins, self._slot.cmaxs)

    @torch.no_grad()
    def observe(self, value: torch.Tensor):
        assert isinstance(value, torch.Tensor), 'TorchMinMaxObserver can only deal with torch Tensor values'
        assert value.numel() > 0, 'You are observing an empty tensor.'
        if not state_is(self._quant_cfg, 'INITIAL'): return
        self._ensure_slot(value)
        if self._quant_cfg.policy.has_property(QuantizationProperty.PER_TENSOR):
            CUDA.MinMax_T(value, self._slot.minmax)
        elif self._quant_cfg.policy.has_property(QuantizationProperty.PER_CHANNEL):
            CUDA.MinMax_C(value, self._quant_cfg.channel_axis, self._slot.cmins, self._slot.cmaxs)
        else:
            raise TypeError('Min-max Observer only work with per-tensor or per-channel quantize policy.')
        self._observed += 1

    def render_quantization_config(self):
        cfg = self._quant_cfg
        if not state_is(cfg, 'INITIAL'): return
        if self._observed == 0:
            raise ValueError('Can not render quantization config yet, Observer data collator is empty. '
                             'Invoke observe() function before render config.')
        sym = cfg.policy.has_property(QuantizationProperty.SYMMETRICAL)
        if not sym and not cfg.policy.has_property(QuantizationProperty.ASYMMETRICAL):
            raise TypeError('Tensor Min Max Observer Excepts either ASYMMETRICAL or SYMMETRICAL quantization config.')
        pow2 = cfg.policy.has_property(QuantizationProperty.POWER_OF_2)
        if cfg.policy.has_property(QuantizationProperty.PER_TENSOR):
            mm = self._slot.minmax
            scale, offset = _ext().MinMax_To_Scale_Offset(mm[0:1], mm[1:2], 1, cfg.quant_min, cfg.quant_max, sym, pow2, _min_scale(cfg))
            cfg.scale, cfg.offset = scale.squeeze(0), offset.squeeze(0)
        else:
            cfg.scale, cfg.offset = _ext().MinMax_To_Scale_Offset(self._slot.cmins, self._slot.cmaxs, 1, cfg.quant_min, cfg.quant_max,
                                                                  sym, pow2, _min_scale(cfg))
        set_state(cfg, 'ACTIVATED')


class TorchHistObserver(TorchMinMaxObserver):
    """range.py:140-309: two-phase KL observer.  Phase 1 = min/max; render -> hist_scale (kept on the device);
    phase 2 = Histogram_T with the device-resident scale; render -> KL search on the device."""

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig, hist_bins: int = OBSERVER_KL_HIST_BINS, slot: StatSlot = None):
        if OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE in quant_cfg.detail:
            hist_bins = quant_cfg.detail[OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE]
        self._phase = 'Detecting Minmax'
        self._hist_bins = hist_bins
        self._min = self._max = None
        super().__init__(watch_on, quant_cfg, slot=slot, bins=hist_bins)

    @property
    def _hist(self):
        return self._slot.hist

    @property
    def _hist_scale(self):
        return self._slot.hist_scale

    def observe(self, value: torch.Tensor):
        if not state_is(self._quant_cfg, 'INITIAL'): return
        assert value.numel() > 0, 'You are observing an empty tensor.'
        if self._phase == 'Detecting Minmax':
            return super().observe(value)
        if self._quant_cfg.policy.has_property(QuantizationProperty.ASYMMETRICAL):
            CUDA.Histogram_Asymmetric_T(self._min, self._max, tensor=value, histogram=self._slot.hist)
        elif self._quant_cfg.policy.has_property(QuantizationProperty.SYMMETRICAL):
            _ext().Histogram_T_DeviceScale(value, self._slot.hist_scale, True, self._slot.hist)
        else:
            raise TypeError('Quantization Property is invalid, expect either ASYMMETRICAL or SYMMETRICAL config here.')

    def _render_phase1(self):
        cfg = self._quant_cfg
        sym = cfg.policy.has_property(QuantizationProperty.SYMMETRICAL)
        hs = _ext().Hist_Scale_From_MinMax(self._slot.minmax, sym, self._hist_bins)
        self._slot.hist_scale.copy_(hs)
        if not sym:
            # the asymmetric kernel takes min / max by value (sort.h:19-23): one host read per tensor, as upstream
            self._min, self._max = (float(v) for v in self._slot.minmax.tolist())
        self._phase = 'Collating Hist'

    def hist_to_scale_offset(self):
        cfg = self._quant_cfg
        if cfg.policy.has_property(QuantizationProperty.ASYMMETRICAL):
            raise PermissionError('KL observer is not designed for ASYMMETRICAL quantization')
        scale, _best = _ext().KL_Search(self._slot.hist.view(1, -1), self._hist_bins, self._slot.hist_scale, self._slot.minmax, cfg.num_of_bits,
                                        cfg.policy.has_property(QuantizationProperty.POWER_OF_2), _min_scale(cfg))
        return scale.squeeze(0), torch.zeros((), dtype=torch.float32, device=scale.device)

    def render_quantization_config(self):
        cfg = self._quant_cfg
        if not state_is(cfg, 'INITIAL'): return
        if not cfg.policy.has_property(QuantizationProperty.PER_TENSOR):
            raise ValueError('Hist observer can only apply with per-tensor quantization config.')
        if self._phase == 'Detecting Minmax':
            if self._observed == 0:
                raise ValueError('Can not render quantization config yet, Observer data collator is empty.')
            self._render_phase1()
        elif self._phase == 'Collating Hist':
            cfg.scale, cfg.offset = self.hist_to_scale_offset()
            set_state(cfg, 'ACTIVATED')


class TorchMSEObserver(TorchHistObserver):
    """range.py:406-520: histogram-accelerated MSE search.  The grid search drives compute_mse_loss exactly like the
    reference does with USING_CUDA_KERNEL=True (ffi.py:263-270 -> hist_mse.cc); histogram collection is the sm_90a kernel."""

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig, bins: int = OBSERVER_MSE_HIST_BINS, slot: StatSlot = None):
        super().__init__(watch_on, quant_cfg, hist_bins=bins, slot=slot)
        self._hist_bins = bins
        self._bins = bins

    def _render_phase1(self):
        super()._render_phase1()
        if self._min is None:
            self._min, self._max = (float(v) for v in self._slot.minmax.tolist())

    def hist_to_scale_offset(self):
        """Device grid search (MSE_Search): every candidate's loss is the bit-exact serial fp32 accumulation of compute_mse_loss, the first
        minimum wins like python's stable sort, the winning range goes through minmax_to_scale_offset in fp64 -- no histogram D2H, no host loop.
        `ppq_b200.search.mse_search_host` keeps the reference's host formulation (CUDA.compute_mse_loss per candidate) for cross-checking."""
        cfg = self._quant_cfg
        if cfg.policy.has_property(QuantizationProperty.PER_CHANNEL):
            raise PermissionError('Torch Mse observer do not support PER_CHANNEL policy now, please wait.')
        scale, offset = _ext().MSE_Search(self._slot.hist.view(1, -1), self._hist_bins, self._slot.minmax,
                                          cfg.quant_min, cfg.quant_max, cfg.policy.has_property(QuantizationProperty.SYMMETRICAL),
                                          cfg.policy.has_property(QuantizationProperty.POWER_OF_2), _min_scale(cfg), OBSERVER_MSE_COMPUTE_INTERVAL)
        return scale.squeeze(0), offset.squeeze(0)


class TorchPercentileObserver(BaseTensorObserver):
    """range.py:312-403: per batch the values at sorted index rn(N*q) / rn(N*(1-q)) (CUDA.Quantile), averaged over batches."""

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig):
        super().__init__(watch_on, quant_cfg)
        self._percentile = quant_cfg.detail.get(OBSERVER_PERCENTILE_MANUL_OVERRIDE, OBSERVER_PERCENTILE)
        self._percentile_collector = []
        self._guess = None                      # thresholds remembered from the previous batch: the select reads a batch once when they still hold

    @torch.no_grad()
    def observe(self, value: torch.Tensor):
        if not state_is(self._quant_cfg, 'INITIAL'): return
        assert value is not None and value.numel() > 0, 'You are observing an empty tensor.'
        if self._quant_cfg.policy.has_property(QuantizationProperty.PER_TENSOR):
            if not value.is_cuda:
                self._percentile_collector.append(CUDA.Quantile(value, self._percentile).view(1, -1))       # raises: there is no CPU path here
            else:
                if self._guess is None or self._guess.device != value.device: self._guess = _ext().Quantile_Guess_Init(1, value)
                self._percentile_collector.append(_ext().Quantile_T_Guess(value, self._percentile, self._guess).view(1, -1))
        elif self._quant_cfg.policy.has_property(QuantizationProperty.PER_CHANNEL):
            raise PermissionError('Percentile observer can not deal with per channel quantization.')
        else:
            raise TypeError('Min-max Observer only work with per-tensor or per-channel quantize policy.')

    def render_quantization_config(self):
        cfg = self._quant_cfg
        if not state_is(cfg, 'INITIAL'): return
        if not cfg.policy.has_property(QuantizationProperty.PER_TENSOR):
            raise PermissionError('Percentile observer can not deal with per channel quantization.')
        if len(self._percentile_collector) == 0:
            raise ValueError('Can not render quantization config yet, Observer data collator is empty. '
                             'Invoke observe() function before render config.')
        mean = torch.cat(self._percentile_collector, dim=0).float().mean(dim=0)      # [upper, lower], fp32 mean as upstream
        scale, offset = _ext().MinMax_To_Scale_Offset(mean[1:2].contiguous(), mean[0:1].contiguous(), 1, cfg.quant_min, cfg.quant_max,
                                                      cfg.policy.has_property(QuantizationProperty.SYMMETRICAL),
                                                      cfg.policy.has_property(QuantizationProperty.POWER_OF_2), _min_scale(cfg))
        cfg.scale, cfg.offset = scale.squeeze(0), offset.squeeze(0)
        set_state(cfg, 'ACTIVATED')


class ConstantObserver(BaseTensorObserver):
    """observer/floating.py:11-48: scale = 1, offset = 0 (FP8 default)."""

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig):
        super().__init__(watch_on, quant_cfg)
        self._value_shape = self._value_device = None

    @torch.no_grad()
    def observe(self, value: torch.Tensor):
        if not state_is(self._quant_cfg, 'INITIAL'): return
        self._value_shape, self._value_device = value.shape, value.device

    def render_quantization_config(self):
        cfg = self._quant_cfg
        if not state_is(cfg, 'INITIAL'): return
        if not cfg.policy.has_property(QuantizationProperty.FLOATING):
            raise TypeError('This Observer is designed for floating quantization.')
        n = 1 if cfg.policy.has_property(QuantizationProperty.PER_TENSOR) else self._value_shape[cfg.channel_axis]
        scale = torch.ones(n, dtype=torch.float32, device=self._value_device)
        offset = torch.zeros(n, dtype=torch.float32, device=self._value_device)
        if cfg.policy.has_property(QuantizationProperty.PER_TENSOR): scale, offset = scale.squeeze(0), offset.squeeze(0)
        cfg.scale, cfg.offset = scale, offset
        set_state(cfg, 'ACTIVATED')


class DirectMSEObserver(BaseTensorObserver):
    """observer/floating.py:51-144: pick the power-of-two scale (7 candidates) with the smallest fake-quant MSE over
    randomly fetched samples.  The fetch uses torch.randint like ppq/utils/fetch.py:26-29 (RNG dependent upstream too)."""
    SCALE_CANDIDATES = [.0078125, .03125, .125, 1.0, 4.0, 16.0, 64.0]

    def __init__(self, watch_on, quant_cfg: TensorQuantizationConfig, is_parameter: bool = False):
        super().__init__(watch_on, quant_cfg)
        if not quant_cfg.policy.has_property(QuantizationProperty.FLOATING):
            raise TypeError('MSE Floating Observer is designed for floating quantization.')
        if not quant_cfg.policy.has_property(QuantizationProperty.POWER_OF_2):
            raise TypeError('MSE Floating Observer is designed for power-of-2 quantization.')
        self._collector, self._fetches, self._is_parameter = [], OBSERVER_FLOATING_MSE_FETCHES, is_parameter

    @torch.no_grad()
    def observe(self, value: torch.Tensor):
        cfg = self._quant_cfg
        if not state_is(cfg, 'INITIAL'): return
        if cfg.policy.has_property(QuantizationProperty.PER_CHANNEL):
            v = torch.transpose(value, 0, cfg.channel_axis).flatten(1)
            if not self._is_parameter:
                idx = torch.randint(0, v.shape[1], (self._fetches,), device=v.device)
                v = v.index_select(1, idx)
            self._collector.append(v)
        else:
            flat = value.flatten()
            idx = torch.randint(0, flat.numel(), (self._fetches,), device=flat.device)
            self._collector.append(flat.index_select(0, idx))

    def render_quantization_config(self):
        from .qfunction import PPQuantFunction
        cfg = self._quant_cfg
        if not state_is(cfg, 'INITIAL'): return
        if not self._collector:
            raise PermissionError('Observer collector is empty, you should invoke observe function before render quantization config.')
        set_state(cfg, 'ACTIVATED')
        per_channel = cfg.policy.has_property(QuantizationProperty.PER_CHANNEL)
        data = torch.cat(self._collector, dim=-1 if per_channel else 0).contiguous()
        n = data.shape[0] if per_channel else 1
        cand = torch.tensor(self.SCALE_CANDIDATES, dtype=torch.float32, device=data.device)
        saved_axis = cfg.channel_axis
        if per_channel: cfg.channel_axis = 0
        cfg.offset = torch.zeros(n, dtype=torch.float32, device=data.device) if per_channel else torch.zeros((), device=data.device)
        losses = []
        for s in self.SCALE_CANDIDATES:
            cfg.scale = torch.full((n,), s, dtype=torch.float32, device=data.device) if per_channel else torch.tensor(s, device=data.device)
            qt = PPQuantFunction(data, cfg)
            losses.append(torch.mean(torch.square(qt - data), dim=-1, keepdim=True) if per_channel else torch.mean(torch.square(qt - data)).view(1))
        best = torch.argmin(torch.cat(losses, dim=-1), dim=-1)
        cfg.channel_axis = saved_axis
        cfg.scale = cand[best] if per_channel else cand[best].squeeze()


OBSERVER_TABLE = {
    'minmax': TorchMinMaxObserver,
    'kl': TorchHistObserver,
    'percentile': TorchPercentileObserver,
    'mse': TorchMSEObserver,
    'constant': ConstantObserver,
    'floating': DirectMSEObserver,
}


class TensorObserverFactroy:
    """observer/__init__.py:25-37 (spelling as upstream)."""

    @classmethod
    def build_observer(cls, variable, config: TensorQuantizationConfig, **kw) -> BaseTensorObserver:
        algorithm = str(config.observer_algorithm.lower())
        if algorithm not in OBSERVER_TABLE:
            raise ValueError(f'Observer type not understand, Except one of {OBSERVER_TABLE.keys()}, while {str(algorithm)} was given.')
        return OBSERVER_TABLE[algorithm](watch_on=variable, quant_cfg=config, **kw)


def Observer(quant_config: TensorQuantizationConfig, variable=None, **kw) -> BaseTensorObserver:
    """ppq/lib/quant.py:47-55."""
    return TensorObserverFactroy.build_observer(variable=variable, config=quant_config, **kw)
