"""Calibration drivers: the mirror of RuntimeCalibrationPass (/root/reference/ppq/quantization/optim/calibration.py:19-213)
re-designed around a device-resident statistics arena and sample-sharded data parallelism (SURVEY.md §8e).

  ArenaCalibrator          the H100-native two-phase calibrator.  All T observed tensors of one forward are collected by ONE
                           multi-tensor launch per phase (Multi_MinMax_T / Multi_Histogram_T) into one contiguous arena:
                               minmax [T,2] fp32,  hist_scale [T] fp32,  hist [T,bins] int32.
                           Rank r of R processes sees samples r, r+R, ...; the whole multi-GPU exchange is
                               phase 1:  ONE all-reduce(MAX) over the packed {-min, max} buffer      (2*T floats)
                               phase 2:  ONE all-reduce(SUM) over the int32 histogram arena           (T*bins ints)
                           both exact and order-independent, so R ranks reproduce the 1-rank result bit for bit.
                           Scales come from the on-device searches (MinMax_To_Scale_Offset, KL_Search): no per-tensor host sync.
  RuntimeCalibrationPass   the reference's hook-driven flow (build observers -> phase 1 over the dataloader -> render -> drop the
                           one-phase observers -> phase 2 -> render) for any executor with forward(inputs, hooks=...), using the
                           observers of ppq_b200.observer; `calib_steps` keeps the reference's 8..512 contract.
"""
from math import ceil
from typing import Callable, Dict, Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist

from .core import (OBSERVER_KL_HIST_BINS, OBSERVER_MIN_SCALE, OBSERVER_MSE_COMPUTE_INTERVAL, OBSERVER_MSE_HIST_BINS, OBSERVER_PERCENTILE,
                   QuantizationProperty, QuantizationStates)


# ---- the two exchange steps (pure torch.distributed; CPU/gloo-testable) --------------------------------------------------------
def pack_minmax_for_max_reduce(minmax: torch.Tensor) -> torch.Tensor:
    """[T,2] {min,max} -> [T,2] {-min, max}: a single MAX all-reduce then reduces both ends exactly."""
    packed = minmax.clone()
    packed[:, 0].neg_()
    return packed


def unpack_minmax_after_max_reduce(packed: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    out.copy_(packed)
    out[:, 0].neg_()
    return out


def allreduce_minmax(minmax: torch.Tensor, group=None) -> torch.Tensor:
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        packed = pack_minmax_for_max_reduce(minmax)
        dist.all_reduce(packed, op=dist.ReduceOp.MAX, group=group)
        unpack_minmax_after_max_reduce(packed, minmax)
    return minmax


def allreduce_hist(hist: torch.Tensor, group=None) -> torch.Tensor:
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(hist, op=dist.ReduceOp.SUM, group=group)
    return hist


def gather_in_sample_order(local: torch.Tensor, group=None) -> torch.Tensor:
    """local: [T, n_local, 2] per-batch statistics of this rank (batch j of rank r is global batch r + j*R).  Returns [T, n_total, 2] in
    global batch order on every rank (all-gather; ranks may hold n_local differing by one)."""
    world = dist.get_world_size(group); rank = dist.get_rank(group)
    n_local = torch.tensor([local.shape[1]], device=local.device)
    counts = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(counts, n_local, group=group)
    counts = [int(c.item()) for c in counts]
    nmax = max(counts)
    pad = torch.zeros(local.shape[0], nmax, local.shape[2], dtype=local.dtype, device=local.device)
    pad[:, :local.shape[1]] = local
    parts = [torch.zeros_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    rows = []
    for j in range(nmax):
        for r in range(world):
            if j < counts[r]: rows.append(parts[r][:, j])
    return torch.stack(rows, dim=1)


def is_dense(t: torch.Tensor) -> bool:
    """Contiguous in some memory format (NCHW or channels_last): per-tensor collectors and element-wise operators are order-independent, so
    such a tensor is processed in storage order without a copy."""
    if t.is_contiguous(): return True
    if t.dim() == 4: return t.is_contiguous(memory_format=torch.channels_last)
    if t.dim() == 5: return t.is_contiguous(memory_format=torch.channels_last_3d)
    return False


def shard_indices(num_samples: int, rank: int, world_size: int) -> range:
    """Sample partition of SURVEY §8e: rank r takes samples r, r + R, r + 2R, ..."""
    return range(rank, num_samples, world_size)


# ---- arena calibrator -------------------------------------------------------------------------------------------------------------
class DescriptorStager:
    """Host -> device upload of small descriptor tables without cudaHostAlloc on the hot path: a ring of persistent pinned staging
    buffers (an event per slot guards reuse), cudaMemcpyAsync on the current stream.  Tables are cached by content (LRU)."""

    def __init__(self, device, columns: int, rows: int = 256, ring: int = 8, cache: int = 128):
        self.device, self.columns, self.ring, self.cache_size = torch.device(device), columns, ring, cache
        self._rows = rows
        self._host = [self._alloc(rows) for _ in range(ring)] if self.device.type == 'cuda' else None
        self._events, self._k, self._cache = [None] * ring, 0, {}

    def _alloc(self, rows):
        return torch.empty(rows, self.columns, dtype=torch.int64).pin_memory()

    def get(self, key: tuple) -> torch.Tensor:
        """key: tuple of row tuples (ints).  Returns the [len(key), columns] int64 device tensor holding it."""
        hit = self._cache.pop(key, None)
        if hit is None:
            table = torch.tensor(key, dtype=torch.int64).reshape(len(key), self.columns)
            if self._host is None:
                hit = table.to(self.device)
            else:
                if len(key) > self._rows:                                # grow every slot once (rare: a bigger network than sized for)
                    torch.cuda.synchronize(self.device)
                    self._rows = max(len(key), 2 * self._rows)
                    self._host = [self._alloc(self._rows) for _ in range(self.ring)]
                    self._events = [None] * self.ring
                i = self._k % self.ring; self._k += 1
                if self._events[i] is not None: self._events[i].synchronize()
                stage = self._host[i][:len(key)]
                stage.copy_(table)
                hit = torch.empty(len(key), self.columns, dtype=torch.int64, device=self.device)
                hit.copy_(stage, non_blocking=True)
                ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(self.device)); self._events[i] = ev
            while len(self._cache) >= self.cache_size: self._cache.pop(next(iter(self._cache)))      # evict the least recently used
        self._cache[key] = hit                                            # (re-)insert as most recent
        return hit


_STAGERS: Dict[tuple, DescriptorStager] = {}


def shared_stager(device, columns: int) -> DescriptorStager:
    """One stager per (device, table width) for the whole process: its pinned buffers are allocated once (cudaHostAlloc / cudaFreeHost synchronise
    the device -- a calibrator that made its own ring paid that on every calibration)."""
    key = (str(torch.device(device)), columns)
    if key not in _STAGERS: _STAGERS[key] = DescriptorStager(device, columns)
    return _STAGERS[key]


TABLE_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def descriptor_rows_by_dtype(tensors: Sequence[torch.Tensor], slots: Sequence[int]) -> Dict[torch.dtype, tuple]:
    """The (data_ptr, numel, slot) rows of a collector table, one tuple of rows per element type: a table carries raw pointers and one
    element type, so a mixed set of tensors (an fp32 network under autocast) becomes one table -- one launch -- per dtype present.  Every
    tensor keeps its slot; groups appear in the order their dtype is first met and rows keep the order of `tensors`."""
    groups: Dict[torch.dtype, list] = {}
    for t, i in zip(tensors, slots):
        groups.setdefault(t.dtype, []).append((t.data_ptr(), t.numel(), i))
    return {dtype: tuple(rows) for dtype, rows in groups.items()}


ARENA_MAX_HIST_BINS = 12287          # the multi-tensor histogram keeps (bins + 1) private counters in 48 KB of shared memory


class ArenaCalibrator:
    """method:  'minmax'      one phase: fused min/max                       -> MinMax_To_Scale_Offset
                'kl'          + phase 2: 4096-bin histogram                  -> KL_Search (symmetric configs only, as upstream)
                'mse'         + phase 2: 2048-bin histogram                  -> MSE_Search (symmetric configs; range.py:406-520)
                'percentile'  one phase: Quantile_T of every tensor and batch (ONE multi-tensor select per forward), fp32 mean over the
                              batches in sample order                        -> MinMax_To_Scale_Offset   (range.py:312-403)
    All T tensors share one per-tensor config: range (quant_min, quant_max, num_of_bits), symmetrical, power_of_2 and min_scale.  The
    histogram of both two-phase methods is symmetric (|x| binned from 0), so asymmetric 'kl' / 'mse' are refused, as are more than
    ARENA_MAX_HIST_BINS bins.
    half_inputs=True also takes fp16 / bf16 tensors (the *_Half table kernels: the same statistics, bit for bit, as on x.float()); the
    tensors of one `observe` call may mix element types and are served by one launch per type present.
    max_batches (percentile only) makes the per-batch rows static, for a forward captured into a CUDA graph: one [max_batches, T, 2] buffer
    and a device int64 batch counter replace the growing list.  The forward writes its quantiles into one static [T, 2] staging row,
    observe_one selects through the slot's guess row (Quantile_T_Guess: exact, one pass when the previous batch's thresholds still hold), and
    end_batch() files the staging row as row `counter` with one scatter and advances the counter.  begin_batch() raises before a batch
    that would overrun the buffer."""

    def __init__(self, num_tensors: int, device, bins: int = None, num_of_bits: int = 8,
                 quant_min: int = -128, quant_max: int = 127, power_of_2: bool = False, min_scale: float = OBSERVER_MIN_SCALE,
                 method: str = 'kl', group=None, percentile: float = OBSERVER_PERCENTILE, select_cap: int = 1 << 16,
                 symmetrical: bool = True, half_inputs: bool = False, max_batches: Optional[int] = None):
        from .ffi import extension
        if method not in ('kl', 'minmax', 'mse', 'percentile'):
            raise ValueError(f"ArenaCalibrator: unknown observer algorithm {method!r} (expected 'kl', 'minmax', 'mse' or 'percentile')")
        if max_batches is not None and (method != 'percentile' or max_batches < 0):
            raise ValueError(f'ArenaCalibrator: max_batches={max_batches} (static per-batch rows serve the percentile observer, >= 0 batches)')
        if method == 'kl' and not symmetrical:
            raise PermissionError('KL observer is not designed for ASYMMETRICAL quantization')
        if method == 'mse' and not symmetrical:
            raise ValueError('ArenaCalibrator: the arena histogram is symmetric; asymmetric mse calibration needs the per-observer '
                             'RuntimeCalibrationPass')
        if bins is None: bins = OBSERVER_MSE_HIST_BINS if method == 'mse' else OBSERVER_KL_HIST_BINS
        if method in ('kl', 'mse') and bins > ARENA_MAX_HIST_BINS:
            raise ValueError(f'ArenaCalibrator: {bins} histogram bins, the multi-tensor histogram holds at most {ARENA_MAX_HIST_BINS}; '
                             'use RuntimeCalibrationPass for larger histograms')
        self.ext = extension()
        self.T, self.bins, self.device, self.group = num_tensors, bins, torch.device(device), group
        self.num_of_bits, self.quant_min, self.quant_max = num_of_bits, quant_min, quant_max
        self.power_of_2, self.min_scale, self.method, self.symmetrical = power_of_2, min_scale, method, symmetrical
        self.percentile, self.select_cap, self.half_inputs = percentile, select_cap, half_inputs
        self.minmax = torch.empty(num_tensors, 2, dtype=torch.float32, device=self.device)
        two_phase = method in ('kl', 'mse')
        self.hist = torch.zeros(num_tensors, bins if two_phase else 1, dtype=torch.int32, device=self.device)
        self.hist_scale = torch.zeros(num_tensors, dtype=torch.float32, device=self.device)
        self.scale = self.offset = self.best_bin_range = None
        self._stager = shared_stager(self.device, 3)
        self._pct: List[torch.Tensor] = []                               # per batch: [T, 2] {upper, lower} quantiles
        self._rows = self._staging = self._count = None
        if max_batches is not None:
            self._rows = torch.zeros(max_batches, num_tensors, 2, dtype=torch.float32, device=self.device)
            self._staging = torch.zeros(num_tensors, 2, dtype=torch.float32, device=self.device)
            self._count = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._begun = 0                                                  # batches begun on the host: guards the static rows
        self._select_ws = None
        # per-slot thresholds remembered from the previous batch: consecutive batches of one activation are selected in ONE pass over the tensor
        self._select_guess = self.ext.Quantile_Guess_Init(num_tensors, self.minmax) if (method == 'percentile' and self.device.type == 'cuda') else None
        self.exchange_events = None                                      # set to a dict to time the exchange steps with CUDA events
        self.launches = 0
        self.reset()

    def reset(self):
        self.minmax[:, 0] = float('inf'); self.minmax[:, 1] = float('-inf')
        self.hist.zero_()
        self._pct = []
        if self._count is not None: self._count.zero_()
        self._begun = 0
        self.phase = 1

    def _descs(self, tensors: Sequence[torch.Tensor], slots: Optional[Sequence[int]] = None):
        if slots is None:
            assert len(tensors) == self.T, f'expected {self.T} tensors per forward, got {len(tensors)}'
            slots = range(self.T)
        allowed = TABLE_DTYPES if self.half_inputs else (torch.float32,)
        for t in tensors:
            if not (t.is_cuda and t.dtype in allowed and is_dense(t)):
                raise RuntimeError('ArenaCalibrator needs dense (contiguous or channels_last) ' +
                                   ('fp32, fp16 or bf16' if self.half_inputs else 'fp32') + ' CUDA tensors')
        return [(dtype, self._stager.get(rows), max(r[1] for r in rows)) for dtype, rows in descriptor_rows_by_dtype(tensors, slots).items()]

    def begin_batch(self):
        """Call before every forward: the percentile observer keeps one {upper, lower} row per batch (range.py:349), whatever number of
        launches the forward's tensors are observed with."""
        if self.method == 'percentile' and self._rows is not None:
            if self._begun >= self._rows.shape[0]:
                raise RuntimeError(f'ArenaCalibrator: batch {self._begun + 1} overruns the {self._rows.shape[0]} per-batch rows allocated '
                                   'for a captured forward (max_batches)')
            self._begun += 1
        elif self.method == 'percentile':
            self._pct.append(torch.zeros(self.T, 2, dtype=torch.float32, device=self.device))

    def end_batch(self):
        """Call after every forward when the rows are static (max_batches; inside the captured graph): the staging row becomes row `counter`
        through one device-indexed scatter, then the counter advances.  No host value is read, so every replay files its own row."""
        if self._rows is None: return
        self._rows.index_copy_(0, self._count, self._staging[None])
        self._count.add_(1)

    def replay_state(self) -> List[torch.Tensor]:
        """The device buffers a forward updates in place: a warm-up forward run before a capture must leave them as it found them."""
        return [t for t in (self.minmax, self.hist, self._select_guess if self._rows is not None else None, self._count) if t is not None]

    def batch_rows(self) -> torch.Tensor:
        """Percentile: [T, batches, 2] {upper, lower} quantiles of this rank's batches, in batch order (static rows: the first `counter`)."""
        if self._rows is not None:
            return self._rows[:int(self._count.item())].transpose(0, 1).contiguous()
        if not self._pct: return torch.zeros(self.T, 0, 2, dtype=torch.float32, device=self.device)
        return torch.stack(self._pct, dim=1)

    def _batch_quantiles(self) -> torch.Tensor:
        if self._staging is not None: return self._staging
        if not self._pct: self.begin_batch()
        return self._pct[-1]

    @torch.no_grad()
    def observe(self, tensors: Sequence[torch.Tensor], slots: Optional[Sequence[int]] = None):
        """One multi-tensor launch per element type present in `tensors` (one for an all-fp32 or all-half forward, two under autocast);
        tensor j accumulates into arena slot slots[j] (default: j)."""
        if len(tensors) == 0: return
        groups = self._descs(tensors, slots)
        if self.method == 'percentile':
            need = self.ext.Multi_Quantile_Workspace_Bytes(len(tensors), self.select_cap)      # sized for the whole set: every group fits
            if self._select_ws is None or self._select_ws.numel() < need:
                self._select_ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        for dtype, descs, max_n in groups:
            half = (dtype,) if dtype != torch.float32 else ()
            ext, suffix = self.ext, '_Half' if half else ''
            if self.method == 'percentile':
                getattr(ext, 'Multi_Quantile_T' + suffix)(descs, max_n, *half, self.percentile, self._batch_quantiles(), 2, self._select_ws,
                                                          self.select_cap, self._select_guess)
                self.launches += 5
            elif self.phase == 1:
                getattr(ext, 'Multi_MinMax_T' + suffix)(descs, max_n, *half, self.minmax)
                self.launches += 1
            else:
                getattr(ext, 'Multi_Histogram_T' + suffix)(descs, max_n, *half, self.hist_scale, True, self.hist, self.bins)
                self.launches += 1

    @torch.no_grad()
    def observe_one(self, index: int, tensor: torch.Tensor):
        """Immediate single-tensor collection into slot `index` (used while a forward is running: later in-place ops of the
        network may overwrite the tensor, so it cannot wait for the end-of-forward multi-tensor launch)."""
        if self.method == 'percentile':
            if self._rows is not None:
                self._staging[index].copy_(self.ext.Quantile_T_Guess(tensor, self.percentile, self._select_guess[index]))
            else:
                quantile = self.ext.Quantile_T if tensor.dtype == torch.float32 else self.ext.Quantile_T_Half
                self._batch_quantiles()[index].copy_(quantile(tensor, self.percentile))
            self.launches += 5
            return
        if self.phase == 1:
            self.ext.MinMax_T(tensor, self.minmax[index])
        else:
            self.ext.Histogram_T_DeviceScale(tensor, self.hist_scale[index:index + 1], True, self.hist[index])
        self.launches += 1

    def _timed_exchange(self, name: str):
        """CUDA events around one exchange step when `self.exchange_events` is a dict (bench.py's scaling report), else a no-op."""
        import contextlib
        ev = self.exchange_events
        if ev is None or not self.minmax.is_cuda: return contextlib.nullcontext()

        @contextlib.contextmanager
        def ctx():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(torch.cuda.current_stream(self.device))
            yield
            b.record(torch.cuda.current_stream(self.device))
            ev.setdefault(name, []).append((a, b))
        return ctx()

    def _distributed(self) -> bool:
        return dist.is_available() and dist.is_initialized() and dist.get_world_size(self.group) > 1

    @torch.no_grad()
    def end_phase(self):
        """Exchange + render of the finished phase.  Returns True when calibration is complete."""
        sym = self.symmetrical
        if self.method == 'percentile':
            rows = self.batch_rows()                                     # [T, batches, 2]
            if rows.shape[1] == 0: raise ValueError('Can not render quantization config yet, Observer data collator is empty.')
            if self._distributed():
                with self._timed_exchange('percentile'):
                    rows = gather_in_sample_order(rows, self.group)
            # fp32 mean over the batches, per tensor on a contiguous [batches, 2] block: the reduction the reference runs
            # (torch.cat(collector, dim=0).float().mean(dim=0), range.py:369), so the summation order is torch's for that shape
            mean = torch.stack([rows[t].mean(dim=0) for t in range(rows.shape[0])])
            self.scale, self.offset = self.ext.MinMax_To_Scale_Offset(mean[:, 1].contiguous(), mean[:, 0].contiguous(), 1, self.quant_min,
                                                                      self.quant_max, sym, self.power_of_2, self.min_scale)
            self.launches += 1
            return True
        if self.phase == 1:
            with self._timed_exchange('minmax'):
                allreduce_minmax(self.minmax, self.group)
            if self.method == 'minmax':
                self.scale, self.offset = self.ext.MinMax_To_Scale_Offset(self.minmax.view(-1), self.minmax.view(-1)[1:], 2, self.quant_min,
                                                                          self.quant_max, sym, self.power_of_2, self.min_scale)
                self.launches += 1
                return True
            self.hist_scale = self.ext.Hist_Scale_From_MinMax(self.minmax, sym, self.bins)
            self.launches += 1
            self.phase = 2
            return False
        with self._timed_exchange('hist'):
            allreduce_hist(self.hist, self.group)
        if self.method == 'kl':
            self.scale, self.best_bin_range = self.ext.KL_Search(self.hist, self.bins, self.hist_scale, self.minmax, self.num_of_bits,
                                                                 self.power_of_2, self.min_scale)
            self.offset = torch.zeros_like(self.scale)
        else:
            self.scale, self.offset = self.ext.MSE_Search(self.hist, self.bins, self.minmax, self.quant_min, self.quant_max, sym,
                                                          self.power_of_2, self.min_scale, OBSERVER_MSE_COMPUTE_INTERVAL)
        self.launches += 1
        return True


# ---- hook-driven pass (reference flow) --------------------------------------------------------------------------------------------
class CalibrationHook:
    """observer/__init__.py:40-72: calls observe() on the fp32 inputs / outputs of one quantable operation."""

    def __init__(self, operation, observer_table: dict):
        self._operation, self._observer_table = operation, observer_table

    def pre_forward_hook(self, inputs: list, quant_inputs: list, quant_configs: list) -> list:
        for input_var, quant_config in zip(inputs, quant_configs):
            ob = self._observer_table.get(id(quant_config))
            if ob is not None: ob.observe(input_var)
        return quant_inputs

    def post_forward_hook(self, outputs: list, quant_outputs: list, quant_configs: list) -> list:
        for output_var, quant_config in zip(outputs, quant_configs):
            ob = self._observer_table.get(id(quant_config))
            if ob is not None: ob.observe(output_var)
        return quant_outputs

    def render_quantization_config(self):
        for ob in self._observer_table.values():
            ob.render_quantization_config()


class OperationObserver:
    """observer/__init__.py:75-124."""

    def __init__(self, operation, monitor_parameter: bool = True, monitor_outputs: bool = True, monitor_inputs: bool = True):
        from .observer import TensorObserverFactroy
        table = {}
        for var, config, is_param in operation.input_configs():
            if config.state == QuantizationStates.INITIAL:
                if is_param and monitor_parameter: table[id(config)] = TensorObserverFactroy.build_observer(var, config)
                elif not is_param and monitor_inputs: table[id(config)] = TensorObserverFactroy.build_observer(var, config)
        if monitor_outputs:
            for var, config in operation.output_configs():
                if config.state == QuantizationStates.INITIAL:
                    table[id(config)] = TensorObserverFactroy.build_observer(var, config)
        self._operation, self._hook = operation, CalibrationHook(operation, table)

    @property
    def hook(self) -> CalibrationHook:
        return self._hook

    def render_quantization_config(self):
        self._hook.render_quantization_config()


class RuntimeCalibrationPass:
    """calibration.py:19-213, including the 8 <= calib_steps <= 512 contract (:136-142).  With torch.distributed initialised the
    dataloader is sharded by sample (rank r keeps batches r, r+R, ...) and the observers' arena is all-reduced at the end of each phase."""

    def __init__(self, method: str = None, override: bool = False, calib_steps: int = 32, group=None):
        self._method, self._override, self._calib_steps, self._group = method, override, calib_steps, group
        self._observers, self._collate_fn = {}, None

    def calibrate(self, dataloader: Iterable, executor, hooks: dict):
        world = dist.get_world_size(self._group) if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank(self._group) if world > 1 else 0
        calib_step = 0
        for _ in range(ceil(self._calib_steps / len(dataloader))):
            for idx, data in enumerate(dataloader):
                if world > 1 and idx % world != rank:
                    calib_step += 1
                    if calib_step >= self._calib_steps: break
                    continue
                if self._collate_fn is not None: data = self._collate_fn(data)
                executor.forward(inputs=data, hooks=hooks)
                calib_step += 1
                if calib_step >= self._calib_steps: break
            if calib_step >= self._calib_steps: break

    def _reduce(self, phase: int):
        """The exchange step of a phase: every statistic of every observer is made global before render (SURVEY 8e).  Per-tensor {min, max}
        and per-channel min / max vectors travel in ONE packed MAX all-reduce ({-min, max}: exact), histograms in ONE SUM all-reduce,
        per-batch percentile pairs in an all-gather re-ordered by sample."""
        from .observer import TorchHistObserver, TorchMinMaxObserver, TorchPercentileObserver
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size(self._group) > 1): return
        obs = [ob for o in self._observers.values() for ob in o.hook._observer_table.values()]
        if phase == 1:
            pct = [ob for ob in obs if isinstance(ob, TorchPercentileObserver)]
            mm = [ob for ob in obs if isinstance(ob, TorchMinMaxObserver)]
            # a rank whose shard was empty has no statistics (and no slots): the collectives below would mismatch or hang, so agree on it first
            fed = all(ob._observed > 0 for ob in mm) and all(len(ob._percentile_collector) > 0 for ob in pct)
            dev = next((ob._slot.minmax.device for ob in mm if ob._slot is not None), None)
            if dev is None: dev = next((ob._percentile_collector[0].device for ob in pct if ob._percentile_collector), torch.device('cpu'))
            if dist.get_backend(self._group) == 'nccl' and dev.type != 'cuda': dev = torch.device('cuda', torch.cuda.current_device())
            flag = torch.tensor([1 if fed else 0], dtype=torch.int32, device=dev)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self._group)
            if int(flag.item()) == 0:
                raise RuntimeError('RuntimeCalibrationPass: at least one rank observed no calibration batch (fewer batches than ranks?); '
                                   'every rank needs >= 1 batch of its shard before the statistics can be reduced.')
            if pct:
                # the percentile observer averages per-batch quantile pairs in fp32 (range.py:369): gather every rank's pairs and put
                # them back in global sample order, so the mean is the same sum, in the same order, as the single-process run
                merged = gather_in_sample_order(torch.stack([torch.cat(ob._percentile_collector, dim=0) for ob in pct]), self._group)
                for ob, rows in zip(pct, merged): ob._percentile_collector = [rows]
            if mm:
                parts = []
                for ob in mm:
                    if ob._slot.cmins is None: parts += [-ob._slot.minmax[0:1], ob._slot.minmax[1:2]]
                    else: parts += [-ob._slot.cmins, ob._slot.cmaxs]
                buf = torch.cat(parts)
                dist.all_reduce(buf, op=dist.ReduceOp.MAX, group=self._group)
                at = 0
                for ob in mm:
                    if ob._slot.cmins is None:
                        ob._slot.minmax[0:1].copy_(-buf[at:at + 1]); ob._slot.minmax[1:2].copy_(buf[at + 1:at + 2]); at += 2
                    else:
                        C = ob._slot.cmins.numel()
                        ob._slot.cmins.copy_(-buf[at:at + C]); ob._slot.cmaxs.copy_(buf[at + C:at + 2 * C]); at += 2 * C
        else:
            hs = [ob for ob in obs if isinstance(ob, TorchHistObserver) and ob._slot is not None]
            if hs:
                buf = torch.stack([ob._slot.hist for ob in hs])
                allreduce_hist(buf, self._group)
                for ob, row in zip(hs, buf): ob._slot.hist.copy_(row)

    def optimize(self, graph, dataloader: Iterable, executor, calib_steps: int = 32, collate_fn: Callable = None, **kwargs) -> None:
        from .observer import TorchHistObserver, TorchMSEObserver
        if collate_fn is not None: self._collate_fn = collate_fn
        if calib_steps is not None: self._calib_steps = calib_steps
        assert calib_steps >= 8, 'Insufficient Calibration Detected (at least 8 calibration steps).'
        assert calib_steps <= 512, 'Calibration steps is too large, ppq can quantize your network within 8-512 calibration steps.'
        if self._override:                                   # calibration.py:147-155: re-calibrate already activated activations
            from .core import set_state, state_is
            for _, operation in graph.quantable_operations():
                for _, config, is_param in operation.input_configs():
                    if not is_param and state_is(config, 'ACTIVATED'): set_state(config, 'INITIAL')
                for _, config in operation.output_configs():
                    if state_is(config, 'ACTIVATED'): set_state(config, 'INITIAL')
        hooks = {}
        for op_name, operation in graph.quantable_operations():
            for _, config, is_param in operation.input_configs():
                if not is_param and self._method is not None: config.observer_algorithm = self._method
            for _, config in operation.output_configs():
                if self._method is not None: config.observer_algorithm = self._method
            observer = OperationObserver(operation=operation, monitor_parameter=False)
            self._observers[op_name], hooks[op_name] = observer, observer.hook
        self.calibrate(dataloader, executor, hooks)
        self._reduce(1)
        for observer in self._observers.values(): observer.render_quantization_config()
        for op_name in [n for n, o in self._observers.items()
                        if all(type(v) not in {TorchHistObserver, TorchMSEObserver} for v in o.hook._observer_table.values())]:
            self._observers.pop(op_name); hooks.pop(op_name)
        if len(hooks) > 0:
            self.calibrate(dataloader, executor, hooks)
            self._reduce(2)
            for observer in self._observers.values(): observer.render_quantization_config()


class MultiWeightQuantizer:
    """All per-channel weights of a network fake-quantised by ONE launch (Multi_QuantizeTensor_LC), or -- with channel_axis=None -- any list
    of per-tensor quantised tensors, each with its own (scale, offset), by ONE Multi_QuantizeTensor_LT launch.  The executor re-quantises
    every Conv/Gemm weight on each forward until ParameterBakingPass freezes them (executor/torch.py:516-518); with ~54 small
    tensors per ResNet-50 forward that is launch-latency, not bandwidth -- one descriptor table turns it into one kernel.
    half_inputs=True takes per-channel weights that are all fp16 or all bf16 (Multi_QuantizeTensor_LC_Half: outputs in the weights' dtype,
    the values QuantizeTensor_LC_Half returns per weight); scales and offsets stay fp32.  The per-tensor table is fp32 only."""

    def __init__(self, weights: Sequence[torch.Tensor], scales: Sequence[torch.Tensor], offsets: Sequence[torch.Tensor],
                 channel_axis: Optional[int] = 0, quant_min: int = -128, quant_max: int = 127, rounding: int = 0,
                 half_inputs: bool = False):
        from .ffi import extension
        self.ext = extension()
        self.quant_min, self.quant_max, self.rounding = quant_min, quant_max, rounding
        self.per_tensor = channel_axis is None
        # the descriptor table carries raw pointers and the table kernels read and write fp32: any other dtype must never reach them
        self.dtype = weights[0].dtype if (half_inputs and not self.per_tensor and weights[0].dtype in TABLE_DTYPES) else torch.float32
        bad = sorted({str(t.dtype) for t in weights if t.dtype != self.dtype} |
                     {str(t.dtype) for t in list(scales) + list(offsets) if t.dtype != torch.float32})
        if bad and not half_inputs: raise TypeError(f'MultiWeightQuantizer takes fp32 weights, scales and offsets only, got {", ".join(bad)}.')
        if bad: raise TypeError('MultiWeightQuantizer(half_inputs=True) takes per-channel weights of ONE dtype (fp32, fp16 or bf16) with fp32 '
                                f'scales and offsets, got {", ".join(bad)} next to {self.dtype} weights.')

        def rows_in_storage_order(w):
            # axis-0 channels of a dense tensor whose dim 0 is outermost in memory (NCHW or channels_last weights): the storage already is [C, epc]
            return channel_axis is not None and w.dim() > 0 and channel_axis % w.dim() == 0 and is_dense(w) and w.numel() > 0 and \
                w.stride(0) == w.numel() // w.shape[0]
        self.weights = [w if (is_dense(w) if self.per_tensor else rows_in_storage_order(w)) else w.contiguous() for w in weights]
        self.outputs = [torch.empty_like(w) for w in self.weights]            # preserve_format: same strides as the input
        self.scales = [s.contiguous() for s in scales]
        self.offsets = [o.contiguous() for o in offsets]
        rows = []
        for w, y, s, o in zip(self.weights, self.outputs, self.scales, self.offsets):
            if self.per_tensor:
                assert s.numel() == 1 and o.numel() == 1
                rows.append([w.data_ptr(), y.data_ptr(), s.data_ptr(), o.data_ptr(), w.numel()])
                continue
            axis = channel_axis % w.dim()
            epc = 1
            for d in w.shape[axis + 1:]: epc *= int(d)
            C = int(w.shape[axis])
            assert s.numel() == C and o.numel() == C
            rows.append([w.data_ptr(), y.data_ptr(), s.data_ptr(), o.data_ptr(), w.numel(), epc, C])
        self.max_n = max(r[4] for r in rows)
        table = torch.tensor(rows, dtype=torch.int64).to(self.weights[0].device)
        self.descs = table
        self._tables = [table[i:i + 4096] for i in range(0, len(rows), 4096)]      # the C ABI takes <= 4096 tensors per launch

    @torch.no_grad()
    def __call__(self) -> List[torch.Tensor]:
        if self.dtype != torch.float32:
            for table in self._tables:
                self.ext.Multi_QuantizeTensor_LC_Half(table, self.max_n, self.dtype, self.quant_min, self.quant_max, self.rounding)
            return self.outputs
        launch = self.ext.Multi_QuantizeTensor_LT if self.per_tensor else self.ext.Multi_QuantizeTensor_LC
        for table in self._tables:
            launch(table, self.max_n, self.quant_min, self.quant_max, self.rounding)
        return self.outputs
