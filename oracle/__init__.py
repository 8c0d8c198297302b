"""CPU oracle for the PPQ quantization-simulation hot path  --  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's `cpu_baseline` / `--impl reference` legs may import
this package.  The product (ppq_b200/) never imports it and fails loudly without its CUDA library.

Contents
  * ctypes bindings to oracle/_build/libppq_oracle.so (plain-C restatement, oracle/ppq_oracle.c):
    device-semantics fake-quant (INT + FP8), histograms, min/max, quantile, compute_mse_loss.
  * numpy / torch restatements of the host-side scale search that the reference runs in Python:
    ppq_numerical_round, ppq_round_to_power_of_2, minmax_to_scale_offset, the KL search
    (hist_to_scale_offset) and the MSE search.  The reference's arithmetic at that boundary *is* PyTorch
    CPU ops + Python doubles (SURVEY.md §8c), so these use the same primitives.
  * `torch_cpu_*`: the reference's USING_CUDA_KERNEL=False CPU path restated with torch CPU ops
    (qfunction/linear.py:27-32, observer/range.py:85-188) -- this is what bench.py times as the
    `cpu_baseline` / `--impl reference` arm ("kind": "port").

Pinning status (tests/test_oracle_pinning.py):
  INT fake-quant T/C, toInt, scalar rounding, minmax->scale/offset, minmax/kl/mse/percentile observers,
  KL search, KL divergence: pinned against tests/golden/ (generated from the real reference, CPU path).
  compute_mse_loss: pinned against the reference's own hist_mse.cc (oracle/_ref/hist_mse_ref.so + fixture).
  FP8 (QuantizeTensor_FT/_FC), Histogram_T/_Asymmetric_T/_C device semantics, Quantile_T:
  the reference has no CPU implementation and no test -> pinned on the GPU against the reference's own
  CUDA kernels compiled for sm_90a (oracle/_ref/PPQ_Cuda_Impls_ref.so, tests/test_gpu_vs_reference_cuda.py);
  fixtures produced there are committed under tests/golden/ref_cuda_*.npz once available.
"""
import ctypes
import math
import os
import subprocess
from decimal import ROUND_HALF_DOWN, ROUND_HALF_EVEN, ROUND_HALF_UP, Decimal

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, '_build', 'libppq_oracle.so')

RND_HALF_EVEN, RND_HALF_UP, RND_HALF_DOWN, RND_HALF_TOWARDS_ZERO = 0, 1, 2, 3
RND_HALF_FAR_FROM_ZERO, RND_TO_NEAR_INT, RND_UP, RND_DOWN = 4, 5, 6, 7


def host_threads() -> int:
    """CPU threads this process may really use: the scheduler affinity mask capped by the cgroup CPU quota.  os.cpu_count() reports
    the whole host (128 on some shared GPU hosts) even when a CPU quota limits the process to a few cores; running torch CPU ops with one thread
    per *host* core then oversubscribes the quota by an order of magnitude."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    for path in ('/sys/fs/cgroup/cpu.max', '/sys/fs/cgroup/cpu/cpu.cfs_quota_us'):
        try:
            txt = open(path).read().split()
            if path.endswith('cpu.max'):
                if txt[0] != 'max': n = min(n, max(1, int(float(txt[0]) / float(txt[1]) + 0.5)))
            else:
                q = int(txt[0]); per = int(open('/sys/fs/cgroup/cpu/cpu.cfs_period_us').read())
                if q > 0: n = min(n, max(1, int(q / per + 0.5)))
            break
        except Exception:
            continue
    return max(1, n)


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, 'ppq_oracle.c')
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', _HERE, '-s'] + (['-B'] if force else []))
    return _SO


_lib = None
_F, _I32, _I64, _P = ctypes.c_float, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_SO)
        L.ora_round2int.restype = ctypes.c_int32
        L.ora_round2int.argtypes = [_F, _I32]
        L.ora_linear_quant_t.argtypes = [_P, _P, _P, _I64, _F, _F, _I32, _I32, _I32]
        L.ora_linear_quant_c.argtypes = [_P, _P, _P, _I64, _I64, _I32, _P, _P, _I32, _I32, _I32]
        L.ora_linear_quant_t_torchpath.argtypes = [_P, _P, _P, _I64, _F, _F, _I32, _I32, _I32]
        L.ora_linear_quant_c_torchpath.argtypes = [_P, _P, _P, _I64, _I64, _I32, _P, _P, _I32, _I32, _I32]
        L.ora_float_quant_scalar.restype = _F
        L.ora_float_quant_scalar.argtypes = [_F, _F, _I32, _I32, _F, _F, _I32]
        L.ora_float_quant_t.argtypes = [_P, _P, _I64, _F, _F, _I32, _I32, _F, _F, _I32]
        L.ora_float_quant_c.argtypes = [_P, _P, _I64, _I64, _I32, _P, _P, _I32, _I32, _F, _F, _I32]
        L.ora_histogram_t.argtypes = [_P, _I64, _F, _I32, _P, _I64]
        L.ora_histogram_asym_t.argtypes = [_P, _I64, _F, _F, _I32, _P, _I64]
        L.ora_histogram_c.argtypes = [_P, _I64, _I64, _I32, _F, _I32, _P, _I64]
        L.ora_compute_mse_loss.restype = _F
        L.ora_compute_mse_loss.argtypes = [_P, _I64, _I32, _I32, _I32]
        L.ora_minmax_t.argtypes = [_P, _I64, _P, _P]
        L.ora_minmax_c.argtypes = [_P, _I64, _I64, _I32, _P, _P]
        L.ora_quantile_t.argtypes = [_P, _I64, _F, _P]
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def channel_geometry(shape, axis):
    """epc = product of the dims after `axis`; C = shape[axis] (floating.cu:118-122)."""
    axis = axis % len(shape) if len(shape) else 0
    epc = 1
    for d in shape[axis + 1:]:
        epc *= int(d)
    return epc, int(shape[axis])


# ---- device-semantics element-wise ops ------------------------------------------------------------
def round2int(v: float, mode: int) -> int:
    return int(lib().ora_round2int(float(np.float32(v)), int(mode)))


def linear_quant_t(x, scale, offset, qmin, qmax, mode=0, return_int=False):
    x = _f32(x); y = np.empty_like(x); q = np.empty(x.shape, np.int32)
    lib().ora_linear_quant_t(x.ctypes.data, y.ctypes.data, q.ctypes.data, x.size,
                             float(np.float32(scale)), float(np.float32(offset)), int(qmin), int(qmax), int(mode))
    return (y, q) if return_int else y


def linear_quant_c(x, scale, offset, axis, qmin, qmax, mode=0, return_int=False):
    x = _f32(x); y = np.empty_like(x); q = np.empty(x.shape, np.int32)
    s = _f32(scale).reshape(-1); o = _f32(offset).reshape(-1)
    epc, C = channel_geometry(x.shape, axis)
    assert s.size == C and o.size == C
    lib().ora_linear_quant_c(x.ctypes.data, y.ctypes.data, q.ctypes.data, x.size, epc, C,
                             s.ctypes.data, o.ctypes.data, int(qmin), int(qmax), int(mode))
    return (y, q) if return_int else y


def linear_quant_t_torchpath(x, scale, offset, qmin, qmax, mode=0, return_int=False):
    x = _f32(x); y = np.empty_like(x); q = np.empty_like(x)
    lib().ora_linear_quant_t_torchpath(x.ctypes.data, y.ctypes.data, q.ctypes.data, x.size,
                                       float(np.float32(scale)), float(np.float32(offset)), int(qmin), int(qmax), int(mode))
    return (y, q) if return_int else y


def linear_quant_c_torchpath(x, scale, offset, axis, qmin, qmax, mode=0, return_int=False):
    x = _f32(x); y = np.empty_like(x); q = np.empty_like(x)
    s = _f32(scale).reshape(-1); o = _f32(offset).reshape(-1)
    epc, C = channel_geometry(x.shape, axis)
    lib().ora_linear_quant_c_torchpath(x.ctypes.data, y.ctypes.data, q.ctypes.data, x.size, epc, C,
                                       s.ctypes.data, o.ctypes.data, int(qmin), int(qmax), int(mode))
    return (y, q) if return_int else y


def float_quant_scalar(x, s=1.0, E=4, M=3, cmin=-448.0, cmax=448.0, mode=0):
    return float(lib().ora_float_quant_scalar(float(np.float32(x)), float(np.float32(s)), E, M, cmin, cmax, mode))


def float_quant_t(x, scale, offset=0.0, E=4, M=3, cmin=-448.0, cmax=448.0, mode=0):
    x = _f32(x); y = np.empty_like(x)
    lib().ora_float_quant_t(x.ctypes.data, y.ctypes.data, x.size, float(np.float32(scale)), float(np.float32(offset)),
                            E, M, float(cmin), float(cmax), int(mode))
    return y


def float_quant_c(x, scale, offset, axis, E=4, M=3, cmin=-448.0, cmax=448.0, mode=0):
    x = _f32(x); y = np.empty_like(x)
    s = _f32(scale).reshape(-1); o = _f32(offset).reshape(-1)
    epc, C = channel_geometry(x.shape, axis)
    lib().ora_float_quant_c(x.ctypes.data, y.ctypes.data, x.size, epc, C, s.ctypes.data, o.ctypes.data,
                            E, M, float(cmin), float(cmax), int(mode))
    return y


# ---- collectors ------------------------------------------------------------------------------------
def histogram_t(x, hist_scale, bins=None, clip_outliers=True, hist=None):
    x = _f32(x)
    if hist is None: hist = np.zeros(bins, np.int32)
    lib().ora_histogram_t(x.ctypes.data, x.size, float(np.float32(hist_scale)), int(clip_outliers), hist.ctypes.data, hist.size)
    return hist


def histogram_asym_t(x, vmin, vmax, bins=None, clip_outliers=True, hist=None):
    x = _f32(x)
    if hist is None: hist = np.zeros(bins, np.int32)
    lib().ora_histogram_asym_t(x.ctypes.data, x.size, float(np.float32(vmin)), float(np.float32(vmax)),
                               int(clip_outliers), hist.ctypes.data, hist.size)
    return hist


def histogram_c(x, axis, hist_scale, bins=None, clip_outliers=True, hist=None):
    x = _f32(x)
    epc, C = channel_geometry(x.shape, axis)
    if hist is None: hist = np.zeros((C, bins), np.int32)
    lib().ora_histogram_c(x.ctypes.data, x.size, epc, C, float(np.float32(hist_scale)), int(clip_outliers),
                          hist.ctypes.data, hist.size // C)
    return hist


def minmax_t(x):
    x = _f32(x); lo = np.zeros(1, np.float32); hi = np.zeros(1, np.float32)
    lib().ora_minmax_t(x.ctypes.data, x.size, lo.ctypes.data, hi.ctypes.data)
    return lo[0], hi[0]


def minmax_c(x, axis):
    x = _f32(x)
    epc, C = channel_geometry(x.shape, axis)
    lo = np.zeros(C, np.float32); hi = np.zeros(C, np.float32)
    lib().ora_minmax_c(x.ctypes.data, x.size, epc, C, lo.ctypes.data, hi.ctypes.data)
    return lo, hi


def quantile_t(x, q):
    x = _f32(x); out = np.zeros(2, np.float32)
    lib().ora_quantile_t(x.ctypes.data, x.size, float(np.float32(q)), out.ctypes.data)
    return out


def compute_mse_loss(hist, start, step, end):
    h = np.ascontiguousarray(hist, dtype=np.int64)
    return float(lib().ora_compute_mse_loss(h.ctypes.data, h.size, int(start), int(step), int(end)))


# ---- host scalar rounding: ppq/utils/round.py:51-95, 115-135 ---------------------------------------
def numerical_round(value: float, mode: int = RND_HALF_EVEN) -> int:
    """`Decimal(value).quantize(1, rounding)`; HALF_UP/HALF_DOWN are *signed* upstream (towards +inf / -inf on
    ties), TOWARDS_ZERO/FAR_FROM_ZERO alias them, TO_NEAR_INT is floor(v+.5)/ceil(v-.5), UP is ceil."""
    value = float(value)
    one = Decimal(1)
    if mode == RND_HALF_EVEN:
        return int(Decimal(value).quantize(one, rounding=ROUND_HALF_EVEN))
    if mode in (RND_HALF_UP, RND_HALF_FAR_FROM_ZERO):
        return int(Decimal(value).quantize(one, rounding=ROUND_HALF_UP if value > 0 else ROUND_HALF_DOWN))
    if mode in (RND_HALF_DOWN, RND_HALF_TOWARDS_ZERO):
        return int(Decimal(value).quantize(one, rounding=ROUND_HALF_DOWN if value > 0 else ROUND_HALF_UP))
    if mode == RND_TO_NEAR_INT:
        return math.floor(value + 0.5) if value > 0 else math.ceil(value - 0.5)
    if mode == RND_UP:
        return math.ceil(value)
    raise ValueError('Unexpected rounding policy found.')


def round_to_power_of_2(value: float, mode: int = RND_UP, ieee: bool = False) -> float:
    """ieee=True: NaN and +-inf, where the reference raises (math.ceil / Decimal of log2(nan) or log2(inf)), are returned unchanged -- what the
    device computes for them (DESIGN.md §2)."""
    if value == 0: return 0
    if ieee and not math.isfinite(value): return value
    sign = 1 if value >= 0 else -1
    return sign * float(pow(2, numerical_round(math.log2(sign * value), mode)))


# ---- minmax_to_scale_offset: ppq/quantization/observer/range.py:22-75 (Python doubles) -------------
def minmax_to_scale_offset(min_val, max_val, qmin, qmax, symmetrical, power_of_2=False, scale_threshold=1e-8, ieee=False):
    """ieee=True: where the reference raises -- int(nan) for the offset of a non-finite asymmetric range, the power-of-two of a NaN or inf
    scale -- return the IEEE result instead (offset NaN, scale unchanged), which is what the device computes."""
    min_val, max_val = float(min_val), float(max_val)
    if min_val > 0: min_val = 0.0
    if max_val < 0: max_val = 0.0
    if symmetrical:
        scale = 2 * float(max(abs(max_val), abs(min_val))) / (qmax - qmin)
        scale = max(scale, scale_threshold)
        offset = 0
    else:
        scale = float(max_val - min_val) / (qmax - qmin)
        scale = max(scale, scale_threshold)
        q = -min_val / scale
        offset = q if (ieee and not math.isfinite(q)) else numerical_round(q)
    if power_of_2:
        scale = round_to_power_of_2(scale, RND_UP, ieee)
    return scale, offset


# ---- KL search: TorchHistObserver.hist_to_scale_offset, range.py:190-282; measure/statistic.py:3-12 -
def kl_divergence(p, q, eps=1e-30):
    import torch
    p = torch.as_tensor(p).double(); q = torch.as_tensor(q).double()
    return torch.dot(p, torch.log10(p + eps) - torch.log10(q + eps)).item()


def kl_search(hist, hist_scale, num_of_bits=8, power_of_2=False, scale_threshold=1e-8, return_losses=False, ieee=False):
    """Candidate clip points bin_range = quant_bins, 2*quant_bins, ... (< bins + quant_bins - 1).  For each:
    P = first bin_range bins with the tail folded into the last one, / total;  Q = the same bins merged into
    quant_bins groups, each group's mass spread evenly over its non-empty bins, normalised;  loss = KL(P||Q) in
    fp64 log10.  First minimum wins.  fp32 tensors / torch CPU reductions exactly as upstream.  ieee: see minmax_to_scale_offset."""
    import torch
    h = torch.as_tensor(np.asarray(hist)).float().clone()
    bins = h.numel()
    quant_bins = 2 ** (num_of_bits - 1)
    dead = int(bins * .002)
    h[:dead] = 0
    h[dead] = 1
    total = torch.sum(h)
    best, best_loss, losses = None, None, []
    for bin_range in range(quant_bins, bins + quant_bins - 1, quant_bins):
        p = torch.zeros(bin_range, dtype=torch.float)
        p[:bin_range].copy_(h[:bin_range])
        p[bin_range - 1] += torch.sum(h[bin_range:])
        p = p / total
        ratio = int(bin_range / quant_bins)
        g = h[:bin_range].clone().reshape((quant_bins, ratio))
        alive = g > 0
        cnt = alive.sum(axis=1, keepdim=True)
        cnt[cnt == 0] = 1
        qd = torch.div(g.sum(axis=1, keepdim=True), cnt).repeat([1, ratio]) * alive
        qd = (qd / torch.sum(qd)).flatten()
        loss = kl_divergence(p, qd)
        losses.append(loss)
        if best is None or loss < best_loss:
            best, best_loss = bin_range, loss
    scale = kl_scale(best, bins, hist_scale, num_of_bits, power_of_2, scale_threshold, ieee)
    if return_losses:
        return scale, 0, best, losses
    return scale, 0


def kl_scale(best, bins, hist_scale, num_of_bits=8, power_of_2=False, scale_threshold=1e-8, ieee=False):
    """The scale of the winning bin range (range.py:271-282): clamp to the minimum scale, power-of-two with the exponent rounded half-up."""
    quant_bins = 2 ** (num_of_bits - 1)
    scale = (best / bins) * hist_scale * (bins / quant_bins)
    scale = max(scale, scale_threshold)
    if power_of_2:
        scale = round_to_power_of_2(scale, RND_HALF_UP, ieee)
    return scale


# ---- MSE search: TorchMSEObserver.hist_to_scale_offset, range.py:456-520 ---------------------------
def mse_search(hist, hist_scale, vmin, qmin, qmax, symmetrical, power_of_2=False, interval=8, loss_fn=None, scale_threshold=1e-8,
               ieee=False):
    """loss_fn defaults to the C++ compute_mse_loss restatement (fp32 accumulate; what CUDA.compute_mse_loss is).
    Pass `mse_loss_python_twin` to follow the USING_CUDA_KERNEL=False branch (Python doubles, range.py:431-454).
    scale_threshold: OBSERVER_MIN_SCALE_MANUL_OVERRIDE, handed to minmax_to_scale_offset; ieee: see there."""
    loss_fn = loss_fn or compute_mse_loss
    hist = [int(v) for v in np.asarray(hist).tolist()]
    bins = len(hist)
    levels = (qmax - qmin) + 1
    cands = []
    step = bins // levels + 1
    cands.append((loss_fn(hist, 0, step, levels * step), 0, levels * step))
    if not symmetrical:
        for start in range(0, bins, interval):
            if (start * hist_scale) + vmin > 0: break
            for step in range(1, bins // levels + 1):
                end = start + levels * step
                if end > (bins + levels): break
                cands.append((loss_fn(hist, start, step, end), start, end))
    else:
        for step in range(1, bins // levels + 1):
            end = levels * step
            if end > (bins + levels): break
            cands.append((loss_fn(hist, 0, step, end), 0, end))
    best = min(cands, key=lambda c: c[0])      # python's min/sorted are stable: first minimum wins
    _, s0, e0 = best
    if symmetrical:
        lo, hi = -(e0 * hist_scale), (e0 * hist_scale)
    else:
        lo, hi = (s0 * hist_scale) + vmin, (e0 * hist_scale) + vmin
    return minmax_to_scale_offset(lo, hi, qmin, qmax, symmetrical, power_of_2, scale_threshold, ieee)


def mse_loss_python_twin(hist, start, step, end):
    total = sum(hist)
    loss = 0
    for idx, b in enumerate(hist):
        if idx < start: err = (start - idx - 1) + 0.5
        elif idx > end: err = (idx - end) + 0.5
        else:
            l = (idx - start) % step
            r = step - l - 1
            err = (l + 0.25) if l == r else min(l + 0.5, r + 0.5)
        loss += (b * err * err) / total
    return loss


# ---- the reference's CPU path restated with torch CPU ops (cpu_baseline / --impl reference arm) ---
def torch_cpu_round(t, mode=0):
    import torch
    if mode == RND_HALF_EVEN: return t.round()
    if mode == RND_UP: return t.ceil()
    if mode == RND_HALF_TOWARDS_ZERO: return torch.sign(t) * torch.ceil(t.abs() - 0.5)
    if mode == RND_HALF_FAR_FROM_ZERO: return torch.sign(t) * torch.floor(t.abs() + 0.5)
    if mode == RND_HALF_DOWN: return torch.ceil(t - 0.5)
    if mode == RND_HALF_UP: return torch.floor(t + 0.5)
    raise NotImplementedError


def torch_cpu_linear_quant_t(x, scale, offset, qmin, qmax, mode=0):
    """qfunction/linear.py:27-32: six out-of-place fp32 tensor ops."""
    import torch
    q = torch.clamp(torch_cpu_round(x / scale, mode) + offset, qmin, qmax)
    return (q - offset) * scale


def torch_cpu_linear_quant_c(x, scale, offset, axis, qmin, qmax, mode=0):
    """qfunction/linear.py:73-81."""
    import torch
    shape = [1 if a != axis else -1 for a in range(x.ndim)]
    s, o = scale.view(shape), offset.view(shape)
    q = torch.clamp(torch_cpu_round(x / s, mode) + o, qmin, qmax)
    return (q - o) * s


def torch_cpu_minmax(x):
    """observer/range.py:91-92: two separate reductions."""
    return x.min(), x.max()


def torch_cpu_hist_sym(x, hist_scale, bins):
    """observer/range.py:183 (CPU branch): torch.histc(abs(x), bins, 0, hist_scale*bins).int().
    NOTE: histc bins `x == max` into the last bin and uses a different edge formula than the CUDA kernel;
    the reference's own test tolerates < 100 counts between the two (tests/test_cuda_kernel.py:197-208)."""
    import torch
    return torch.histc(torch.abs(x), bins, min=0, max=hist_scale * bins).int()
