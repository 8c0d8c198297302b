"""Oracle for the layerwise error analysis -- test infrastructure, imported by tests/ and tools/bench_layerwise.py.

  exact_moments(p, r)        {sum (p - r)^2, sum r^2, sum p^2, sum p r} per row in exact arithmetic, rounded once to fp64 (math.fsum over
                             an exact expansion of every term; beyond 2^20 elements, of 2^20-element partials); rows with a NaN or an infinity follow IEEE fp64: the plain sum of the
                             fp64 terms, which is NaN when a term is NaN or +inf meets -inf and +-inf otherwise, whatever the order.
  abs_moments(p, r)          the same sums over |term|: the scale of the error bound (k + 1) 2^-53 sum |terms|.
  torch_snr_error / torch_mean_square_error / torch_cosine_similarity
                             the reference's measures (ppq/quantization/measure/norm.py:3-99, cosine.py:6-28) restated from their
                             semantics: per-sample sums of out-of-place fp32 (or the input's) tensor ops, then the mean over samples.
  MeasureRecorder            analyse/util/__init__.py:8-47 with reduce='mean': `.item()` per update, running mean in Python doubles.
  reference_layerwise(...)   layerwise.py:73-134 restated on ppq_b200's executor: operation-outer, an fp32 and a single-operation forward
                             per operation and batch, the torch measures above, one `.item()` per update.
"""
import math

import numpy as np
import torch

SPLIT = 134217729.0                  # 2^27 + 1 (Veltkamp split of a double into two 26-bit halves)
CHUNK = 1 << 20                      # rows longer than this are summed as correctly rounded 2^20-element partials: within 2^-52 sum |terms|


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _two_prod(a, b):
    x = a * b
    ca, cb = SPLIT * a, SPLIT * b
    ah, bh = ca - (ca - a), cb - (cb - b)
    al, bl = a - ah, b - bh
    return x, al * bl - (((x - ah * bh) - al * bh) - ah * bl)


def _as_f64_rows(x, rows):
    x = np.asarray(x)
    if x.dtype != np.float32: x = np.asarray(torch.as_tensor(x).float().numpy())
    return x.astype(np.float64).reshape(rows, -1)


def _rows(x):
    x = np.asarray(x) if not isinstance(x, torch.Tensor) else x
    return 1 if x.ndim == 1 else int(x.shape[0])


def _f32(t):
    """fp32 numpy view of a tensor / array (fp16 and bf16 upcast exactly)."""
    if isinstance(t, torch.Tensor): return t.detach().cpu().float().numpy()
    return np.asarray(t, dtype=np.float32)


def exact_moments(p, r) -> np.ndarray:
    """[rows, 4] fp64."""
    rows = _rows(p)
    P, R = _as_f64_rows(_f32(p), rows), _as_f64_rows(_f32(r), rows)
    out = np.zeros((rows, 4))
    for i in range(rows):
        a, b = P[i], R[i]
        if not (np.isfinite(a).all() and np.isfinite(b).all()):
            with np.errstate(invalid='ignore', over='ignore'):
                d = a - b
                out[i] = [np.sum(d * d), np.sum(b * b), np.sum(a * a), np.sum(a * b)]
            continue
        parts = [[], [], [], []]
        for c in range(0, max(a.size, 1), CHUNK):
            ac, bc = a[c:c + CHUNK], b[c:c + CHUNK]
            h, lo = _two_sum(ac, -bc)                                      # p - r = h + lo exactly
            terms = [*_two_prod(h, h), *_two_prod(2.0 * h, lo), *_two_prod(lo, lo)]
            parts[0].append(math.fsum(np.concatenate(terms)))
            parts[1].append(math.fsum(bc * bc))                            # products of fp32 values are exact in fp64
            parts[2].append(math.fsum(ac * ac))
            parts[3].append(math.fsum(ac * bc))
        out[i] = [math.fsum(q) for q in parts]
    return out


def abs_moments(p, r) -> np.ndarray:
    rows = _rows(p)
    P, R = _as_f64_rows(_f32(p), rows), _as_f64_rows(_f32(r), rows)
    with np.errstate(invalid='ignore', over='ignore'):
        return np.stack([((P - R) ** 2).sum(1), (R * R).sum(1), (P * P).sum(1), np.abs(P * R).sum(1)], axis=1)


def chain_length(row_len: int) -> int:
    """The longest addition chain of a Multi_Paired_Moments launch for a row of `row_len` elements (include/ppq_b200.h)."""
    return 74 + -(-row_len // 16384)


def moments_bound(p, r, row_len=None) -> np.ndarray:
    """|got - exact| allowed per row and moment: (k + 1) 2^-53 sum |terms|, with two more roundings per term for sum (p - r)^2 (the fp64
    difference p - r and its square)."""
    n = row_len if row_len is not None else int(np.asarray(_f32(p)).size // max(_rows(p), 1))
    k = chain_length(n) + (2 if n > CHUNK else 0)                          # the oracle's own partials beyond 2^20 elements
    a = abs_moments(p, r)
    return a * np.array([k + 3, k + 1, k + 1, k + 1]) * 2.0 ** -53


def moments_agree(got, want, bound) -> bool:
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    same_special = (np.isnan(got) & np.isnan(want)) | (np.isinf(want) & (got == want))
    finite = np.isfinite(want)
    with np.errstate(invalid='ignore'):
        close = finite & (np.abs(got - want) <= bound)
    return bool((same_special | close).all())


# ---------------------------------------------------------------- the reference's measures, restated
def _flat(y_pred, y_real):
    if y_pred.shape != y_real.shape: raise ValueError('shapes differ')
    if y_pred.ndim == 1: y_pred, y_real = y_pred.unsqueeze(0), y_real.unsqueeze(0)
    return y_pred.flatten(start_dim=1), y_real.flatten(start_dim=1)


def torch_snr_error(y_pred, y_real):
    p, r = _flat(y_pred, y_real)
    noise = torch.pow(p - r, 2).sum(dim=-1)
    signal = torch.pow(r, 2).sum(dim=-1)
    return torch.mean(noise / (signal + 1e-7))


def torch_mean_square_error(y_pred, y_real):
    p, r = _flat(y_pred, y_real)
    return torch.mean(torch.mean(torch.pow(p - r, 2), dim=-1))


def torch_cosine_similarity(y_pred, y_real):
    p, r = _flat(y_pred, y_real)
    return torch.mean(torch.cosine_similarity(p.float(), r.float(), dim=-1))


MEASURE_FNS = {'snr': torch_snr_error, 'mse': torch_mean_square_error, 'cosine': torch_cosine_similarity}


class MeasureRecorder:
    def __init__(self, method):
        self.fn, self.n, self.measure, self.updates = MEASURE_FNS[method], 0, 0, 0

    def update(self, y_pred, y_real):
        elements = y_pred.shape[0]
        result = self.fn(y_pred, y_real).item()
        self.measure = self.measure * self.n + result * elements
        self.n += elements
        self.measure /= self.n
        self.updates += 1


def outputs_of(executor, x, interested_outputs):
    """The interested outputs of one forward, as layerwise_error_analyse collects them."""
    if interested_outputs is None:
        out = executor.forward(x)
        return list(out) if isinstance(out, (tuple, list)) else [out]
    store = {}

    class Tap:
        def __init__(self, n): self.n = n
        def pre_forward_hook(self, **kw): pass
        def post_forward_hook(self, outputs, quant_outputs, quant_configs): store[self.n] = quant_outputs[0].clone()
    executor.forward(x, hooks={n: Tap(n) for n in interested_outputs})
    return [store[n] for n in interested_outputs]


@torch.no_grad()
def reference_layerwise(executor, batches, interested_outputs=None, method='snr', steps=8):
    """layerwise.py:73-134 on our executor: for each computing operation, for each batch: fp32 forward, that operation quantised, forward,
    one recorder update per output; `if idx >= steps: break` after the updates."""
    from ppq_b200.executor import COMPUTING_OP
    if isinstance(interested_outputs, str): interested_outputs = [interested_outputs]
    names = [n for n, op in executor.quantable_operations() if op.kind in COMPUTING_OP]
    recorders = {n: MeasureRecorder(method) for n in names}
    executor.dequantize()
    try:
        for n in names:
            for idx, x in enumerate(batches):
                fp = outputs_of(executor, x, interested_outputs)
                executor.quantize_only(n)
                qt = outputs_of(executor, x, interested_outputs)
                for f, q in zip(fp, qt): recorders[n].update(y_pred=q, y_real=f)
                executor.quantize_only(None)
                if idx >= steps: break
    finally:
        if executor._dequantized is not None: executor.quantize_only(None)
        executor.restore_quantize_state()
    return {n: recorders[n].measure for n in names}
