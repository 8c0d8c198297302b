"""Quantisation-error measures on the device: the sums behind ppq/quantization/measure/norm.py:3-99 and measure/cosine.py:6-28, for a table of
(prediction, reference) tensor pairs in one kernel launch (Multi_Paired_Moments), reduced in fp64 with a fixed summation order.

    paired_moments(preds, reals)    [rows, 4] fp64 = {sum (p - r)^2, sum r^2, sum p^2, sum p r} per sample row, pairs one after the other
    measure_rows(moments, ...)      the reference's per-sample snr / mse / cosine from those sums, in fp64

A sample row is the outermost dimension of a tensor, or the whole tensor when it is 1-d (norm.py:36-38).  fp16 / bf16 pairs are measured on
their exact upcasts.
"""
from typing import List, Sequence, Tuple

import torch

from .calibration import TABLE_DTYPES, is_dense, shared_stager

MEASURES = ('snr', 'mse', 'cosine')
COSINE_EPS = 1e-8                    # torch.cosine_similarity's default: each norm is clamped to it before the division


def rows_of(t: torch.Tensor) -> Tuple[int, int]:
    """(rows, row_len) of a tensor measured sample by sample."""
    if t.dim() == 0: raise ValueError('paired_moments: a 0-d tensor has no sample dimension')
    rows = 1 if t.dim() == 1 else int(t.shape[0])
    return rows, (t.numel() // rows if rows else 0)


def _sample_blocks(p: torch.Tensor, r: torch.Tensor):
    """p and r with every sample one contiguous block, the elements of a sample in the same storage order in both (a contiguous or
    channels_last pair is read as it is; anything else is made contiguous)."""
    def ok(t):
        return is_dense(t) and (t.dim() <= 1 or t.shape[0] <= 1 or t.stride(0) == t.numel() // t.shape[0])
    if ok(p) and ok(r) and p.stride() == r.stride(): return p, r
    return p.contiguous(), r.contiguous()


def paired_moments(preds: Sequence[torch.Tensor], reals: Sequence[torch.Tensor], out: torch.Tensor = None) -> torch.Tensor:
    """One Multi_Paired_Moments launch per element type present (pairs of one dtype each); rows are numbered pair after pair in the given
    order.  Nothing is synchronised."""
    from .ffi import extension
    if len(preds) != len(reals): raise ValueError('paired_moments: as many predictions as references are needed')
    pairs, total_rows = [], 0
    for p, r in zip(preds, reals):
        if p.shape != r.shape: raise ValueError(f'paired_moments: shapes differ ({tuple(p.shape)} and {tuple(r.shape)})')
        if p.dtype != r.dtype or p.dtype not in TABLE_DTYPES: raise TypeError(f'paired_moments: pairs of one fp32 / fp16 / bf16 dtype, got {p.dtype} and {r.dtype}')
        if p.device != r.device or p.device.type != 'cuda': raise ValueError('paired_moments: both tensors of a pair on one CUDA device')
        p, r = _sample_blocks(p, r)
        rows, row_len = rows_of(p)
        pairs.append((p, r, rows, row_len, total_rows))
        total_rows += rows
    if not pairs: return torch.zeros(0, 4, dtype=torch.float64) if out is None else out
    dev = pairs[0][0].device
    if out is None: out = torch.empty(total_rows, 4, dtype=torch.float64, device=dev)
    if out.shape != (total_rows, 4): raise ValueError(f'paired_moments: out must be [{total_rows}, 4]')
    ext = extension()
    groups = {}
    for p, r, rows, row_len, row0 in pairs:
        groups.setdefault(p.dtype, []).append((p, r, rows, row_len, row0))
    stager = shared_stager(dev, 5)
    for dtype, group in groups.items():
        elems = sum(rows * row_len for _, _, rows, row_len, _ in group)
        ws = torch.empty(ext.Multi_Paired_Moments_Workspace_Bytes(total_rows, elems), dtype=torch.uint8, device=dev)
        descs = stager.get(tuple((p.data_ptr(), r.data_ptr(), rows, row_len, row0) for p, r, rows, row_len, row0 in group))
        ext.Multi_Paired_Moments(descs, elems, dtype, out, ws)
    return out


def measure_rows(moments: torch.Tensor, row_len, method: str) -> torch.Tensor:
    """Per-sample measure (fp64) from paired moments: snr = sum (p - r)^2 / (sum r^2 + 1e-7) (norm.py:52-93), mse = sum (p - r)^2 / D
    (norm.py:3-50), cosine = sum p r / (max(|p|, eps) max(|r|, eps)) with torch.cosine_similarity's eps = 1e-8 (cosine.py:6-28).
    row_len: the element count D of every row (a number, or a tensor of one per row)."""
    d2, r2, p2, pr = moments.unbind(1)
    if method == 'snr': return d2 / (r2 + 1e-7)
    if method == 'mse': return d2 / row_len
    if method == 'cosine': return pr / (p2.sqrt().clamp_min(COSINE_EPS) * r2.sqrt().clamp_min(COSINE_EPS))
    raise ValueError(f"Unsupported measurement {method!r}: 'snr', 'mse' and 'cosine' are supported")


def batch_measures(preds: List[torch.Tensor], reals: List[torch.Tensor], method: str, out: torch.Tensor = None) -> torch.Tensor:
    """The reference's per-update value of every pair -- the mean over its samples of the per-sample measure (reduction='mean') -- as one fp64
    tensor [len(preds)] on the device, from one paired-moment launch.  `out` (optional) receives it."""
    m = paired_moments(preds, reals)
    shapes = [rows_of(p) for p in preds]
    if len({s for s in shapes}) == 1:                                   # every pair has the same rows and row length: one reshape
        rows, row_len = shapes[0]
        vals = measure_rows(m, row_len, method).view(len(preds), rows).mean(dim=1)
    else:
        vals, row0 = [], 0
        for rows, row_len in shapes:
            vals.append(measure_rows(m[row0:row0 + rows], row_len, method).mean())
            row0 += rows
        vals = torch.stack(vals)
    if out is not None:
        out.copy_(vals)
        return out
    return vals
