#!/usr/bin/env python
"""Ours vs the reference's own CUDA kernels (oracle/_ref/PPQ_Cuda_Impls_ref.so: ppq/csrc compiled unmodified for sm_90a) on the same GPU,
same tensors, CUDA events, rotating buffers > L2.  A measurement tool (not part of bench.py): output is kept in profiles/."""
import importlib.util
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ppq_b200.ffi import extension  # noqa: E402

PEAK = float(json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs']) if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else 6650.0


def load_ref():
    so = os.path.join(ROOT, 'oracle', '_ref', 'PPQ_Cuda_Impls_ref.so')
    spec = importlib.util.spec_from_file_location('PPQ_Cuda_Impls_ref', so)
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    return m


def timeit(fn, reps, nbuf):
    for i in range(min(nbuf, 2)): fn(i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    for i in range(reps): fn(i % nbuf)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def main():
    ours, ref = extension(), load_ref()
    dev = torch.device('cuda')
    n, nbuf = 32 * 12 * 512 * 512 // 2, 6
    xs = [torch.randn(n, device=dev) for _ in range(nbuf)]
    xr = [torch.relu(x) for x in xs]
    s, o = torch.tensor([0.05], device=dev), torch.tensor([0.0], device=dev)
    rows = []

    def row(name, bpe, f_ours, f_ref, reps=10, ref_reps=None):
        to = timeit(f_ours, reps, nbuf); tr = timeit(f_ref, ref_reps or reps, nbuf)
        go, gr = bpe * n / to / 1e9, bpe * n / tr / 1e9
        rows.append((name, to * 1e6, go, go / PEAK, tr * 1e6, gr, gr / PEAK, tr / to))
        print(f'{name:44s} ours {to*1e6:9.1f} us {go:8.1f} GB/s {go/PEAK:6.1%} | reference {tr*1e6:10.1f} us {gr:8.1f} GB/s {gr/PEAK:6.1%} | x{tr/to:7.1f}', flush=True)

    row('QuantizeTensor_LT INT8 (50.3M elem)', 8, lambda i: ours.QuantizeTensor_LT(xs[i], s, o, -128, 127, 0), lambda i: ref.QuantizeTensor_LT(xs[i], s, o, -128, 127, 0))
    C = 768
    v = [x[:(n // 4608) * 4608].view(-1, 4608) for x in xs]
    sc = torch.rand(v[0].shape[0], device=dev) * 0.1 + 0.01; oc = torch.zeros_like(sc)
    row('QuantizeTensor_LC axis 0, epc 4608', 8, lambda i: ours.QuantizeTensor_LC(v[i], sc, oc, -128, 127, 0, 0), lambda i: ref.QuantizeTensor_LC(v[i], sc, oc, -128, 127, 0, 0))
    one = torch.ones(1, device=dev)
    row('QuantizeTensor_FT E4M3', 8, lambda i: ours.QuantizeTensor_FT(xs[i], one, o, 4, 3, -448.0, 448.0, 0), lambda i: ref.QuantizeTensor_FT(xs[i], one, o, 4, 3, -448.0, 448.0, 0))
    h = torch.zeros(4096, dtype=torch.int32, device=dev)
    hs = float(xs[0].abs().max().item()) / 4096
    row('Histogram_T 4096 bins, randn', 4, lambda i: ours.Histogram_T(xs[i], hs, True, h), lambda i: ref.Histogram_T(xs[i], hs, True, h), ref_reps=3)
    row('Histogram_T 4096 bins, relu(randn)', 4, lambda i: ours.Histogram_T(xr[i], hs, True, h), lambda i: ref.Histogram_T(xr[i], hs, True, h), ref_reps=2)
    row('Quantile_T q=0.9999', 4, lambda i: ours.Quantile_T(xs[i], 0.9999), lambda i: ref.Quantile_T(xs[i], 0.9999), reps=5, ref_reps=3)
    mm = torch.empty(2, device=dev); ours.MinMax_Init(mm[0:1], mm[1:2])
    row('min+max (ours fused / torch .min() + .max())', 4, lambda i: ours.MinMax_T(xs[i], mm), lambda i: (xs[i].min(), xs[i].max()))
    # the small tensors of BASELINE config 1: latency
    small = [torch.randn(1, 512, 28, 28, device=dev) for _ in range(64)]
    to = timeit(lambda i: ours.QuantizeTensor_LT(small[i], s, o, -128, 127, 0), 200, 64); tr = timeit(lambda i: ref.QuantizeTensor_LT(small[i], s, o, -128, 127, 0), 200, 64)
    print(f'QuantizeTensor_LT 1x512x28x28 latency: ours {to*1e6:.2f} us, reference {tr*1e6:.2f} us')
    out = os.path.join(ROOT, 'gpurun_out', 'vs_reference_kernels.md')
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, 'w') as f:
        f.write(f'# ours vs the reference\'s own CUDA kernels (compiled for sm_90a) on the same GPU -- {torch.cuda.get_device_name(0)}\n\n')
        f.write(f'50.3 M fp32 elements per call, {nbuf} rotating buffers (1.2 GB), CUDA events; peak = {PEAK:.0f} GB/s (measured copy).\n\n')
        f.write('| op | ours us | ours GB/s | ours % peak | reference us | reference GB/s | reference % peak | speed-up |\n|---|---|---|---|---|---|---|---|\n')
        for r in rows: f.write(f'| {r[0]} | {r[1]:.1f} | {r[2]:.0f} | {r[3]:.1%} | {r[4]:.1f} | {r[5]:.0f} | {r[6]:.1%} | {r[7]:.1f}x |\n')
        f.write(f'\nQuantizeTensor_LT 1x512x28x28 (BASELINE config 1, launch-latency bound): ours {to*1e6:.2f} us, reference {tr*1e6:.2f} us per call.\n')


if __name__ == '__main__':
    main()
