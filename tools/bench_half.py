#!/usr/bin/env python
"""Rates of the single-tensor kernels on fp32, bf16 and fp16 inputs of the same element count, alternated in one process.

    python tools/bench_half.py [--mi 64] [--reps 9] [--launches 20]

Each dtype cycles through 4 buffers of `--mi` Mi elements (beyond the 50 MB L2).  A sample is `--launches` back-to-back launches between one
pair of CUDA events (so the host's dispatch overlaps the previous kernel), divided by their number; per kernel and dtype the script prints one
JSON line with the median of `--reps` samples, taken with the dtypes alternating sample by sample, and the rate at the algorithmic bytes:
elements x element size read, plus the same written for the fake-quant kernel, with its share of the read (or copy) ceiling that
tools/hbm_ceiling.py measures in the same run.  The first line names the card, its power limit and the SM clocks sampled during the run.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mi', type=int, default=64)
    ap.add_argument('--reps', type=int, default=9)
    ap.add_argument('--launches', type=int, default=20)
    args = ap.parse_args()
    here = os.path.dirname(os.path.abspath(__file__))
    probe = subprocess.run([sys.executable, os.path.join(here, 'hbm_ceiling.py')], check=True, capture_output=True, text=True).stdout
    ceiling = [json.loads(line) for line in probe.splitlines() if line.startswith('{') and '"summary"' in line][-1]
    from ppq_b200.ffi import extension
    ext = extension()
    import pynvml
    pynvml.nvmlInit()
    index = torch.cuda.current_device()
    vis = [v.strip() for v in os.environ.get('CUDA_VISIBLE_DEVICES', '').split(',') if v.strip()]
    if index < len(vis) and vis[index].isdigit(): index = int(vis[index])       # NVML counts physical devices
    h = pynvml.nvmlDeviceGetHandleByIndex(index)
    name = pynvml.nvmlDeviceGetName(h)
    clocks, stop = [], threading.Event()

    def sample():
        while not stop.is_set():
            clocks.append(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
            time.sleep(0.05)

    n = args.mi << 20
    g = torch.Generator(device='cuda').manual_seed(0)
    dtypes = [torch.float32, torch.bfloat16, torch.float16]
    bufs = {dt: [torch.randn(n, device='cuda', generator=g).to(dt) for _ in range(4)] for dt in dtypes}
    relu = {dt: [torch.clamp(b, min=0) for b in bufs[dt]] for dt in dtypes}
    s, o = torch.tensor([0.05], device='cuda'), torch.zeros(1, device='cuda')
    mm = torch.empty(2, device='cuda')
    hist = torch.zeros(4096, dtype=torch.int32, device='cuda')
    hs = torch.tensor([4.0 / 4096], device='cuda')
    guess = ext.Quantile_Guess_Init(1, s)

    def lt(x):
        return ext.QuantizeTensor_LT(x, s, o, -128, 127, 0) if x.dtype == torch.float32 else ext.QuantizeTensor_LT_Half(x, s, o, -128, 127, 0)

    kernels = {
        'linear_quant_t': (lambda x, i: lt(x), 2),
        'minmax_t': (lambda x, i: ext.MinMax_T(x, mm), 1),
        'histogram_t_dscale_relu': (lambda x, i: ext.Histogram_T_DeviceScale(relu[x.dtype][i], hs, True, hist), 1),
        'quantile_t_guess': (lambda x, i: ext.Quantile_T_Guess(x, 0.9999, guess), 1),
    }
    th = threading.Thread(target=sample, daemon=True)
    th.start()
    results = {}
    try:
        for _ in range(2):                                              # warm-up round, then the measured round
            results.clear()
            for kname, (fn, passes) in kernels.items():
                for rep in range(args.reps):
                    for dt in dtypes:                                   # alternate the dtypes sample by sample
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        for k in range(args.launches): fn(bufs[dt][k % 4], k % 4)
                        b.record()
                        b.synchronize()
                        results.setdefault((kname, dt), []).append(a.elapsed_time(b) * 1e-3 / args.launches)
    finally:
        stop.set(); th.join()
    clocks.sort()
    print(json.dumps({'card': name.decode() if isinstance(name, bytes) else name,
                      'power_limit_w': pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                      'sm_mhz_sampled': {'min': clocks[0], 'median': clocks[len(clocks) // 2], 'max': clocks[-1]} if clocks else None,
                      'elements': n, 'read_ceiling_gbs': ceiling['read_ceiling_gbs'], 'copy_ceiling_gbs': ceiling['copy_ceiling_gbs']}), flush=True)
    for (kname, dt), ts in results.items():
        ts.sort()
        t = ts[len(ts) // 2]
        esz = torch.tensor([], dtype=dt).element_size()
        gbs = n * esz * kernels[kname][1] / t / 1e9
        roof = ceiling['copy_ceiling_gbs'] if kernels[kname][1] == 2 else ceiling['read_ceiling_gbs']
        print(json.dumps({'kernel': kname, 'dtype': str(dt).replace('torch.', ''), 'median_ms': round(t * 1e3, 4), 'gbs': round(gbs, 1),
                          'share_of_ceiling': round(gbs / roof, 3), 'gelem_s': round(n / t / 1e9, 2)}), flush=True)


if __name__ == '__main__':
    sys.exit(main())
