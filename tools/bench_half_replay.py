#!/usr/bin/env python
"""The ResNet-50 calibration replay of bench.py on fp32 and on bf16 copies of the same tensors, alternated in one process.

    python tools/bench_half_replay.py [--batch 32] [--rotate 3] [--batches 4] [--reps 7] [--launches 6]

The activation and weight shapes are bench.resnet50_tensor_table(); every bf16 tensor is the cast of its fp32 twin.  Per kernel -- the
multi-tensor min/max (phase 1), the multi-tensor 4096-bin histogram (phase 2) and the per-channel INT8 weight table -- a sample is
`--launches` back-to-back launches between one pair of CUDA events, each over the next of `--rotate` activation sets (every set is far
beyond the 50 MB L2, so every pass reads HBM), divided by their number; fp32 and bf16 alternate sample by sample and the median of `--reps`
samples is reported with the rate at the algorithmic bytes (elements x element size read; the weight table also writes them) and its share
of the read (or copy) ceiling tools/hbm_ceiling.py measures in the same run.  A step is one replayed calibration of `--batches` batches:
phase 1 (weight table + min/max per batch, exchange, hist scales), phase 2 (weight table + histogram per batch, exchange, KL search); its
time is reported for both dtypes, alternated the same way.  The first line names the card, its power limit and the SM clocks sampled
during the run.  There is no CPU path: without a GPU the script fails.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--rotate', type=int, default=3)
    ap.add_argument('--batches', type=int, default=4, help='calibration batches per phase of a step')
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--launches', type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available(): raise SystemExit('bench_half_replay.py measures on a GPU; none is visible')
    here = os.path.dirname(os.path.abspath(__file__))
    probe = subprocess.run([sys.executable, os.path.join(here, 'hbm_ceiling.py')], check=True, capture_output=True, text=True).stdout
    ceiling = [json.loads(line) for line in probe.splitlines() if line.startswith('{') and '"summary"' in line][-1]
    import bench
    from ppq_b200.calibration import ArenaCalibrator, MultiWeightQuantizer
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

    wl = bench.Workload(torch.device('cuda'), 'resnet50', args.batch, args.rotate, seed=1234)
    dtypes = [torch.float32, torch.bfloat16]
    sets = {torch.float32: wl.sets, torch.bfloat16: [[t.to(torch.bfloat16) for t in ts] for ts in wl.sets]}
    weights = {torch.float32: wl.w, torch.bfloat16: [w.to(torch.bfloat16) for w in wl.w]}
    cal = {dt: ArenaCalibrator(len(wl.acts), 'cuda', bins=bench.BINS, num_of_bits=8, method='kl', half_inputs=True) for dt in dtypes}
    wq = {dt: MultiWeightQuantizer(weights[dt], wl.w_scale, wl.w_offset, channel_axis=0, half_inputs=True) for dt in dtypes}

    def step(dt):
        c = cal[dt]
        c.reset()
        for k in range(args.batches):
            wq[dt](); c.observe(sets[dt][k % args.rotate])
        c.end_phase()
        for k in range(args.batches):
            wq[dt](); c.observe(sets[dt][k % args.rotate])
        c.end_phase()

    for dt in dtypes: step(dt)                                          # leaves every calibrator with hist scales and launch-ready tables
    torch.cuda.synchronize()

    def in_phase(dt, phase):
        def run(k):
            cal[dt].phase = phase
            cal[dt].observe(sets[dt][k % args.rotate])
        return run
    kernels = {
        'multi_minmax_t': (lambda dt: in_phase(dt, 1), wl.act_elems, 1),
        'multi_histogram_t': (lambda dt: in_phase(dt, 2), wl.act_elems, 1),
        'multi_linear_quant_c': (lambda dt: (lambda k: wq[dt]()), wl.w_elems, 2),
        'step': (lambda dt: (lambda k: step(dt)), None, 0),
    }
    th = threading.Thread(target=sample, daemon=True)
    th.start()
    results = {}
    try:
        for _ in range(2):                                              # warm-up round at the timed shape, then the measured round
            results.clear()
            for kname, (make, _, _) in kernels.items():
                launches = 1 if kname == 'step' else args.launches
                for rep in range(args.reps):
                    for dt in dtypes:                                   # alternate the dtypes sample by sample
                        fn = make(dt)
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        for k in range(launches): fn(k)
                        b.record()
                        b.synchronize()
                        results.setdefault((kname, dt), []).append(a.elapsed_time(b) * 1e-3 / launches)
    finally:
        stop.set(); th.join()
    clocks.sort()
    print(json.dumps({'card': name.decode() if isinstance(name, bytes) else name,
                      'power_limit_w': pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                      'sm_mhz_sampled': {'min': clocks[0], 'median': clocks[len(clocks) // 2], 'max': clocks[-1]} if clocks else None,
                      'batch': args.batch, 'observed_tensors': len(wl.acts), 'act_elems_per_batch': wl.act_elems, 'weight_tensors': len(wl.w),
                      'weight_elems': wl.w_elems, 'batches_per_phase': args.batches,
                      'read_ceiling_gbs': ceiling['read_ceiling_gbs'], 'copy_ceiling_gbs': ceiling['copy_ceiling_gbs']}), flush=True)
    for (kname, dt), ts in results.items():
        ts.sort()
        t = ts[len(ts) // 2]
        row = {'kernel': kname, 'dtype': str(dt).replace('torch.', ''), 'median_ms': round(t * 1e3, 4), 'min_ms': round(ts[0] * 1e3, 4),
               'max_ms': round(ts[-1] * 1e3, 4)}
        _, elems, passes = kernels[kname]
        if elems is not None:
            gbs = elems * torch.tensor([], dtype=dt).element_size() * passes / t / 1e9
            roof = ceiling['copy_ceiling_gbs'] if passes == 2 else ceiling['read_ceiling_gbs']
            row.update(gbs=round(gbs, 1), share_of_ceiling=round(gbs / roof, 3), gelem_s=round(elems / t / 1e9, 2))
        print(json.dumps(row), flush=True)


if __name__ == '__main__':
    sys.exit(main())
