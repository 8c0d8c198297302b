#!/usr/bin/env python
"""Measure the HBM read ceiling and the read+write ceiling of the current GPU (tools/hbm_ceiling.cu), with the card, its power limit and the SM
clocks sampled while the probe runs.

    python tools/hbm_ceiling.py [--buffer-mib 384] [--buffers 4] [--reps 40]

The probe is compiled for sm_90a into a temporary directory and removed afterwards; it is not part of libppq_b200.  Prints one JSON line per
configuration and a final summary line with the best read and copy rates.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--buffer-mib', type=int, default=384)
    ap.add_argument('--buffers', type=int, default=4, help='rotating input buffers (their total should exceed 1 GB)')
    ap.add_argument('--reps', type=int, default=40)
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix='hbm_ceiling_')
    try:
        exe = os.path.join(tmp, 'hbm_ceiling')
        subprocess.run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', os.path.join(HERE, 'hbm_ceiling.cu'), '-o', exe],
                       check=True)
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0].strip()
        h = pynvml.nvmlDeviceGetHandleByIndex(int(vis) if vis.isdigit() else 0)
        name = pynvml.nvmlDeviceGetName(h)
        card = {'card': name.decode() if isinstance(name, bytes) else name,
                'power_limit_w': pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                'sm_max_mhz': pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM),
                'mem_max_mhz': pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_MEM)}
        print(json.dumps(card), flush=True)
        clocks, stop = [], threading.Event()

        def sample():
            while not stop.is_set():
                clocks.append(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
                time.sleep(0.05)
        th = threading.Thread(target=sample, daemon=True)
        th.start()
        try:
            out = subprocess.run([exe, str(args.buffer_mib), str(args.buffers), str(args.reps)], check=True, capture_output=True, text=True).stdout
        finally:
            stop.set(); th.join()
        rows = [json.loads(line) for line in out.splitlines() if line.strip()]
        for r in rows: print(json.dumps(r), flush=True)
        best = {}
        for r in rows:
            if 'kind' in r and r['gbs'] > best.get(r['kind'], {'gbs': 0})['gbs']: best[r['kind']] = r
        clocks.sort()
        print(json.dumps({'summary': True, **card,
                          'read_ceiling_gbs': max(best[k]['gbs'] for k in ('read_ldg', 'read_bulk')),
                          'copy_ceiling_gbs': best['copy_ldg']['gbs'],
                          'best': {k: f"{v['config']} x {v['ctas_per_sm']} CTAs/SM, {v['depth_kb_per_sm']} KB/SM in flight" for k, v in best.items()},
                          'sm_mhz_sampled': {'min': clocks[0], 'median': clocks[len(clocks) // 2], 'max': clocks[-1], 'samples': len(clocks)}
                          if clocks else None}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    sys.exit(main())
