#!/usr/bin/env python
"""Time percentile calibration with a captured forward (calibrate_arena(method='percentile', graphs=True)) against the eager flow
(graphs=False, deferred='auto': one multi-tensor select per forward).

    python tools/bench_percentile_graphs.py [--nets resnet50,bert] [--batches 8,32] [--rounds 3] [--out RESULT.json]

Networks, fp32, TF32 off, random weights, device-resident random batches:
  * resnet50: torchvision ResNet-50 (bench_models.build), batch 32 x 3 x 224 x 224;
  * bert: the 12-layer BERT-base stack of tools/bench_encoder.py (H 768, 12 heads, FFN 3072), batch 32 x 128 tokens.
For every network and number of batches the two arms alternate `rounds` times in one process after one warm-up calibration each; a sample is
one whole calibration between CUDA events, ending in a device synchronise (the graph arm's capture and instantiation included).  Reported:
best of the rounds, the spread (min - max) and every sample, best graphs / best eager, and whether both arms gave bit-identical scales and
offsets.  The card's name, power limit and maximum SM clock are read in the same run, before and after.
Without a CUDA device the script exits with an error; there is no CPU fall-back.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import torch  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'card': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip() if q.returncode == 0 else None}


def network(name, batches):
    from ppq_b200.executor import TorchExecutor
    torch.manual_seed(0)
    g = torch.Generator(device='cuda').manual_seed(1)
    if name == 'resnet50':
        import bench_models
        model = bench_models.build('resnet50').cuda()
        xs = [torch.rand(32, 3, 224, 224, generator=g, device='cuda') for _ in range(batches)]
    else:
        import netspec_encoder as enc
        model = enc.stacked_encoder(12, 128, 768, 12, 3072).cuda()
        xs = [torch.randn(32 * 128, 768, generator=g, device='cuda') for _ in range(batches)]
    ex = TorchExecutor(model, xs[0], fuse_bn=False) if name == 'bert' else TorchExecutor(model, torch.zeros(2, 3, 224, 224, device='cuda'))
    ex.quantize_parameters()
    return ex, xs


def calibrate_ms(ex, xs, graphs):
    """One whole calibration between CUDA events; returns (ms, the scales and offsets as int32 bits), with the configs made INITIAL again."""
    from ppq_b200.core import QuantizationStates
    from ppq_b200.executor import calibrate_arena
    cfgs = ex.observed_configs()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    calibrate_arena(ex, xs, method='percentile', graphs=graphs)
    b.record(); torch.cuda.synchronize()
    bits = torch.stack([torch.cat([c.scale.reshape(-1), c.offset.reshape(-1)]) for c in cfgs]).float().cpu().view(torch.int32)
    for c in cfgs: c.state = QuantizationStates.INITIAL
    return a.elapsed_time(b), bits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--nets', default='resnet50,bert')
    ap.add_argument('--batches', default='8,32', help='calibration set sizes, comma-separated')
    ap.add_argument('--rounds', type=int, default=3, help='timed calibrations per arm, alternated')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_percentile_graphs: no CUDA device; this script measures the H100 and has no CPU fall-back')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sizes = [int(s) for s in args.batches.split(',')]
    res = {'args': vars(args), 'card_before': card()}
    for name in args.nets.split(','):
        ex, xs = network(name, max(sizes))
        res[name] = {'observed_tensors': len(ex.observed_configs())}
        for S in sizes:
            arms = {'eager': False, 'graphs': True}
            samples, bits = {k: [] for k in arms}, {}
            for k, g in arms.items(): _, bits[k] = calibrate_ms(ex, xs[:S], g)          # warm-up: cuDNN / cuBLAS, descriptor tables, allocator
            for _ in range(args.rounds):
                for k, g in arms.items():
                    ms, bits[k] = calibrate_ms(ex, xs[:S], g)
                    samples[k].append(round(ms, 2))
            row = {k: {'best_ms': min(v), 'spread_ms': [min(v), max(v)], 'ms': v} for k, v in samples.items()}
            row['graphs_over_eager'] = round(min(samples['graphs']) / min(samples['eager']), 3)
            row['same_scales'] = bool(torch.equal(bits['eager'], bits['graphs']))
            res[name][f'{S}_batches'] = row
            print(json.dumps({name: {S: row}}), flush=True)
        del ex, xs
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f: f.write(line + '\n')


if __name__ == '__main__':
    main()
