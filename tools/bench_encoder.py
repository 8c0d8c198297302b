#!/usr/bin/env python
"""Time calibration and layerwise error analysis of a BERT-base-shaped encoder stack through ppq_b200's executor.

    python tools/bench_encoder.py [--layers 12] [--hidden 768] [--heads 12] [--seq 128] [--ffn 3072] [--batch 32] [--batches 8]
                                  [--steps 3] [--analyse-steps 1] [--out RESULT.json]

The network is `layers` post-LN encoder blocks (tests/netspec_encoder.py: Gemm Q / K / V, Reshape / Transpose heads, MatMul -> Softmax ->
MatMul, output Gemm, Add, LayerNorm, Gemm -> Gelu -> Gemm, Add, LayerNorm) on a token matrix [batch * seq, hidden], random weights, TF32 off.
Reported, each with the card's name and power limit read in the same run:
  * calibrate_arena ('kl' and 'percentile', deferred='auto') over `batches` device-resident batches, fp32 and bf16 (half_inputs=True):
    milliseconds per whole calibration, `steps` timed after one warm-up, CUDA events around work that ends in a synchronise;
  * the multi-tensor collectors alone on one forward's observed tensors (Multi_MinMax_T, Multi_Histogram_T, Multi_Quantile_T and their
    *_Half forms): kernel time from CUDA events over repeated launches, bytes read computed from the tensors' sizes, and that rate against the
    HBM read ceiling tools/hbm_ceiling.py measures in the same run;
  * layerwise_error_analyse on the kl-calibrated, aligned and baked fp32 network (`analyse_steps` + 1 batches).
Without a CUDA device the script exits with an error; there is no CPU fall-back.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import torch  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return {'card': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip() if q.returncode == 0 else None}


def read_ceiling():
    """The best HBM read rate (GB/s) of tools/hbm_ceiling.py, run now on this card."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'hbm_ceiling.py')], capture_output=True, text=True)
    for line in reversed(r.stdout.splitlines()):
        try:
            d = json.loads(line)
        except ValueError:
            continue
        if d.get('summary'): return d['read_ceiling_gbs']
    raise RuntimeError('tools/hbm_ceiling.py gave no summary: ' + r.stderr[-2000:])


def synced_ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    for _ in range(reps): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def build(args, dtype):
    import netspec_encoder as enc
    from ppq_b200.executor import TorchExecutor
    model = enc.stacked_encoder(args.layers, args.seq, args.hidden, args.heads, args.ffn).cuda().to(dtype)
    g = torch.Generator(device='cuda').manual_seed(1)
    xs = [torch.randn(args.batch * args.seq, args.hidden, generator=g, device='cuda').to(dtype) for _ in range(max(args.batches, args.analyse_steps + 1))]
    ex = TorchExecutor(model, xs[0], fuse_bn=False)
    ex.quantize_parameters()
    return ex, xs


def calibration_times(ex, xs, method, half, steps):
    from ppq_b200.core import QuantizationStates
    from ppq_b200.executor import calibrate_arena
    cfgs = ex.observed_configs()

    def run():
        calibrate_arena(ex, xs, method=method, half_inputs=half)
        for c in cfgs: c.state = QuantizationStates.INITIAL
    run()                                                                  # warm-up: cuBLAS heuristics, descriptor tables, allocator
    times = [synced_ms(run) for _ in range(steps)]
    return {'ms_per_calibration': [round(t, 2) for t in times], 'ms_per_calibration_min': round(min(times), 2),
            'batches': len(xs), 'passes_over_the_batches': 2 if method == 'kl' else 1, 'observed_tensors': len(cfgs)}


def collector_rates(ex, x, half, ceiling_gbs, reps=20):
    """Each multi-tensor collector on one forward's observed tensors: kernel time (CUDA events over `reps` launches) and bytes read / s."""
    from ppq_b200.calibration import ArenaCalibrator
    from ppq_b200.calibration import is_dense
    _, ts = ex.forward(x, collect=True)
    ts = [t if is_dense(t) else t.contiguous() for t in ts]
    nbytes = sum(t.numel() * t.element_size() for t in ts)
    out = {'tensors': len(ts), 'bytes_per_pass': nbytes}
    for method, phases in (('kl', ('minmax', 'histogram')), ('percentile', ('quantile',))):
        cal = ArenaCalibrator(len(ts), x.device, method=method, half_inputs=half)
        for phase in phases:
            if phase == 'histogram':
                cal.observe(ts); cal.end_phase()                          # min/max of the tensors -> histogram scales, then phase 2
            if phase == 'quantile': cal.begin_batch()
            cal.observe(ts)                                                # warm-up launch
            ms = synced_ms(lambda: cal.observe(ts), reps)
            gbs = nbytes / (ms * 1e-3) / 1e9
            out[phase] = {'ms': round(ms, 4), 'GB_per_s': round(gbs, 1), 'of_read_ceiling': round(gbs / ceiling_gbs, 3)}
    del ts
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, default=12)
    ap.add_argument('--hidden', type=int, default=768)
    ap.add_argument('--heads', type=int, default=12)
    ap.add_argument('--seq', type=int, default=128)
    ap.add_argument('--ffn', type=int, default=3072)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--batches', type=int, default=8, help='calibration batches')
    ap.add_argument('--steps', type=int, default=3, help='timed calibrations per configuration')
    ap.add_argument('--analyse-steps', type=int, default=1, help="layerwise_error_analyse's `steps` (steps + 1 batches)")
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_encoder: no CUDA device; this script measures the H100 and has no CPU fall-back')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {'shape': vars(args), 'card_before': card()}
    ceiling = read_ceiling()
    res['hbm_read_ceiling_GB_per_s'] = round(ceiling, 1)
    from ppq_b200.executor import calibrate_arena, layerwise_error_analyse
    for name, dtype in (('fp32', torch.float32), ('bf16', torch.bfloat16)):
        ex, xs = build(args, dtype)
        half = dtype != torch.float32
        cal_xs = xs[:args.batches]
        res[name] = {m: calibration_times(ex, cal_xs, m, half, args.steps) for m in ('kl', 'percentile')}
        res[name]['collectors'] = collector_rates(ex, xs[0], half, ceiling)
        if dtype == torch.float32:
            calibrate_arena(ex, cal_xs, method='kl')
            ex.align_quantization(); ex.bake_parameters()
            layerwise_error_analyse(ex, xs[:2], steps=0)                     # warm-up
            torch.cuda.synchronize(); t0 = time.perf_counter()
            report = layerwise_error_analyse(ex, xs, steps=args.analyse_steps)
            torch.cuda.synchronize()
            res['fp32']['layerwise_error_analyse'] = {'s': round(time.perf_counter() - t0, 3), 'operations': len(report),
                                                      'batches': min(len(xs), args.analyse_steps + 1),
                                                      'snr_max': max(report.values()), 'all_finite': all(v == v for v in report.values())}
        del ex, xs
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f: f.write(line + '\n')


if __name__ == '__main__':
    main()
