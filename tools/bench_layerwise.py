#!/usr/bin/env python
"""Time layerwise_error_analyse against the reference's algorithm on the same executor, and the Multi_Paired_Moments kernel on its own.

    python tools/bench_layerwise.py [--nets resnet50,yolov5s] [--batch 32] [--steps 8] [--rounds 2] [--out RESULT.json]

Networks: torchvision ResNet-50 (random init, BN folded) at 224 x 224 and YOLOv5s (bench_models) at 640 x 640, both calibrated with
calibrate_arena('kl'), aligned and baked.  Two arms, alternated `rounds` times in one process, each ending in a device synchronise:
  (a) reference: ppq/quantization/analyse/layerwise.py:73-134 restated on ppq_b200's executor (operation-outer, an fp32 and a single-operation
      forward per operation and batch, the reference's torch measures, `.item()` per update: tests/layerwise_oracle.reference_layerwise);
  (b) layerwise_error_analyse (batch-outer, one paired-moment launch per quantised forward, one copy to the host at the end).
Reports forward counts (a module hook), wall-clock per arm, the largest relative difference of the two reports, the kernel time of one
Multi_Paired_Moments launch over the network's outputs (CUDA events, many launches) with bytes / s from the shapes against the data-sheet 3.35 TB/s
and the read ceiling tools/hbm_ceiling.py measures in the same run, and the card's name and power limit read in the same run.
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

DATASHEET_TBS = 3.35


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return {'card': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip() if q.returncode == 0 else None}


def read_ceiling():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'hbm_ceiling.py')], capture_output=True, text=True)
    for line in reversed(r.stdout.splitlines()):
        try:
            d = json.loads(line)
        except ValueError:
            continue
        if d.get('summary'): return d['read_ceiling_gbs'] / 1e3
    return None


def network(name, batch, steps, device):
    import bench_models
    from ppq_b200.executor import TorchExecutor, calibrate_arena
    torch.manual_seed(0)
    image = (3, 640, 640) if name == 'yolov5s' else (3, 224, 224)
    model = bench_models.build(name).to(device)
    ex = TorchExecutor(model, torch.zeros((2,) + image, device=device))
    ex.quantize_parameters()
    g = torch.Generator(device=device).manual_seed(1)
    xs = [torch.rand((batch,) + image, generator=g, device=device) for _ in range(steps + 1)]
    calibrate_arena(ex, xs[:4], method='kl')
    ex.align_quantization()
    ex.bake_parameters()
    return ex, xs


def kernel_time(outputs, reps=200):
    """One Multi_Paired_Moments launch over (outputs, outputs + noise), staged once; CUDA events around `reps` launches."""
    from ppq_b200.ffi import extension
    ext = extension()
    reals = [t.detach().contiguous() for t in outputs]
    preds = [t + 1e-3 * torch.randn_like(t) for t in reals]
    rows = [(1 if t.dim() == 1 else t.shape[0]) for t in reals]
    row0 = [sum(rows[:k]) for k in range(len(rows))]
    descs = torch.tensor([(p.data_ptr(), r.data_ptr(), n, p.numel() // n, o) for p, r, n, o in zip(preds, reals, rows, row0)],
                         dtype=torch.int64, device=reals[0].device)
    elems = sum(t.numel() for t in reals)
    out = torch.empty(sum(rows), 4, dtype=torch.float64, device=reals[0].device)
    ws = torch.empty(ext.Multi_Paired_Moments_Workspace_Bytes(sum(rows), elems), dtype=torch.uint8, device=reals[0].device)
    for _ in range(20): ext.Multi_Paired_Moments(descs, elems, reals[0].dtype, out, ws)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    for _ in range(reps): ext.Multi_Paired_Moments(descs, elems, reals[0].dtype, out, ws)
    b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    nbytes = 2 * elems * reals[0].element_size()
    return {'ms': round(ms, 4), 'bytes': nbytes, 'rows': sum(rows), 'elements_per_pair_table': elems, 'tbs': round(nbytes / (ms * 1e-3) / 1e12, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--nets', default='resnet50,yolov5s')
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available(): raise SystemExit('bench_layerwise needs a CUDA device')
    import layerwise_oracle as lo
    from ppq_b200.executor import COMPUTING_OP, layerwise_error_analyse
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    device = torch.device('cuda', 0)
    result = {'card': card(), 'read_ceiling_tbs': read_ceiling(), 'datasheet_tbs': DATASHEET_TBS, 'nets': {}}
    for name in args.nets.split(','):
        ex, xs = network(name, args.batch, args.steps, device)
        K = sum(op.kind in COMPUTING_OP for _, op in ex.quantable_operations())
        calls = []
        hook = ex.model.register_forward_hook(lambda m, a, o: calls.append(1))
        arms = {'reference': lambda: lo.reference_layerwise(ex, xs, method='snr', steps=args.steps),
                'ours': lambda: layerwise_error_analyse(ex, xs, method='snr', steps=args.steps)}
        times, forwards, reports = {k: [] for k in arms}, {}, {}
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                calls.clear()
                torch.cuda.synchronize(); t0 = time.perf_counter()
                reports[arm] = fn()
                torch.cuda.synchronize(); times[arm].append(round(time.perf_counter() - t0, 3))
                forwards[arm] = len(calls)
        hook.remove()
        a, b = reports['reference'], reports['ours']
        assert list(a) == list(b)
        diff = max(abs(a[n] - b[n]) / max(abs(a[n]), 1e-30) for n in a)
        with torch.no_grad():
            out = ex.forward(xs[0])
        outs = list(out) if isinstance(out, (tuple, list)) else [out]
        kt = kernel_time(outs)
        if result['read_ceiling_tbs']: kt['of_read_ceiling'] = round(kt['tbs'] / result['read_ceiling_tbs'], 3)
        kt['of_datasheet'] = round(kt['tbs'] / DATASHEET_TBS, 3)
        result['nets'][name] = {'batch': args.batch, 'steps': args.steps, 'batches_measured': min(len(xs), args.steps + 1),
                                'computing_operations': K, 'forwards': forwards, 'seconds': times,
                                'max_relative_difference_of_reports': diff, 'outputs': [list(t.shape) for t in outs],
                                'multi_paired_moments': kt}
        print(json.dumps({name: result['nets'][name]}), flush=True)
        del ex, xs
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f: json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
