#!/usr/bin/env python
"""Time layerwise_error_analyse sharded by batch over N GPUs, one process per GPU over NCCL, and check that every N returns the N = 1 report.

    python tools/bench_sharded_analysis.py [--nets resnet50,yolov5s] [--gpus 1,2,4,8] [--batch 32] [--steps 8] [--rounds 2] [--out RESULT.json]

Networks as in tools/bench_layerwise.py: torchvision ResNet-50 (random init, BN folded) at 224 x 224 and YOLOv5s (bench_models) at 640 x 640,
calibrated with calibrate_arena('kl'), aligned and baked, batch 32, S = 8 (9 batches), deterministic cuDNN.  Every rank builds the same
network and batches from the same seeds on its own GPU.  N = 1 calls the function without a group; N > 1 passes the NCCL world group.  After
one untimed call, `rounds` calls are timed on the host clock between a barrier and a device synchronise; a round's time is the slowest rank's.
An N larger than the machine's GPU count is reported as not measured.  The card's name and power limit are read in the same run.
"""
import argparse
import datetime
import json
import os
import socket
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tools')]

import torch  # noqa: E402


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


def worker(rank, world, port, name, batch, steps, rounds, out_dir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tools')]
    import torch.distributed as dist

    from bench_layerwise import network
    from ppq_b200.executor import COMPUTING_OP, layerwise_error_analyse
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.cuda.set_device(rank)
    device = torch.device('cuda', rank)
    group = None
    if world > 1:
        os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=device, timeout=datetime.timedelta(seconds=600))
        group = dist.group.WORLD
    ex, xs = network(name, batch, steps, device)
    K = sum(op.kind in COMPUTING_OP for _, op in ex.quantable_operations())
    layerwise_error_analyse(ex, xs, steps=steps, group=group)                 # untimed: lazy initialisation, allocator growth
    seconds = []
    for _ in range(rounds):
        if group is not None: dist.barrier()
        torch.cuda.synchronize(); t0 = time.perf_counter()
        report = layerwise_error_analyse(ex, xs, steps=steps, group=group)
        torch.cuda.synchronize(); t = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device=device)
        if group is not None: dist.all_reduce(t, op=dist.ReduceOp.MAX)
        seconds.append(round(t.item(), 3))
    if rank == 0:
        with open(os.path.join(out_dir, 'result.json'), 'w') as f:
            json.dump({'seconds': seconds, 'report': report, 'K': K, 'batches_measured': min(len(xs), steps + 1)}, f)
    if group is not None:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--nets', default='resnet50,yolov5s')
    ap.add_argument('--gpus', default='1,2,4,8')
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available(): raise SystemExit('bench_sharded_analysis needs a CUDA device')
    import torch.multiprocessing as mp

    from bench_layerwise import card
    have = torch.cuda.device_count()
    result = {'card': card(), 'gpus_on_machine': have, 'batch': args.batch, 'steps': args.steps, 'nets': {}}
    print(json.dumps({'card': result['card'], 'gpus_on_machine': have}), flush=True)
    for name in args.nets.split(','):
        rows, n1 = {}, None
        for n in [int(v) for v in args.gpus.split(',')]:
            if n > have:
                rows[n] = 'not measured'
            else:
                with tempfile.TemporaryDirectory() as tmp:
                    mp.spawn(worker, args=(n, _free_port(), name, args.batch, args.steps, args.rounds, tmp), nprocs=n, join=True)
                    with open(os.path.join(tmp, 'result.json')) as f: got = json.load(f)
                if n1 is None and n == 1: n1 = got['report']
                rows[n] = {'seconds': got['seconds'], 'forwards': (got['K'] + 1) * got['batches_measured'],
                           'report_equals_n1': None if n1 is None else got['report'] == n1}
            print(json.dumps({name: {n: rows[n]}}), flush=True)
        result['nets'][name] = rows
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f: json.dump(result, f, indent=1)
    if any(isinstance(r, dict) and r['report_equals_n1'] is False for rows in result['nets'].values() for r in rows.values()):
        raise SystemExit('a sharded report differs from the N = 1 report')


if __name__ == '__main__':
    main()
