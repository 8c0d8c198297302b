"""graphwise_error_analyse and layerwise_error_analyse sharded by batch on the GPU: two and three processes on one device over gloo, and two
devices over NCCL where the machine has them.  With deterministic cuDNN every rank's report equals the single-process report (group=None)
with == on every value, and every config's state, scale and offset and every weight are as before the call, on every rank.

The batches: 7 of them (divisible by neither world size), the last one with 2 samples instead of 4 (the layerwise running mean weighs it
less), except under graphs=True, which replays one batch shape; and 2 batches, fewer than three ranks."""
import datetime
import os
import socket
import sys
import time

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


def _deterministic():
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False


def _calibrated(name, device, dtype=torch.float32):
    import netspec
    from ppq_b200.executor import TorchExecutor, calibrate_arena
    spec = netspec.SPECS[name]
    model = netspec.SpecNet(spec, netspec.make_params(spec, 3)).to(device).to(dtype)
    xs = [torch.from_numpy(x).to(device).to(dtype) for x in netspec.make_data(name, 4, 7, 4)]
    ex = TorchExecutor(model, xs[0], fuse_bn=False)
    ex.quantize_parameters()
    calibrate_arena(ex, xs, method='kl', half_inputs=dtype != torch.float32)
    ex.align_quantization()
    ex.bake_parameters()
    return ex, xs


def _snapshot(ex):
    def bits(t):
        return None if t is None else t.detach().reshape(-1).cpu().clone().view(torch.int16 if t.element_size() == 2 else torch.int32)
    rows = []
    for n, op in ex.quantable_operations():
        for c in ex._configs_of(op): rows.append((n, c.state, bits(c._scale), bits(c._offset)))
        if op.weight_cfg is not None: rows.append((n, bits(op.module.weight.data), bits(op.stored_weight)))
    return rows


def _same(a, b):
    if len(a) != len(b): return False
    for x, y in zip(a, b):
        if len(x) != len(y): return False
        for u, v in zip(x, y):
            if isinstance(u, torch.Tensor) or isinstance(v, torch.Tensor):
                if u is None or v is None or not torch.equal(u, v): return False
            elif u != v: return False
    return True


def _cases(name, dtype):
    """(key, analysis, which batches, keywords) for one network."""
    g, lw = 'graphwise', 'layerwise'
    if dtype != torch.float32:
        return [((name, 'bf16', lw, 'snr'), lw, 'mixed', {}), ((name, 'bf16', g, 'whole tensors'), g, 'mixed', {})]
    outs = {'tinyres': ['conv4#0', 'add1#0', 'fc#0'], 'tinycat': ['mix#0', 'head#0']}[name]
    return ([((name, lw, m), lw, 'mixed', dict(method=m)) for m in ('snr', 'mse', 'cosine')] +
            [((name, lw, 'named outputs'), lw, 'mixed', dict(interested_outputs=outs)),
             ((name, lw, 'two batches'), lw, 'two', {}),
             ((name, g, 'whole tensors'), g, 'mixed', {}),
             ((name, g, 'fetchs=4096'), g, 'mixed', dict(fetchs=4096)),
             ((name, g, 'graphs=True'), g, 'fixed', dict(graphs=True)),
             ((name, g, 'two batches'), g, 'two', {})])


def _run_all(rank, device, group, nets):
    """Every case sharded over `group` on every rank; rank 0 also runs it with group=None.  Returns what the parent checks."""
    import torch.distributed as dist
    from ppq_b200.executor import graphwise_error_analyse, layerwise_error_analyse
    fns = {'graphwise': graphwise_error_analyse, 'layerwise': layerwise_error_analyse}
    sharded, whole, kept = {}, {}, {}
    for name, dtype in nets:
        ex, xs = _calibrated(name, device, dtype)
        data = {'mixed': xs[:6] + [xs[6][:2]], 'fixed': xs, 'two': xs[:2]}
        before = _snapshot(ex)
        for key, which, batches, kw in _cases(name, dtype):
            sharded[key] = fns[which](ex, data[batches], group=group, **kw)
            if rank == 0: whole[key] = fns[which](ex, data[batches], **kw)
            dist.barrier(group)
        kept[(name, str(dtype))] = _same(before, _snapshot(ex))
    return {'sharded': sharded, 'whole': whole, 'kept': kept}


NETS = [('tinyres', torch.float32), ('tinycat', torch.float32), ('tinyres', torch.bfloat16)]


def _gloo_worker(rank, world, port, out_dir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    import torch.distributed as dist
    _deterministic()
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    out = _run_all(rank, torch.device('cuda', 0), dist.group.WORLD, NETS)
    torch.save(out, os.path.join(out_dir, f'g{rank}.pt'))
    dist.barrier()
    dist.destroy_process_group()


def _nccl_worker(rank, world, port, out_dir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    import torch.distributed as dist
    _deterministic()
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank),
                            timeout=datetime.timedelta(seconds=120))
    out = _run_all(rank, torch.device('cuda', rank), dist.group.WORLD, NETS[:1])
    torch.save(out, os.path.join(out_dir, f'n{rank}.pt'))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(worker, world, out_dir, limit=600):
    import torch.multiprocessing as mp
    ctx = mp.spawn(worker, args=(world, _free_port(), out_dir), nprocs=world, join=False)
    deadline = time.monotonic() + limit
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                if p.is_alive(): p.kill()
            pytest.fail(f'world {world}: the ranks did not finish within {limit} s')


def _check(got, nets):
    keys = [key for name, dtype in nets for key, _, _, _ in _cases(name, dtype)]
    whole = got[0]['whole']
    assert list(whole) == keys
    for r, res in enumerate(got):
        assert list(res['sharded']) == keys
        for key in keys:
            s, w = res['sharded'][key], whole[key]
            assert list(s) == list(w) and all(s[n] == w[n] for n in w), (r, key, s, w)
        assert all(res['kept'].values()), (r, res['kept'])
    assert len(set(whole[('tinyres', 'layerwise', 'snr')].values())) > 1


@pytest.mark.parametrize('world', [2, 3])
def test_sharded_reports_equal_the_single_process_reports_on_one_gpu(world, tmp_path):
    if not torch.cuda.is_available(): pytest.skip('no CUDA device')
    _spawn(_gloo_worker, world, str(tmp_path))
    _check([torch.load(tmp_path / f'g{r}.pt') for r in range(world)], NETS)


def test_sharded_reports_over_nccl_on_two_gpus(tmp_path):
    if torch.cuda.device_count() < 2: pytest.skip('needs 2 GPUs')
    _spawn(_nccl_worker, 2, str(tmp_path))
    _check([torch.load(tmp_path / f'n{r}.pt') for r in range(2)], NETS[:1])
