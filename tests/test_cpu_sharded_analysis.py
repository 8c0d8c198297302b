"""graphwise_error_analyse and layerwise_error_analyse sharded by batch over gloo (CPU, world 2 and 3): every rank returns the single-process
report bit for bit, whatever the batch count does against the world size, and a failure on one rank fails every rank without a hang.

The per-batch values come from the real executor on the tinyres network on the host: fake-quant is a fixed 1/16 grid instead of the CUDA
kernels, and the measure is the fp64 paired-moment formula on the host instead of Multi_Paired_Moments.  The batches mix shape[0] (3, 1, 2, 4),
so the layerwise running mean weighs its updates unequally.  Each rank runs its forwards on one thread, so a batch gives the same values on
every rank."""
import datetime
import os
import socket
import sys
import time

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (3, 1, 2, 4)
COUNTS = (6, 7, 2, 1, 0)                 # divisible by 2 and 3; by neither; fewer than 3 ranks; fewer than 2; none
CUTS = ((7, 2), (7, 0), (3, 8))          # layerwise (len(batches), steps): the steps cut, one batch, no cut


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


def _grid(t, cfg=None):
    return torch.round(t * 16) / 16


def _host_batch_measures(preds, reals, method, out=None):
    from ppq_b200.measure import measure_rows
    vals = []
    for p, r in zip(preds, reals):
        p, r = p.double().flatten(1), r.double().flatten(1)
        m = torch.stack([((p - r) ** 2).sum(1), (r * r).sum(1), (p * p).sum(1), (p * r).sum(1)], 1)
        vals.append(measure_rows(m, p.shape[1], method).mean())
    out.copy_(torch.stack(vals))
    return out


def _executor():
    """tinyres on the host with every config given a state and every weight baked on the 1/16 grid by hand."""
    import netspec
    from ppq_b200.core import QuantizationStates as S
    from ppq_b200.executor import TorchExecutor
    spec = netspec.SPECS['tinyres']
    ex = TorchExecutor(netspec.SpecNet(spec, netspec.make_params(spec, 1)), torch.zeros(1, 3, 32, 32), fuse_bn=False)
    ex._quant_fn = _grid
    for _, op in ex.quantable_operations():
        for c in op.input_cfgs + [op.output_cfg]:
            if c.state == S.INITIAL: c.state = S.ACTIVATED
        if op.weight_cfg is not None:
            op.stored_weight = op.module.weight.data
            op.module.weight.data = _grid(op.stored_weight)
            op.weight_cfg.state = S.BAKED
    return ex


def _snapshot(ex):
    return [(n, [c.state for c in ex._configs_of(op)], None if op.weight_cfg is None else op.module.weight.data.clone(),
             None if op.stored_weight is None else op.stored_weight.clone()) for n, op in ex.quantable_operations()]


def _same(a, b):
    for (n, s0, w0, st0), (m, s1, w1, st1) in zip(a, b):
        if n != m or s0 != s1: return False
        for u, v in ((w0, w1), (st0, st1)):
            if (u is None) != (v is None) or (u is not None and not torch.equal(u, v)): return False
    return len(a) == len(b)


def _batches(n):
    g = torch.Generator().manual_seed(99)
    return [torch.rand(SIZES[i % len(SIZES)], 3, 32, 32, generator=g) for i in range(n)]


class _Failing(list):
    """Batch 3 cannot be read."""

    def __getitem__(self, i):
        if i == 3: raise RuntimeError('batch 3 is broken')
        return list.__getitem__(self, i)


def _worker(rank, world, port, out_dir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    torch.set_num_threads(1)
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))
    import ppq_b200.measure as measure
    from ppq_b200.executor import graphwise_error_analyse, layerwise_error_analyse
    measure.batch_measures = _host_batch_measures
    group = dist.group.WORLD
    ex = _executor()
    before = _snapshot(ex)
    runs, errors, typeerrors = {}, {}, {}

    def both(key, fn, data, **kw):
        runs[key] = (fn(ex, data, group=group, **kw), fn(ex, data, **kw))

    for n in COUNTS:
        data = _batches(n)
        for fetchs in (None, 4096):
            both(('graphwise', n, fetchs), graphwise_error_analyse, data, fetchs=fetchs)
        both(('layerwise', n, 'snr'), layerwise_error_analyse, data, steps=8)
    data = _batches(7)
    for method in ('mse', 'cosine'):
        both(('layerwise', 7, method), layerwise_error_analyse, data, method=method)
    for n in (7, 1):
        both(('layerwise', n, 'two outputs'), layerwise_error_analyse, _batches(n), interested_outputs=['conv4#0', 'fc#0'])
    for n, steps in CUTS:
        both(('layerwise cut', n, steps), layerwise_error_analyse, _batches(n), steps=steps)

    for name, fn in (('graphwise', graphwise_error_analyse), ('layerwise', layerwise_error_analyse)):
        try:
            fn(ex, _Failing(_batches(7)), group=group)
            errors[name] = None
        except Exception as e:                                           # noqa: BLE001  (what each rank raises is the result)
            errors[name] = f'{type(e).__name__}: {e}'
    forwards = []
    hook = ex.model.register_forward_hook(lambda m, a, o: forwards.append(1))
    for name, fn in (('graphwise', graphwise_error_analyse), ('layerwise', layerwise_error_analyse)):
        try:
            fn(ex, iter(_batches(4)), group=group)
            typeerrors[name] = None
        except TypeError as e:
            typeerrors[name] = str(e)
    hook.remove()
    after = _snapshot(ex)

    # group=None on rank 0 alone, with every collective and query of torch.distributed made to fail
    alone = None
    if rank == 0:
        names = ('all_reduce', 'all_gather', 'broadcast', 'barrier', 'get_world_size', 'get_rank', 'get_backend', 'is_initialized')
        saved = {k: getattr(dist, k) for k in names}

        def refuse(*a, **k): raise AssertionError('torch.distributed was called with group=None')
        for k in names: setattr(dist, k, refuse)
        try:
            data = _batches(7)
            alone = (graphwise_error_analyse(ex, data) == runs[('graphwise', 7, None)][1],
                     layerwise_error_analyse(ex, data) == runs[('layerwise', 7, 'snr')][1])
        finally:
            for k, v in saved.items(): setattr(dist, k, v)
    torch.save({'runs': runs, 'errors': errors, 'typeerrors': typeerrors, 'forwards_before_typeerror': len(forwards),
                'state_kept': _same(before, after), 'state_kept_alone': _same(before, _snapshot(ex)), 'alone': alone},
               os.path.join(out_dir, f'r{rank}.pt'))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(world, out_dir, limit=240):
    """mp.spawn with a deadline: a rank left waiting in a collective fails the test instead of hanging it."""
    ctx = mp.spawn(_worker, args=(world, _free_port(), out_dir), nprocs=world, join=False)
    deadline = time.monotonic() + limit
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                if p.is_alive(): p.kill()
            pytest.fail(f'world {world}: the ranks did not finish within {limit} s')


@pytest.fixture(scope='module', params=[2, 3], ids=['world2', 'world3'])
def ranks(request, tmp_path_factory):
    out = tmp_path_factory.mktemp(f'sharded{request.param}')
    _spawn(request.param, str(out))
    return [torch.load(out / f'r{r}.pt') for r in range(request.param)]


def test_every_rank_returns_the_single_process_report_bit_for_bit(ranks):
    keys = list(ranks[0]['runs'])
    assert len(keys) == 2 * len(COUNTS) + len(COUNTS) + 2 + 2 + len(CUTS)
    for r, got in enumerate(ranks):
        assert list(got['runs']) == keys
        for key, (sharded, whole) in got['runs'].items():
            assert list(sharded) == list(whole) and sharded == whole, (r, key, sharded, whole)
            assert whole == ranks[0]['runs'][key][1], (r, key)            # the same batch gives the same values on every rank
    zero = ranks[0]['runs'][('layerwise', 0, 'snr')][0]
    assert zero and all(v == 0.0 for v in zero.values())
    assert all(v == 0.0 for v in ranks[0]['runs'][('graphwise', 0, None)][0].values())
    assert len(set(ranks[0]['runs'][('layerwise', 7, 'snr')][0].values())) > 1


def test_a_batch_that_raises_on_one_rank_fails_every_rank_and_keeps_the_state(ranks):
    owner = 3 % len(ranks)
    for r, got in enumerate(ranks):
        for name in ('graphwise', 'layerwise'):
            err = got['errors'][name]
            if r == owner: assert err == 'RuntimeError: batch 3 is broken', (r, name, err)
            else: assert err is not None and 'raised on another rank' in err, (r, name, err)
        assert got['state_kept'], r


def test_an_unsized_iterable_is_refused_before_any_forward(ranks):
    for got in ranks:
        assert all(e is not None and 'sequence' in e for e in got['typeerrors'].values()), got['typeerrors']
        assert got['forwards_before_typeerror'] == 0


def test_group_none_runs_alone_without_torch_distributed(ranks):
    assert ranks[0]['alone'] == (True, True)
    assert ranks[0]['state_kept_alone']
