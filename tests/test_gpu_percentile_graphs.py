"""calibrate_arena(method='percentile', graphs=True): one captured forward replayed for every batch, the per-batch {upper, lower} rows filed
on the device by a batch counter.  With deterministic cuDNN / no TF32 it must give every observed config the scale, offset and state of the
eager runs (graphs=False, deferred=True and 'auto') bit for bit, on tinyres, tinycat and the post-LN encoder block, in fp32 and in bf16
(half_inputs=True):

  * the per-batch rows equal the eager rows, the percentile override is honoured, there is exactly one capture per calibration;
  * batches that send the guarded (guess-remembering) select down other routes from replay to replay still match, and the guess words left
    behind equal those of the same select sequence run eagerly from a fresh guess: the warm-up forward before the capture leaves none behind;
  * the counter ends at len(batches), a second calibration on the same executor starts from zero, a sequence that yields more batches than
    its length raises before the extra replay;
  * two and three processes on one GPU (gloo), and two GPUs over NCCL where the machine has them, with `group=` give the one-process scales."""
import datetime
import os
import socket
import sys
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NETS = ['tinyres', 'tinycat', 'encoder']
DTYPES = {'fp32': torch.float32, 'bf16': torch.bfloat16}


def _deterministic():
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(scope='module', autouse=True)
def gpu():
    if not torch.cuda.is_available(): pytest.skip('no CUDA device')
    _deterministic()


def _net(name, dtype, device='cuda', steps=7, data=None):
    """A fresh executor with quantised weights and its batches (`data`: host arrays instead of the spec's own)."""
    from ppq_b200.executor import TorchExecutor
    if name == 'encoder':
        import netspec_encoder as enc
        model = enc.EncoderNet(enc.ENCODER, enc.make_params(enc.ENCODER, 11))
        xs = enc.make_data(12, steps) if data is None else data
    else:
        import netspec
        spec = netspec.SPECS[name]
        model = netspec.SpecNet(spec, netspec.make_params(spec, 3))
        xs = netspec.make_data(name, 4, steps, 4) if data is None else data
    model = model.to(device).to(dtype)
    batches = [torch.from_numpy(x).to(device).to(dtype) for x in xs]
    ex = TorchExecutor(model, batches[0], fuse_bn=False)
    ex.quantize_parameters()
    return ex, batches


def _bits(t):
    t = t.detach().reshape(-1).float().cpu()
    return t.view(torch.int32)


def _result(cfgs):
    return [(c.state.name, _bits(c.scale), _bits(c.offset)) for c in cfgs]


def _same(a, b, tag):
    assert len(a) == len(b), tag
    for k, ((sa, xa, oa), (sb, xb, ob)) in enumerate(zip(a, b)):
        assert sa == sb, (tag, k, sa, sb)
        assert torch.equal(xa, xb), (tag, k, 'scale', xa, xb)
        assert torch.equal(oa, ob), (tag, k, 'offset', oa, ob)


class _Counting:
    """torch.cuda.CUDAGraph with a count of instantiations."""

    def __init__(self, monkeypatch):
        self.n = 0
        base, outer = torch.cuda.CUDAGraph, self

        class Graph(base):
            def __init__(self, *a, **kw):
                outer.n += 1
                super().__init__(*a, **kw)
        monkeypatch.setattr(torch.cuda, 'CUDAGraph', Graph)


def _calibrate(name, dtype, graphs, deferred='auto', data=None, steps=7, override=None):
    from ppq_b200.core import OBSERVER_PERCENTILE_MANUL_OVERRIDE
    from ppq_b200.executor import calibrate_arena
    ex, batches = _net(name, dtype, data=data, steps=steps)
    cfgs = ex.observed_configs()
    if override is not None:
        for c in cfgs: c.detail[OBSERVER_PERCENTILE_MANUL_OVERRIDE] = override
    cal = calibrate_arena(ex, batches, method='percentile', graphs=graphs, deferred=deferred, half_inputs=dtype != torch.float32)
    return ex, batches, cfgs, cal


@pytest.mark.parametrize('dtype', list(DTYPES))
@pytest.mark.parametrize('name', NETS)
def test_graphs_equal_the_eager_runs(monkeypatch, name, dtype):
    dt = DTYPES[dtype]
    eager = {}
    for deferred in (True, 'auto'):
        _, _, cfgs, cal = _calibrate(name, dt, False, deferred)
        eager[deferred] = (_result(cfgs), cal.batch_rows())
    count = _Counting(monkeypatch)
    ex, batches, cfgs, cal = _calibrate(name, dt, True)
    assert count.n == 1, count.n
    assert int(cal._count.item()) == len(batches) and cal._rows.shape[0] == len(batches)
    for deferred, (want, rows) in eager.items():
        _same(_result(cfgs), want, f'{name}/{dtype} graphs vs deferred={deferred}')
        assert torch.equal(cal.batch_rows(), rows), (name, dtype, deferred)
    assert rows.shape == (len(cfgs), len(batches), 2)


def test_percentile_override_is_honoured():
    _, _, cfgs_e, cal_e = _calibrate('tinyres', torch.float32, False, override=0.99)
    _, _, cfgs_g, cal_g = _calibrate('tinyres', torch.float32, True, override=0.99)
    _, _, cfgs_d, _ = _calibrate('tinyres', torch.float32, True)
    assert cal_g.percentile == cal_e.percentile == 0.99
    _same(_result(cfgs_g), _result(cfgs_e), 'override 0.99')
    assert torch.equal(cal_g.batch_rows(), cal_e.batch_rows())
    assert any(not torch.equal(a[1], b[1]) for a, b in zip(_result(cfgs_g), _result(cfgs_d))), 'the override did not change any scale'


def _route_data():
    """tinyres at batch 96 (conv1 output 1.5 M elements): 0 images (cold), 1 other images (the thresholds hold: hit), 2 images x 50 (a miss),
    3 other images x 50 (hit), 4 every input value within 1024 ulps of 100.0 (the input's selected bucket holds more keys than the
    single-tensor workspace: histogram refinement down to pass 2), 5 images again (a miss)."""
    r = np.random.RandomState(31)
    shape = (96, 3, 32, 32)
    img = lambda: r.rand(*shape).astype(np.float32)
    n = int(np.prod(shape))
    close = (np.float32(100.0).view(np.uint32) + r.randint(0, 1024, n).astype(np.uint32)).view(np.float32).reshape(shape)
    return [img(), img(), img() * 50, img() * 50, close, img()]


def test_select_routes_change_between_replays_and_the_guess_words_match_eager(monkeypatch):
    from ppq_b200.ffi import extension
    ext = extension()
    data = _route_data()
    _, _, want, _ = _calibrate('tinyres', torch.float32, False, True, data=data)
    _, _, want_auto, _ = _calibrate('tinyres', torch.float32, False, 'auto', data=data)
    count = _Counting(monkeypatch)
    _, batches, cfgs, cal = _calibrate('tinyres', torch.float32, True, data=data)
    assert count.n == 1
    _same(_result(cfgs), _result(want), 'routes: graphs vs deferred=True')
    _same(_result(cfgs), _result(want_auto), "routes: graphs vs deferred='auto'")
    # the same selects eagerly, slot by slot, from a fresh guess: what the replays must leave in the guess words
    ex, xs = _net('tinyres', torch.float32, data=data)
    guess = ext.Quantile_Guess_Init(len(ex.observed_configs()), xs[0])
    rows = []
    for x in xs:
        row = torch.zeros(len(cfgs), 2, device='cuda')
        ex.forward(x, sink=lambda k, t: row[k].copy_(ext.Quantile_T_Guess(t, cal.percentile, guess[k])))
        rows.append(row)
    assert torch.equal(cal._select_guess, guess)
    assert torch.equal(cal.batch_rows(), torch.stack(rows, dim=1))


def test_counter_and_a_second_calibration(monkeypatch):
    from ppq_b200.core import QuantizationStates
    from ppq_b200.executor import calibrate_arena
    ex, batches, cfgs, cal = _calibrate('tinycat', torch.float32, True)
    assert int(cal._count.item()) == len(batches)
    first = _result(cfgs)
    for c in cfgs: c.state = QuantizationStates.INITIAL
    count = _Counting(monkeypatch)
    cal2 = calibrate_arena(ex, iter(batches[:5]), method='percentile', graphs=True)      # a one-shot iterator: sized before the first batch
    assert count.n == 1 and cal2 is not cal
    assert int(cal2._count.item()) == 5 and cal2._rows.shape[0] == 5
    assert torch.equal(cal2.batch_rows(), cal.batch_rows()[:, :5])
    for c in cfgs: c.state = QuantizationStates.INITIAL
    cal3 = calibrate_arena(ex, batches, method='percentile', graphs=True)
    assert int(cal3._count.item()) == len(batches)
    _same(_result(cfgs), first, 'second full calibration on the same executor')


class _LongerThanItsLength(list):
    def __len__(self): return super().__len__() - 1


def test_more_batches_than_rows_raise_before_the_replay(monkeypatch):
    from ppq_b200.executor import calibrate_arena
    ex, batches = _net('tinyres', torch.float32)
    calls, real = [], torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, 'replay', lambda self: (calls.append(1), real(self))[1])
    with pytest.raises(RuntimeError, match='overruns the 6 per-batch rows'):
        calibrate_arena(ex, _LongerThanItsLength(batches), method='percentile', graphs=True)
    assert len(calls) == len(batches) - 1


# ------------------------------------------------------------------------------------------------------------------ sharded
def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


SHARDED = [('tinyres', torch.float32), ('tinycat', torch.float32), ('encoder', torch.float32), ('tinyres', torch.bfloat16)]


def _calibrate_all(name, dtype, device, rank=0, world=1, group=None):
    """The percentile calibration of `name` over this rank's share of the 7 batches; returns (batches calibrated here, configs)."""
    from ppq_b200.calibration import shard_indices
    from ppq_b200.executor import calibrate_arena
    ex, xs = _net(name, dtype, device=device)
    cfgs = ex.observed_configs()
    mine = [xs[i] for i in shard_indices(len(xs), rank, world)]
    cal = calibrate_arena(ex, mine, method='percentile', graphs=True, group=group, half_inputs=dtype != torch.float32)
    return int(cal._count.item()), _result(cfgs)


def _run_sharded(rank, world, device, group, nets):
    return {(name, str(dtype)): _calibrate_all(name, dtype, device, rank, world, group) for name, dtype in nets}


def _worker(rank, world, port, out_dir, backend):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    import torch.distributed as dist
    _deterministic()
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    device = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(device)
    kw = {'device_id': device} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120), **kw)
    out = _run_sharded(rank, world, device, dist.group.WORLD, SHARDED if backend == 'gloo' else SHARDED[:1])
    torch.save(out, os.path.join(out_dir, f'{backend}{rank}.pt'))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(world, out_dir, backend, limit=600):
    import torch.multiprocessing as mp
    ctx = mp.spawn(_worker, args=(world, _free_port(), out_dir, backend), nprocs=world, join=False)
    deadline = time.monotonic() + limit
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                if p.is_alive(): p.kill()
            pytest.fail(f'world {world}: the ranks did not finish within {limit} s')


def _check(got, world, nets):
    """Every rank's scales equal those of one process calibrating all 7 batches (here, outside any process group)."""
    for name, dtype in nets:
        key = (name, str(dtype))
        seen, whole = _calibrate_all(name, dtype, torch.device('cuda', 0))
        assert seen == 7 and sum(g[key][0] for g in got) == 7
        for r, g in enumerate(got):
            assert g[key][0] == len(range(r, 7, world))
            _same(g[key][1], whole, f'{key} rank {r} of {world}')


@pytest.mark.parametrize('world', [2, 3])
def test_sharded_graphs_equal_one_process_on_one_gpu(world, tmp_path):
    _spawn(world, str(tmp_path), 'gloo')
    _check([torch.load(tmp_path / f'gloo{r}.pt') for r in range(world)], world, SHARDED)


def test_sharded_graphs_over_nccl_on_two_gpus(tmp_path):
    if torch.cuda.device_count() < 2: pytest.skip('needs 2 GPUs')
    _spawn(2, str(tmp_path), 'nccl')
    _check([torch.load(tmp_path / f'nccl{r}.pt') for r in range(2)], 2, SHARDED[:1])
