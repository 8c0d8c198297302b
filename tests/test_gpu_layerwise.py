"""Layerwise error analysis on the GPU.

Multi_Paired_Moments is held to the exact-moment oracle (tests/layerwise_oracle.py) within (k + 1) 2^-53 sum |terms| (k + 3 for
sum (p - r)^2), for fp32 / fp16 / bf16 pairs, rows of 1 to 2^24 + 5 elements, pointers off the 16-byte grid, channels_last pairs, big and empty
tables, special values and zero rows; two launches and two replays of a captured CUDA graph are bit-identical.
layerwise_error_analyse is held to the reference's loop restated on the same executor (operation-outer, torch measures, .item() per update)
on tinyres, tinycat, a two-output network and a bf16 network, with deterministic cuDNN."""
import numpy as np
import pytest
import torch

import layerwise_oracle as lo
import netspec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _cuda():
    if not torch.cuda.is_available(): pytest.skip('no CUDA device')
    flags = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32,
             torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = flags


DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def rand_pair(shape, dtype, seed, offsets=(0, 0), scale=1.0):
    """p, r of `shape` carved from larger buffers at element offsets `offsets` (off the 16-byte grid when non-zero)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    n = int(np.prod(shape))
    out = []
    for off in offsets:
        base = torch.randn(n + off, generator=g, device='cuda') * scale
        out.append(base.to(dtype)[off:].view(shape))
    return out


def check(preds, reals, got):
    got = got.cpu().numpy()
    row = 0
    for p, r in zip(preds, reals):
        rows = 1 if p.dim() == 1 else p.shape[0]
        pc, rc = p.contiguous(), r.contiguous()                          # the exact sums do not depend on the order of the elements
        want = lo.exact_moments(pc, rc)
        bound = lo.moments_bound(pc, rc)
        assert lo.moments_agree(got[row:row + rows], want, bound), (tuple(p.shape), p.dtype, got[row:row + rows], want)
        row += rows
    assert row == got.shape[0]


# long rows: one aligned and one mismatched layout; short rows: every offset pair
SHAPE_CASES = [(rows, row_len, off) for rows, row_len in [(1, 1), (64, 1), (5, 3), (64, 1000), (1, 16384), (2, 16385)]
               for off in [(0, 0), (1, 1), (3, 3), (1, 2), (0, 3)]] + [(3, 2 ** 20 + 3, (0, 0)), (3, 2 ** 20 + 3, (1, 2))]


@pytest.mark.parametrize('dtype', DTYPES, ids=['fp32', 'fp16', 'bf16'])
@pytest.mark.parametrize('rows,row_len,offsets', SHAPE_CASES)
def test_kernel_vs_oracle_shapes_and_offsets(dtype, rows, row_len, offsets):
    from ppq_b200.measure import paired_moments
    p, r = rand_pair((rows, row_len), dtype, rows * 131 + row_len + sum(offsets), offsets)
    got = paired_moments([p], [r])
    check([p], [r], got)
    again = paired_moments([p], [r])
    assert torch.equal(got.view(torch.int64), again.view(torch.int64))


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_kernel_row_above_2_pow_24(dtype):
    from ppq_b200.measure import paired_moments
    p, r = rand_pair((2 ** 24 + 5,), dtype, 24, (1, 1))
    got = paired_moments([p], [r])
    check([p], [r], got)


@pytest.mark.parametrize('dtype', DTYPES, ids=['fp32', 'fp16', 'bf16'])
def test_kernel_channels_last_1d_and_many_pairs(dtype):
    from ppq_b200.measure import paired_moments
    rng = np.random.default_rng(1)
    preds, reals = [], []
    for k in range(300):
        kind = k % 4
        if kind == 0: shape = (int(rng.integers(1, 9)), int(rng.integers(1, 3000)))
        elif kind == 1: shape = (int(rng.integers(1, 5)), 3, int(rng.integers(1, 20)), int(rng.integers(1, 20)))
        elif kind == 2: shape = (int(rng.integers(1, 70000)),)
        else: shape = (2, 8, 5, 7)
        p, r = rand_pair(shape, dtype, 1000 + k, (k % 3, k % 3))
        if kind == 3: p, r = p.contiguous(memory_format=torch.channels_last), r.contiguous(memory_format=torch.channels_last)
        preds.append(p); reals.append(r)
    got = paired_moments(preds, reals)
    check(preds, reals, got)
    assert torch.equal(got.view(torch.int64), paired_moments(preds, reals).view(torch.int64))


@pytest.mark.parametrize('dtype', DTYPES, ids=['fp32', 'fp16', 'bf16'])
def test_kernel_special_values_and_zero_rows(dtype):
    from ppq_b200.measure import paired_moments
    p, r = rand_pair((8, 5000), dtype, 7)
    p, r = p.clone(), r.clone()
    p[0] = 0; r[0] = 0                                                   # all-zero row
    r[1] = 0                                                             # zero reference
    p[2, 17] = float('nan')
    p[3, 4000] = float('inf')
    p[4, 10] = float('inf'); r[4, 10] = float('inf')                     # inf - inf
    r[5, 123] = float('-inf')
    p[6, 9] = float('inf'); r[6, 9] = 0                                  # inf * 0
    p[7] = r[7]                                                          # identical rows
    got = paired_moments([p], [r])
    check([p], [r], got)
    g = got.cpu().numpy()
    assert (g[0] == 0).all() and g[7, 0] == 0 and np.isnan(g[4, 0]) and np.isnan(g[6, 3])


def test_kernel_empty_table_and_malformed_table():
    from ppq_b200.ffi import extension
    from ppq_b200.measure import paired_moments
    ext = extension()
    out = torch.full((3, 4), 7.0, dtype=torch.float64, device='cuda')
    ws = torch.empty(64, dtype=torch.uint8, device='cuda')
    ext.Multi_Paired_Moments(torch.empty(0, 5, dtype=torch.int64, device='cuda'), 0, torch.float32, out, ws)
    assert paired_moments([], []).shape == (0, 4)
    p = torch.ones(2, 8, device='cuda')
    bad = torch.tensor([[p.data_ptr(), p.data_ptr(), 2, 8, 2]], dtype=torch.int64, device='cuda')     # rows 2..3 of a 3-row result
    ws = torch.empty(ext.Multi_Paired_Moments_Workspace_Bytes(3, 16), dtype=torch.uint8, device='cuda')
    ext.Multi_Paired_Moments(bad, 16, torch.float32, out, ws)
    assert torch.isnan(out).all()
    good = torch.tensor([[p.data_ptr(), p.data_ptr(), 2, 8, 1]], dtype=torch.int64, device='cuda')
    out.fill_(7.0)
    ext.Multi_Paired_Moments(good, 16, torch.float32, out, ws)
    assert out[0].eq(7.0).all() and out[1:].cpu().tolist() == [[0.0, 8.0, 8.0, 8.0]] * 2
    with pytest.raises(RuntimeError, match='too small'):
        ext.Multi_Paired_Moments(good, 10 ** 6, torch.float32, out, ws)


@pytest.mark.parametrize('dtype', DTYPES, ids=['fp32', 'fp16', 'bf16'])
def test_kernel_is_bit_identical_under_cuda_graph_replay(dtype):
    from ppq_b200.ffi import extension
    from ppq_b200.measure import paired_moments
    ext = extension()
    pairs = [rand_pair((32, 70001), dtype, 3, (1, 1)), rand_pair((32, 1000), dtype, 4, (0, 0)), rand_pair((4, 3), dtype, 5, (1, 2))]
    preds, reals = [p for p, _ in pairs], [r for _, r in pairs]
    eager = paired_moments(preds, reals)
    rows = [(p.data_ptr(), r.data_ptr(), p.shape[0], p[0].numel(), row0) for (p, r), row0 in zip(pairs, (0, 32, 64))]
    descs = torch.tensor(rows, dtype=torch.int64, device='cuda')
    elems = sum(p.numel() for p in preds)
    out = torch.zeros(68, 4, dtype=torch.float64, device='cuda')
    ws = torch.empty(ext.Multi_Paired_Moments_Workspace_Bytes(68, elems), dtype=torch.uint8, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ext.Multi_Paired_Moments(descs, elems, dtype, out, ws)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ext.Multi_Paired_Moments(descs, elems, dtype, out, ws)
    replays = []
    for _ in range(2):
        out.zero_(); graph.replay(); torch.cuda.synchronize(); replays.append(out.clone())
    for rep in replays: assert torch.equal(rep.view(torch.int64), eager.view(torch.int64))


# ---------------------------------------------------------------- layerwise_error_analyse
class TwoHeads(torch.nn.Module):
    """Two outputs of different shapes, as a detector returns several heads."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(11)
        self.stem = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.act = torch.nn.ReLU()
        self.head_a = torch.nn.Conv2d(8, 4, 1)
        self.pool = torch.nn.AdaptiveAvgPool2d(1)
        self.flat = torch.nn.Flatten(1)
        self.head_b = torch.nn.Linear(8, 10)
        with torch.no_grad():
            for p in self.parameters(): p.copy_(torch.randn(p.shape, generator=g) * 0.3)

    def forward(self, x):
        y = self.act(self.stem(x))
        return self.head_a(y), self.head_b(self.flat(self.pool(y)))


def calibrated(name, dtype=torch.float32, batches=8, batch=4):
    from ppq_b200.executor import TorchExecutor, calibrate_arena
    if name == 'twoheads':
        model = TwoHeads()
        data = [np.random.RandomState(5 + k).rand(batch, 3, 16, 16).astype(np.float32) for k in range(batches)]
    else:
        spec = netspec.SPECS[name]
        model = netspec.SpecNet(spec, netspec.make_params(spec, 3))
        data = netspec.make_data(name, 4, batches, batch)
    model = model.cuda().to(dtype)
    xs = [torch.from_numpy(x).cuda().to(dtype) for x in data]
    ex = TorchExecutor(model, xs[0], fuse_bn=False)
    ex.quantize_parameters()
    calibrate_arena(ex, xs, method='kl', half_inputs=dtype != torch.float32)
    ex.align_quantization()
    ex.bake_parameters()
    return ex, xs


def snapshot(ex):
    def bits(t):
        return None if t is None else t.detach().reshape(-1).clone().view(torch.int16 if t.element_size() == 2 else torch.int32)
    rows = []
    for n, op in ex.quantable_operations():
        for c in ex._configs_of(op): rows.append((n, c.state, bits(c._scale) if c._scale is not None else None, bits(c._offset) if c._offset is not None else None))
        if op.weight_cfg is not None: rows.append((n, bits(op.module.weight.data), bits(op.stored_weight)))
    return rows


def same_snapshot(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert len(x) == len(y) and x[0] == y[0]
        for u, v in zip(x[1:], y[1:]):
            if isinstance(u, torch.Tensor) or isinstance(v, torch.Tensor): assert u is not None and v is not None and torch.equal(u, v), x[0]
            else: assert u == v, x[0]


def close(got, want, method, rel=1e-5):
    assert list(got) == list(want)
    for n in want:
        g, w = got[n], want[n]
        tol = rel * abs(w) + (2e-6 if method == 'cosine' else 1e-12)
        assert abs(g - w) <= tol, (n, method, g, w)


@pytest.mark.parametrize('name', ['tinyres', 'tinycat', 'twoheads'])
@pytest.mark.parametrize('method', ['snr', 'mse', 'cosine'])
def test_layerwise_equals_the_restated_reference_loop(name, method):
    """Same keys in the same order; values within the difference of fp32 torch sums and exact sums (1e-5 relative: rows of at most a few
    thousand elements summed in fp32, then the mean of a 4-sample batch)."""
    from ppq_b200.executor import layerwise_error_analyse
    ex, xs = calibrated(name)
    before = snapshot(ex)
    for steps in (8, 1):
        want = lo.reference_layerwise(ex, xs, method=method, steps=steps)
        got = layerwise_error_analyse(ex, xs, method=method, steps=steps)
        close(got, want, method)
        assert all(np.isfinite(v) for v in got.values())
    same_snapshot(before, snapshot(ex))


def test_layerwise_counts_forwards_and_reads_steps_plus_one_batches():
    from ppq_b200.executor import COMPUTING_OP, layerwise_error_analyse
    ex, xs = calibrated('tinyres')
    K = sum(op.kind in COMPUTING_OP for _, op in ex.quantable_operations())
    assert K == 5
    calls = []
    h = ex.model.register_forward_hook(lambda m, a, o: calls.append(a[0].data_ptr()))
    try:
        for steps, seen in ((8, 8), (1, 2), (0, 1), (20, 8)):
            calls.clear()
            layerwise_error_analyse(ex, iter(xs), steps=steps)                    # a one-shot iterator is enough: the loop is batch-outer
            assert len(calls) == (K + 1) * seen, (steps, len(calls))
            assert calls == [x.data_ptr() for x in xs[:seen] for _ in range(K + 1)]
    finally:
        h.remove()


def test_layerwise_interested_outputs_by_operation_name():
    from ppq_b200.executor import layerwise_error_analyse
    ex, xs = calibrated('tinyres')
    for outs in (['conv4#0'], ['add1#0', 'fc#0'], 'relu1#0'):
        want = lo.reference_layerwise(ex, xs, interested_outputs=outs, method='snr', steps=3)
        got = layerwise_error_analyse(ex, xs, interested_outputs=outs, method='snr', steps=3)
        close(got, want, 'snr')
    with pytest.raises(KeyError):
        layerwise_error_analyse(ex, xs, interested_outputs=['nope'])


def test_layerwise_bf16_network_is_measured_on_the_exact_upcasts():
    """The reference measures a bf16 output in bf16 arithmetic (2^-8 relative per sum); ours is the exact value on the upcast: it equals the
    restated loop fed with the upcast outputs within fp32 accuracy, and the bf16-arithmetic loop within bf16 accuracy."""
    from ppq_b200.executor import layerwise_error_analyse
    ex, xs = calibrated('tinyres', torch.bfloat16)
    before = snapshot(ex)
    got = layerwise_error_analyse(ex, xs, method='snr')
    fwd = ex.forward

    def upcast(x, **kw):
        out = fwd(x, **kw)
        return out.float() if isinstance(out, torch.Tensor) else out
    ex.forward = upcast
    try:
        want = lo.reference_layerwise(ex, xs, method='snr')
    finally:
        del ex.forward
    close(got, want, 'snr')
    close(got, lo.reference_layerwise(ex, xs, method='snr'), 'snr', rel=5e-2)
    same_snapshot(before, snapshot(ex))


def test_layerwise_leaves_state_and_weights_untouched_when_a_batch_raises():
    from ppq_b200.executor import layerwise_error_analyse
    ex, xs = calibrated('tinycat')
    before = snapshot(ex)

    def batches():
        yield xs[0]
        yield xs[1]
        raise RuntimeError('broken loader')
    with pytest.raises(RuntimeError, match='broken loader'):
        layerwise_error_analyse(ex, batches())
    same_snapshot(before, snapshot(ex))
    assert ex._dequantized is None and ex._only is None
    close(layerwise_error_analyse(ex, xs, steps=2), lo.reference_layerwise(ex, xs, steps=2), 'snr')


# ---------------------------------------------------------------- against the reference function's values (tests/golden/layerwise_ref.npz)
@pytest.mark.parametrize('net', ['tinyres', 'tinycat'])
def test_layerwise_agrees_with_the_reference_fixture(net):
    """The reference's layerwise_error_analyse ran on the CPU on its own minmax-quantised graph.  Here: the same network on our executor with
    the fixture's scales and offsets loaded into the configs, aligned and baked as upstream.  Every value agrees within 1e-3 relative; what
    differs is the convolution arithmetic (cuDNN against the CPU) of the activations, and the measure's summation (exact here, fp32 there)."""
    import json
    import os
    from ppq_b200.executor import TorchExecutor, calibrate_arena, layerwise_error_analyse
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'layerwise_ref.npz'))
    meta = json.loads(bytes(z['meta']).decode())
    spec = netspec.SPECS[net]
    xs = [torch.from_numpy(x).cuda() for x in netspec.make_data(net, meta['data_seed'], meta['steps'], meta['batch'])]
    ex = TorchExecutor(netspec.SpecNet(spec, netspec.make_params(spec, meta['param_seed'])).cuda(), xs[0], fuse_bn=False)
    ex.quantize_parameters()
    calibrate_arena(ex, xs, method='minmax')
    ours = {}
    ops = dict(ex.quantable_operations())
    for o in spec:
        op = ops[o['name'] + '#0']
        for i, v in enumerate(o['inputs']): ours[(o['name'], v)] = op.input_cfgs[i]
        ours[(o['name'], o['out'])] = op.output_cfg
    loaded = 0
    for r in meta['nets'][net]['final']:
        if r['var'].endswith(('.w', '.b')) or r['dominator'] is not None or r['state'] not in ('ACTIVATED', 'PASSIVE'): continue
        c = ours[(r['op'], r['var'])]
        if c._scale is None: continue                                   # a config our calibration does not own (the alignment sets it)
        c._scale = torch.from_numpy(z[r['scale']]).cuda().reshape(c._scale.shape)
        c._offset = torch.from_numpy(z[r['offset']]).cuda().reshape(c._offset.shape)
        loaded += 1
    assert loaded >= 4
    ex.align_quantization()
    ex.bake_parameters()
    for run in meta['nets'][net]['runs']:
        got = layerwise_error_analyse(ex, xs[:run['batches']], method=run['method'], steps=run['steps'])
        assert list(got) == [n + '#0' for n in run['ops']]
        want = z[run['values']]
        rel = np.abs(np.array(list(got.values())) - want) / np.abs(want)
        assert (rel <= 1e-3).all(), (net, run['method'], run['steps'], list(got.values()), want.tolist())
