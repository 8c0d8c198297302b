"""Encoder-level parity on the CPU: tests/golden/graph_pipeline_encoder.npz was produced by the UNMODIFIED reference pipeline (TRT_INT8
quantizer's own pass list) on a one-block post-LN BERT encoder built programmatically (tests/netspec_encoder.py,
tests/golden/make_encoder_golden.py).  Checked here:
  * oracle/cpu_pipeline.py's CPU restatement of the reference pipeline, with the transformer kinds of tests/encoder_pipeline.py, reproduces it
    bit for bit: observed set, dominators, states, scales / offsets of all four observers after
    calibration and after alignment / baking, the baked Gemm weights and the quantised output;
  * ppq_b200.executor's topology passes give the same states / dominators / observed set (MatMul with two activation inputs, passive
    Reshape / Transpose, LayerNorm with FP32 gamma / beta, Gemm -> Gelu fusion);
  * a network written with plain nn.LayerNorm / torch.matmul / .view / .transpose gets exactly the configs it got before the new kinds
    existed (they are opt-in);
  * where the reference checkout is present, the fixture is regenerated live and must not have drifted.
"""
import json
import sys

import numpy as np
import pytest
import torch

import netspec_encoder as enc
import refppq
from conftest import load_golden

FIXTURE = 'graph_pipeline_encoder.npz'
METHODS = ('kl', 'minmax', 'percentile', 'mse')


@pytest.fixture(scope='module')
def fx():
    z = load_golden(FIXTURE)
    return z, json.loads(bytes(z['meta']).decode())


def labels(spec):
    """fixture (op, var) -> (operation name, 'in<i>' / 'out' / 'w') as the CPU pipeline and ppq_b200.executor name them."""
    m = {}
    for o in spec:
        for i, v in enumerate(o['inputs']): m[(o['name'], v)] = (f"{o['name']}#0", f'in{i}')
        m[(o['name'], o['out'])] = (f"{o['name']}#0", 'out')
        if o['op'] == 'Gemm': m[(o['name'], o['name'] + '.w')] = (f"{o['name']}#0", 'w')
    return m


def net_and_data(meta):
    spec = enc.ENCODER
    params = enc.make_params(spec, meta['param_seed'])
    data = [torch.from_numpy(x) for x in enc.make_data(meta['data_seed'], meta['steps'])]
    return spec, params, data


def bits(a):
    return np.asarray(a, dtype=np.float32).reshape(-1).view(np.uint32)


def test_fixture_covers_the_encoder_topology(fx):
    """What the reference's dispatcher and QuantizeFusionPass do with the transformer operators (the rules ppq_b200.executor mirrors)."""
    _, meta = fx
    rows = {(r['op'], r['var']): r for r in meta['methods']['kl']['calibrated']}
    for name in ('q_heads', 'k_heads', 'v_heads', 'ctx_flat'):
        assert rows[(name, name + '.shape')]['state'] == 'FP32'                         # Reshape's constant shape: an FP32 config, never observed
        assert rows[(name, name + '.o')]['state'] == 'OVERLAPPED'                       # passive
    for name in ('ln1', 'ln2'):
        assert rows[(name, name + '.gamma')]['state'] == rows[(name, name + '.beta')]['state'] == 'FP32'
        assert rows[(name, name + '.o')]['state'] == 'ACTIVATED'
    assert rows[('scores', 'scores.o')]['state'] == 'ACTIVATED' and rows[('scores', 'k_t.o')]['dominator'] == 'k|k.o'   # MatMul: two activation inputs
    assert not any(r['var'].startswith(('scores.w', 'context.w')) for r in rows.values())
    assert rows[('ffn1', 'ffn1.o')]['dominator'] == 'gelu|gelu.o'                       # Gemm -> Gelu fusion
    assert rows[('probs', 'probs.o')]['state'] == 'ACTIVATED'                           # the Softmax input (scores.o) and output are both observed


@pytest.mark.parametrize('method', METHODS)
def test_cpu_pipeline_port_reproduces_the_reference_encoder(fx, method):
    from encoder_pipeline import EncoderCpuPipeline
    z, meta = fx
    torch.set_num_threads(1)
    spec, params, data = net_and_data(meta)
    lab = labels(spec)
    pipe = EncoderCpuPipeline(enc.EncoderNet(spec, params), data[0])
    port = {}
    for op in pipe.ops:
        for i, c in enumerate(op.ins): port[(op.name, f'in{i}')] = c
        port[(op.name, 'out')] = op.out
        if op.w is not None: port[(op.name, 'w')] = op.w
    entry = meta['methods'][method]
    want = [lab[(r['op'], r['var'])] for r in entry['calibrated'] if r['state'] == 'ACTIVATED' and not r['var'].endswith('.w')]
    got = [tuple(label.split('|')) for label, _ in pipe.observed()]
    assert got == want
    pipe.quantize_parameters()
    pipe.calibrate(data, method)

    def check(stage):
        for r in entry[stage]:
            if r['state'] == 'FP32': continue                                  # bias, Reshape shape, LayerNorm gamma / beta
            c = port[lab[(r['op'], r['var'])]]
            assert c.state == r['state'], (stage, r['op'], r['var'], c.state, r['state'])
            if r['dominator'] is not None:
                dop, dvar = r['dominator'].split('|')
                assert c.root is port[lab[(dop, dvar)]], (stage, r['op'], r['var'])
            assert np.array_equal(bits(c.scale), bits(z[r['scale']])), (stage, r['op'], r['var'], c.scale, z[r['scale']])
            assert np.array_equal(bits(c.offset), bits(z[r['offset']]))
    check('calibrated')
    pipe.align(); pipe.bake()
    check('final')
    for o in spec:
        if o['op'] == 'Gemm':
            assert np.array_equal(bits(getattr(pipe.model, o['name']).weight.data.numpy()), bits(z[f"{method}.baked.{o['name']}.w"])), o['name']
    out = pipe.forward(data[0]).numpy()
    assert np.array_equal(bits(out), bits(z[f'{method}.output'])), np.abs(out - z[f'{method}.output']).max()


def test_executor_topology_matches_the_reference_passes(fx):
    """QuantizeFusionPass + QuantizeSimplifyPass as mirrored by ppq_b200.executor on the encoder (tracing runs on the CPU)."""
    from ppq_b200.executor import TorchExecutor
    _, meta = fx
    spec, params, data = net_and_data(meta)
    lab = labels(spec)
    ex = TorchExecutor(enc.EncoderNet(spec, params), data[0], fuse_bn=False)
    ours = {}
    for name, op in ex.quantable_operations():
        for i, c in enumerate(op.input_cfgs): ours[(name, f'in{i}')] = c
        ours[(name, 'out')] = op.output_cfg
        if op.weight_cfg is not None: ours[(name, 'w')] = op.weight_cfg
    assert {n: op.kind for n, op in ex.quantable_operations()} == {o['name'] + '#0': o['op'] for o in spec}
    rows = meta['methods']['kl']['calibrated']
    assert len([r for r in rows if r['state'] != 'FP32']) == len(ours)
    for r in rows:
        if r['state'] == 'FP32': continue
        c = ours[lab[(r['op'], r['var'])]]
        want = 'OVERLAPPED' if r['state'] == 'OVERLAPPED' else 'INITIAL'
        assert c.state.name == want, (r['op'], r['var'], c.state, r['state'])
        if r['dominator'] is not None:
            dop, dvar = r['dominator'].split('|')
            assert c.dominated_by is ours[lab[(dop, dvar)]], (r['op'], r['var'])
        else:
            assert c.dominated_by is c
    want = [ours[lab[(r['op'], r['var'])]] for r in rows if r['state'] == 'ACTIVATED' and not r['var'].endswith('.w')]
    got = ex.observed_configs()
    assert len(got) == len(want) and all(a is b for a, b in zip(got, want))
    for name, op in ex.quantable_operations():
        if op.kind in ('MatMul', 'LayerNormalization', 'Reshape', 'Transpose'): assert op.weight_cfg is None, name


class FunctionalBlock(torch.nn.Module):
    """The same attention written the way most torch code writes it: torch.matmul, .view / .transpose, a plain nn.LayerNorm."""

    def __init__(self, hidden=32, heads=4, seq=8):
        super().__init__()
        self.heads, self.seq, self.d = heads, seq, hidden // heads
        self.q, self.k, self.v, self.o = (torch.nn.Linear(hidden, hidden) for _ in range(4))
        self.softmax, self.ln, self.ffn1, self.gelu, self.ffn2 = (torch.nn.Softmax(-1), torch.nn.LayerNorm(hidden), torch.nn.Linear(hidden, 64),
                                                                  torch.nn.GELU(), torch.nn.Linear(64, hidden))

    def forward(self, x):
        def heads(t): return t.view(-1, self.seq, self.heads, self.d).transpose(1, 2)
        p = self.softmax(torch.matmul(heads(self.q(x)), heads(self.k(x)).transpose(-1, -2)))
        c = torch.matmul(p, heads(self.v(x))).transpose(1, 2).reshape(x.shape)
        h = self.ln(self.o(c) + x)
        return self.ffn2(self.gelu(self.ffn1(h))) + h


def describe(ex):
    """Every config of every operation: (operation, kind, slot, state, dominator slot or None, weight channel axis or None), slots as
    'operation:in<i>' / ':weight' / ':out', then the observed configs in calibration order."""
    slot = {}
    for name, op in ex.quantable_operations():
        for i, c in enumerate(op.input_cfgs): slot[id(c)] = f'{name}:in{i}'
        if op.weight_cfg is not None: slot[id(op.weight_cfg)] = f'{name}:weight'
        slot[id(op.output_cfg)] = f'{name}:out'
    rows = []
    for name, op in ex.quantable_operations():
        for c in op.input_cfgs + ([op.weight_cfg] if op.weight_cfg is not None else []) + [op.output_cfg]:
            rows.append((name, op.kind, slot[id(c)], c.state.name, None if c.dominated_by is c else slot[id(c.dominated_by)],
                         c.channel_axis if c is op.weight_cfg else None))
    return rows + [('observed', tuple(slot[id(c)] for c in ex.observed_configs()))]


# describe() of FunctionalBlock, recorded with the executor as it was before MatMul / Reshape / Transpose / LayerNorm became operator kinds
FUNCTIONAL_CONFIGS = [
    ('q#0', 'Gemm', 'q#0:in0', 'INITIAL', None, None),
    ('q#0', 'Gemm', 'q#0:weight', 'INITIAL', None, 0),
    ('q#0', 'Gemm', 'q#0:out', 'INITIAL', None, None),
    ('k#0', 'Gemm', 'k#0:in0', 'INITIAL', None, None),
    ('k#0', 'Gemm', 'k#0:weight', 'INITIAL', None, 0),
    ('k#0', 'Gemm', 'k#0:out', 'INITIAL', None, None),
    ('softmax#0', 'Softmax', 'softmax#0:in0', 'INITIAL', None, None),
    ('softmax#0', 'Softmax', 'softmax#0:out', 'INITIAL', None, None),
    ('v#0', 'Gemm', 'v#0:in0', 'INITIAL', None, None),
    ('v#0', 'Gemm', 'v#0:weight', 'INITIAL', None, 0),
    ('v#0', 'Gemm', 'v#0:out', 'INITIAL', None, None),
    ('o#0', 'Gemm', 'o#0:in0', 'INITIAL', None, None),
    ('o#0', 'Gemm', 'o#0:weight', 'INITIAL', None, 0),
    ('o#0', 'Gemm', 'o#0:out', 'INITIAL', None, None),
    ('ffn1#0', 'Gemm', 'ffn1#0:in0', 'INITIAL', None, None),
    ('ffn1#0', 'Gemm', 'ffn1#0:weight', 'INITIAL', None, 0),
    ('ffn1#0', 'Gemm', 'ffn1#0:out', 'OVERLAPPED', 'gelu#0:out', None),
    ('gelu#0', 'Gelu', 'gelu#0:in0', 'OVERLAPPED', 'gelu#0:out', None),
    ('gelu#0', 'Gelu', 'gelu#0:out', 'INITIAL', None, None),
    ('ffn2#0', 'Gemm', 'ffn2#0:in0', 'OVERLAPPED', 'gelu#0:out', None),
    ('ffn2#0', 'Gemm', 'ffn2#0:weight', 'INITIAL', None, 0),
    ('ffn2#0', 'Gemm', 'ffn2#0:out', 'INITIAL', None, None),
    ('observed', ('q#0:in0', 'q#0:out', 'k#0:in0', 'k#0:out', 'softmax#0:in0', 'softmax#0:out', 'v#0:in0', 'v#0:out', 'o#0:in0', 'o#0:out',
                  'ffn1#0:in0', 'gelu#0:out', 'ffn2#0:out')),
]


def test_plain_layernorm_and_functional_attention_keep_their_configs():
    """The new kinds are opt-in: a network with nn.LayerNorm, torch.matmul and view / transpose gets exactly the configs it got before."""
    from ppq_b200.executor import TorchExecutor
    torch.manual_seed(0)
    ex = TorchExecutor(FunctionalBlock(), torch.randn(32, 32), fuse_bn=False)
    assert describe(ex) == FUNCTIONAL_CONFIGS


@pytest.fixture
def reference():
    """The reference package.  Importing it puts stand-in `onnx` modules into sys.modules; the ones it added are taken out again afterwards,
    so that a later `import torchvision` (which probes for onnx) does not find a module without a spec."""
    if refppq.root() != '/root/reference':
        pytest.skip('the read-only reference checkout is only present in the build container')
    stand_ins = lambda: {m for m in sys.modules if m == 'onnx' or m.startswith('onnx.')}   # noqa: E731
    before = stand_ins()
    yield refppq.load()
    for m in stand_ins() - before: del sys.modules[m]


def test_fixture_is_what_the_reference_produces_today(fx, reference):
    ppq = reference
    z, meta = fx
    torch.set_num_threads(1)
    spec = enc.ENCODER
    params = enc.make_params(spec, meta['param_seed'])
    data = enc.make_data(meta['data_seed'], meta['steps'])
    res = enc.run_reference_pipeline(ppq, spec, params, data, 'kl')
    entry = meta['methods']['kl']
    assert res['passes'] == entry['passes']
    for stage in ('calibrated', 'final'):
        assert len(res[stage]) == len(entry[stage])
        for row, r in zip(res[stage], entry[stage]):
            assert (row['op'], row['var'], row['state'], row['dominator']) == (r['op'], r['var'], r['state'], r['dominator'])
            if row['scale'] is not None: assert np.array_equal(bits(row['scale']), bits(z[r['scale']]))
    assert np.array_equal(bits(res['output']), bits(z['kl.output']))
    for k, v in res['baked'].items(): assert np.array_equal(bits(v), bits(z[f'kl.baked.{k}'])), k
