"""The post-LN BERT encoder block (tests/netspec_encoder.py) through ppq_b200's executor on the GPU: MatMul with two activation inputs,
Reshape / Transpose, Softmax, LayerNorm, Gemm -> Gelu.

  * both calibration flows (RuntimeCalibrationPass with the per-observer collectors, calibrate_arena with its multi-tensor launches, deferred
    True and 'auto', CUDA graphs for kl / minmax / mse) give the fixture's observed set, states and dominators;
  * every scale / offset equals the oracle chain applied to the GPU's own observed activations, bit for bit, and the two flows agree bit for bit;
  * a bf16 copy of the network calibrates through the half-precision tables to the oracle chain on the exact upcasts;
  * the scales agree with the reference's CPU-path fixture (tests/golden/graph_pipeline_encoder.npz) within DESIGN.md §2 deviation 5: cuBLAS vs
    CPU matmul rounding, a KL / MSE search that may move by one candidate;
  * after align_quantization() and bake_parameters() the configs match the fixture's final stage and every baked Gemm weight is the oracle's
    per-channel fake-quant of the fp32 weight;
  * graphwise_error_analyse and layerwise_error_analyse report every MatMul and Gemm with finite values and leave configs and weights alone.
"""
import json

import numpy as np
import pytest
import torch

import netspec_encoder as enc
from conftest import load_golden
from test_gpu_calibration_configs import CONFIGS, assert_same, expected

pytestmark = pytest.mark.gpu
METHODS = ['kl', 'minmax', 'percentile', 'mse']


@pytest.fixture(scope='module')
def env():
    if not torch.cuda.is_available(): pytest.skip('no CUDA device')
    torch.backends.cudnn.deterministic = True
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    z = load_golden('graph_pipeline_encoder.npz')
    meta = json.loads(bytes(z['meta']).decode())
    params = enc.make_params(enc.ENCODER, meta['param_seed'])
    data = enc.make_data(meta['data_seed'], meta['steps'])
    return dict(z=z, meta=meta, params=params, data=data)


def executor(env, dtype=torch.float32):
    from ppq_b200.executor import TorchExecutor
    model = enc.EncoderNet(enc.ENCODER, env['params']).cuda().to(dtype)
    batches = [torch.from_numpy(x).cuda().to(dtype) for x in env['data']]
    ex = TorchExecutor(model, batches[0], fuse_bn=False)
    ex.quantize_parameters()
    return ex, batches


def rows_of(ex):
    """fixture (op, var) -> our config."""
    ops, out = dict(ex.quantable_operations()), {}
    for o in enc.ENCODER:
        op = ops[o['name'] + '#0']
        for i, v in enumerate(o['inputs']): out[(o['name'], v)] = op.input_cfgs[i]
        out[(o['name'], o['out'])] = op.output_cfg
        if op.weight_cfg is not None: out[(o['name'], o['name'] + '.w')] = op.weight_cfg
    return out


def check_topology(ex, rows, tag):
    """States and dominators of every non-FP32 fixture row (bias, Reshape shape, LayerNorm gamma / beta are FP32 there and have no config here)."""
    ours = rows_of(ex)
    assert len([r for r in rows if r['state'] != 'FP32']) == len(ours), tag
    for r in rows:
        if r['state'] == 'FP32': continue
        c = ours[(r['op'], r['var'])]
        assert c.state.name == r['state'], (tag, r['op'], r['var'], c.state, r['state'])
        if r['dominator'] is not None:
            dop, dvar = r['dominator'].split('|')
            assert c.dominated_by is ours[(dop, dvar)], (tag, r['op'], r['var'])
        else:
            assert c.dominated_by is c, (tag, r['op'], r['var'])


def observed_tensors(env, dtype=torch.float32):
    """Per observed slot, the fp32 host copies (exact upcasts) of what the observers see, batch by batch: a fresh executor's collect list."""
    ex, batches = executor(env, dtype)
    per_slot = None
    for x in batches:
        _, ts = ex.forward(x, collect=True)
        if per_slot is None: per_slot = [[] for _ in ts]
        for k, t in enumerate(ts): per_slot[k].append(t.float().cpu().numpy().copy())
    return per_slot


_want = {}


def oracle_scales(env, oracle, method, dtype=torch.float32):
    key = (method, dtype)
    if key not in _want:
        _want[key] = [expected(oracle, method, CONFIGS['int8_sym'], xs) for xs in observed_tensors(env, dtype)]
    return _want[key]


def check_oracle(ex, want, tag):
    cfgs = ex.observed_configs_all()
    assert len(cfgs) == len(want) == 17, tag
    for k, (c, (ws, wo)) in enumerate(zip(cfgs, want)):
        assert_same(c.scale, ws, f'{tag} slot {k} scale')
        assert_same(c.offset, wo, f'{tag} slot {k} offset')


def snapshot(ex):
    out = {}
    for name, op in ex.quantable_operations():
        for i, c in enumerate(op.input_cfgs + ([op.weight_cfg] if op.weight_cfg is not None else []) + [op.output_cfg]):
            out[(name, i)] = (c.state, None if c.scale is None else c.scale.detach().clone(), None if c.offset is None else c.offset.detach().clone())
        if op.kind in ('Gemm', 'LayerNormalization'): out[(name, 'w')] = op.module.weight.data.clone()
    return out


def same_snapshot(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
            continue
        assert a[k][0] == b[k][0], k
        for x, y in zip(a[k][1:], b[k][1:]):
            assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), k


@pytest.mark.parametrize('method', METHODS)
def test_both_flows_reproduce_the_fixture_topology_and_the_oracle(env, oracle, method):
    from ppq_b200.calibration import RuntimeCalibrationPass
    from ppq_b200.executor import calibrate_arena
    rows = env['meta']['methods'][method]['calibrated']
    want = oracle_scales(env, oracle, method)
    hook, batches = executor(env)
    RuntimeCalibrationPass(method=method).optimize(hook, batches, hook, calib_steps=len(batches))
    check_topology(hook, rows, f'hooks/{method}')
    check_oracle(hook, want, f'hooks/{method}')
    flows = [('auto', False), (True, False)] + ([] if method == 'percentile' else [('auto', True)])
    for deferred, graphs in flows:
        ex, batches = executor(env)
        calibrate_arena(ex, batches, method=method, deferred=deferred, graphs=graphs)
        tag = f'arena(deferred={deferred}, graphs={graphs})/{method}'
        check_topology(ex, rows, tag)
        check_oracle(ex, want, tag)
        for a, b in zip(hook.observed_configs_all(), ex.observed_configs_all()):       # the two flows: bit-identical scales and offsets
            assert torch.equal(a.scale.cpu(), b.scale.cpu()) and torch.equal(a.offset.cpu(), b.offset.cpu()), tag


@pytest.mark.parametrize('method', ['kl', 'percentile'])
def test_bf16_encoder_calibrates_to_the_oracle_on_the_upcasts(env, oracle, method):
    from ppq_b200.calibration import RuntimeCalibrationPass
    from ppq_b200.executor import calibrate_arena
    want = oracle_scales(env, oracle, method, torch.bfloat16)
    ex, batches = executor(env, torch.bfloat16)
    calibrate_arena(ex, batches, method=method, half_inputs=True)
    check_topology(ex, env['meta']['methods'][method]['calibrated'], f'bf16/{method}')
    check_oracle(ex, want, f'bf16 arena/{method}')
    hook, batches = executor(env, torch.bfloat16)
    RuntimeCalibrationPass(method=method).optimize(hook, batches, hook, calib_steps=len(batches))
    check_oracle(hook, want, f'bf16 hooks/{method}')


@pytest.mark.parametrize('method', METHODS)
def test_scales_agree_with_the_cpu_path_fixture(env, method):
    """DESIGN.md §2 deviation 5: the fixture is the reference's CPU path (torch.histc bins, int()-truncated kthvalue ranks, CPU matmuls).
    Weights: bit for bit.  The network input's min / max: bit for bit.  Other activations: min-max and percentile scales within 1e-4 relative
    (CPU vs cuBLAS / device LayerNorm and Softmax rounding), KL and MSE within [0.8, 1.25] (the search may settle one candidate away)."""
    from ppq_b200.executor import calibrate_arena
    z, entry = env['z'], env['meta']['methods'][method]
    ex, batches = executor(env)
    calibrate_arena(ex, batches, method=method)
    ours = rows_of(ex)
    for r in entry['calibrated']:
        if r['state'] != 'ACTIVATED': continue
        got, ref = ours[(r['op'], r['var'])].scale.float().cpu().numpy().reshape(-1), z[r['scale']].reshape(-1)
        tag = (method, r['op'], r['var'], got, ref)
        if r['var'].endswith('.w') or (r['var'] == 'x' and method == 'minmax'):
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), tag
        elif method in ('minmax', 'percentile'):
            np.testing.assert_allclose(got, ref, rtol=1e-4, err_msg=str(tag))
        else:
            assert np.all((got / ref >= 0.8) & (got / ref <= 1.25)), tag


@pytest.mark.parametrize('method', ['kl', 'minmax'])
def test_alignment_and_baking(env, oracle, method):
    """align_quantization(): the two residual Adds ('Align to Large', force overlap) give the fixture's final states and dominators.
    bake_parameters(): every Gemm weight is the oracle's per-channel fake-quant of its fp32 weight, bit for bit; LayerNorm gamma / beta
    are untouched."""
    from ppq_b200.executor import calibrate_arena
    ex, batches = executor(env)
    calibrate_arena(ex, batches, method=method)
    fp32 = {n: op.module.weight.data.clone() for n, op in ex.quantable_operations() if op.kind in ('Gemm', 'LayerNormalization')}
    ex.align_quantization()
    ex.bake_parameters()
    check_topology(ex, env['meta']['methods'][method]['final'], f'final/{method}')
    for name, op in ex.quantable_operations():
        if op.kind == 'LayerNormalization':
            assert torch.equal(op.module.weight.data, fp32[name]), name
        if op.kind != 'Gemm': continue
        w = fp32[name].cpu().numpy()
        want = oracle.linear_quant_c(w, op.weight_cfg.scale.cpu().numpy(), op.weight_cfg.offset.cpu().numpy(), 0, -128, 127)
        assert_same(op.module.weight.data, want, f'baked {name}')
    out = ex.forward(batches[0])
    assert out.shape == batches[0].shape and bool(torch.isfinite(out).all())


def test_error_analyses_report_every_matmul_and_gemm(env):
    from ppq_b200.executor import calibrate_arena, graphwise_error_analyse, layerwise_error_analyse
    ex, batches = executor(env)
    calibrate_arena(ex, batches, method='kl')
    ex.align_quantization(); ex.bake_parameters()
    before = snapshot(ex)
    computing = [n for n, op in ex.quantable_operations() if op.kind in ('MatMul', 'Gemm')]
    assert len(computing) == 8
    full = graphwise_error_analyse(ex, batches)
    assert list(full) == [n for n, _ in ex.quantable_operations()] and all(np.isfinite(v) for v in full.values()), full
    same_snapshot(before, snapshot(ex))
    sampled = graphwise_error_analyse(ex, batches, fetchs=4096)
    assert list(sampled) == computing and all(np.isfinite(v) for v in sampled.values()), sampled
    same_snapshot(before, snapshot(ex))
    for method in ('snr', 'cosine'):
        lw = layerwise_error_analyse(ex, batches, method=method, steps=3)
        assert list(lw) == computing and all(np.isfinite(v) for v in lw.values()), (method, lw)
        same_snapshot(before, snapshot(ex))
