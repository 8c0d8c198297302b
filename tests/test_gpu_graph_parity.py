"""Graph-level parity ON THE GPU with the REAL reference package (VERDICT r1 items 1 and 2, ADVICE r1 high):

  A. the unmodified reference pipeline (`ppq` from PPQ_REFERENCE_ROOT, TRT_INT8 quantizer's own pass list, TorchExecutor(device='cuda'), inside
     `with ENABLE_CUDA_KERNEL():`) gives IDENTICAL results -- every config's state / dominator / scale / offset, the baked weights, the
     quantised network output, bit for bit -- whether ppq.core.ffi serves the reference's own CUDA extension (compiled unmodified for
     sm_90a: oracle/_ref) or ppq_b200/_C.so installed by ppq_b200.install.install();
  B. the same with the device-resident observers swapped in (install(replace_observers=True)): the reference's RuntimeCalibrationPass keeps
     them for phase 2 (type identity, calibration.py:195), every activation config ends ACTIVATED with the same scale;
  C. ppq_b200's own executor + RuntimeCalibrationPass / calibrate_arena on the equivalent torch module reproduce those results;
  D. the GPU results agree with the committed CPU-path fixture (tests/golden/graph_pipeline.npz) to float tolerance (cuDNN vs CPU convs),
     weights and the network input bit for bit.

The reference pipeline runs where PPQ_REFERENCE_ROOT names an upstream checkout; its results on the GPU are stored in
tests/golden/ref_graph_runs.pkl.gz and replayed without one, so A and B then compare the stored runs, and our executor (C, the live
halves of A / B) is checked against them.  PPQ_RECORD_REFERENCE=<dir> (with the package and oracle/_ref) writes <dir>/ref_graph_runs.pkl.gz.
"""
import atexit
import gzip
import json
import os
import pickle

import numpy as np
import pytest
import torch

import netspec
import refppq
from conftest import GOLDEN, load_golden

pytestmark = pytest.mark.gpu
METHODS = ['kl', 'minmax', 'percentile', 'mse']
RUNS = os.path.join(GOLDEN, 'ref_graph_runs.pkl.gz')
_recorded, _stored = {}, []


def stored_run(key):
    """A reference pipeline run recorded on the GPU (tests/golden/ref_graph_runs.pkl.gz)."""
    if not _stored:
        with gzip.open(RUNS, 'rb') as f:
            _stored.append(pickle.load(f))
    assert key in _stored[0], f'no recorded reference run {key} in {RUNS}'
    return _stored[0][key]


def record_run(key, res):
    out_dir = os.environ.get('PPQ_RECORD_REFERENCE')
    if not out_dir: return
    if not _recorded:
        def write():
            os.makedirs(out_dir, exist_ok=True)
            with gzip.open(os.path.join(out_dir, 'ref_graph_runs.pkl.gz'), 'wb') as f:
                pickle.dump(_recorded, f, protocol=4)
        atexit.register(write)
    _recorded[key] = res


def make_env(fixture):
    if not torch.cuda.is_available(): pytest.skip('no CUDA device')
    ppq = refppq.load()
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    z = load_golden(fixture)
    meta = json.loads(bytes(z['meta']).decode())
    spec = netspec.SPECS[meta['net']]
    params = netspec.make_params(spec, meta['param_seed'])
    data = netspec.make_data(meta['net'], meta['data_seed'], meta['steps'], meta['batch'])
    from ppq_b200.ffi import extension
    return dict(ppq=ppq, z=z, meta=meta, spec=spec, params=params, data=data, ours=extension(), cache={}, fixture=fixture)


@pytest.fixture(scope='module')
def env():
    return make_env('graph_pipeline.npz')


@pytest.fixture(scope='module')
def env_cat():
    """The second graph: Concat ('Align to Output'), conv -> Sigmoid fusion, AveragePool, a max-pool whose producer has two consumers."""
    return make_env('graph_pipeline_tinycat.npz')


def bits(a):
    return np.asarray(a, dtype=np.float32).reshape(-1).view(np.uint32)


def reference_run(env, which, method):
    """The real reference pipeline on cuda with extension `which` in ('ref', 'ours', 'ours+observers'); cached per module run."""
    key = (which, method)
    if key in env['cache']: return env['cache'][key]
    name = f"{env['fixture']}:{which}:{method}"
    if env['ppq'] is None:
        env['cache'][key] = stored_run(name)
        return env['cache'][key]
    import ppq_b200.install as inst
    if which == 'ref':
        mod = refppq.reference_cuda_extension()
        if mod is None: pytest.skip('oracle/_ref/PPQ_Cuda_Impls_ref.so not built')
        with refppq.use_extension(mod):
            res = netspec.run_reference_pipeline(env['ppq'], env['spec'], env['params'], env['data'], method, device='cuda', cuda_kernel=True)
    else:
        inst.install(replace_observers=(which == 'ours+observers'))
        try:
            import ppq.core.ffi as ffi
            assert ffi.CUDA_COMPLIER.CUDA_EXTENSION is env['ours']
            res = netspec.run_reference_pipeline(env['ppq'], env['spec'], env['params'], env['data'], method, device='cuda', cuda_kernel=True)
        finally:
            inst.uninstall()
    record_run(name, res)
    env['cache'][key] = res
    return res


def assert_same(a, b, what):
    for stage in ('calibrated', 'final'):
        assert len(a[stage]) == len(b[stage])
        for ra, rb in zip(a[stage], b[stage]):
            tag = (what, stage, ra['op'], ra['var'])
            assert (ra['op'], ra['var'], ra['state'], ra['dominator']) == (rb['op'], rb['var'], rb['state'], rb['dominator']), tag
            for k in ('scale', 'offset'):
                assert (ra[k] is None) == (rb[k] is None), tag
                if ra[k] is not None: assert np.array_equal(bits(ra[k]), bits(rb[k])), tag + (k, ra[k], rb[k])
    for k in a['baked']: assert np.array_equal(bits(a['baked'][k]), bits(b['baked'][k])), (what, 'baked', k)
    assert np.array_equal(bits(a['output']), bits(b['output'])), (what, 'output', np.abs(a['output'] - b['output']).max())


@pytest.mark.parametrize('method', METHODS)
def test_reference_pipeline_is_identical_with_our_extension_installed(env, method):
    """A: same unmodified Python pipeline, two native extensions, identical results."""
    assert_same(reference_run(env, 'ref', method), reference_run(env, 'ours', method), f'ref-ext vs ours [{method}]')
    r = reference_run(env, 'ours', method)
    acts = [row for row in r['calibrated'] if not row['var'].endswith(('.w', '.b'))]
    assert all(row['state'] in ('ACTIVATED', 'OVERLAPPED') for row in acts) and sum(row['state'] == 'ACTIVATED' for row in acts) == 8
    from ppq_b200.executor import calibrate_arena
    ex, batches = our_executor(env)                                        # our kernels through our executor == the reference extension's run
    calibrate_arena(ex, batches, method=method)
    check_against(ex, env, reference_run(env, 'ref', method)['calibrated'], f'ref-ext vs our executor [{method}]')


@pytest.mark.parametrize('method', METHODS)
def test_reference_pipeline_with_device_resident_observers(env, method):
    """B (ADVICE r1 high): with the observers replaced the reference pass must still run phase 2 and activate every config."""
    a, b = reference_run(env, 'ours', method), reference_run(env, 'ours+observers', method)
    for row in b['calibrated']:
        if not row['var'].endswith('.b'): assert row['state'] in ('ACTIVATED', 'OVERLAPPED'), row
    assert_same(a, b, f'reference observers vs device-resident observers [{method}]')
    from ppq_b200.calibration import RuntimeCalibrationPass
    ex, batches = our_executor(env)                                        # our device-resident observers in our calibration pass
    RuntimeCalibrationPass(method=method).optimize(ex, batches, ex, calib_steps=len(batches))
    check_against(ex, env, b['calibrated'], f'device-resident observers, our pass [{method}]')


def our_executor(env):
    from ppq_b200.executor import TorchExecutor
    model = netspec.SpecNet(env['spec'], env['params']).cuda()
    batches = [torch.from_numpy(x).cuda() for x in env['data']]
    ex = TorchExecutor(model, batches[0], fuse_bn=False)
    ex.quantize_parameters()
    return ex, batches


def rows_of(ex, spec):
    """our configs keyed like the fixture rows: (op, var) -> config."""
    out = {}
    ops = dict(ex.quantable_operations())
    for o in spec:
        op = ops[o['name'] + '#0']
        for i, v in enumerate(o['inputs']): out[(o['name'], v)] = op.input_cfgs[i]
        out[(o['name'], o['out'])] = op.output_cfg
        if op.weight_cfg is not None: out[(o['name'], o['name'] + '.w')] = op.weight_cfg
    return out


def check_against(ex, env, want_rows, tag):
    ours = rows_of(ex, env['spec'])
    for r in want_rows:
        if r['state'] == 'FP32': continue
        c = ours[(r['op'], r['var'])]
        assert c.state.name == r['state'], (tag, r['op'], r['var'], c.state, r['state'])
        if r['dominator'] is not None:
            dop, dvar = r['dominator'].split('|')
            assert c.dominated_by is ours[(dop, dvar)], (tag, r['op'], r['var'])
        assert np.array_equal(bits(c.scale.cpu().numpy()), bits(r['scale'])), (tag, r['op'], r['var'], c.scale, r['scale'])
        assert np.array_equal(bits(c.offset.cpu().numpy()), bits(r['offset'])), (tag, r['op'], r['var'])


@pytest.mark.parametrize('flow,method', [('hooks', m) for m in METHODS] + [('arena', m) for m in METHODS] + [('arena-deferred', 'kl')])
def test_our_executor_reproduces_the_reference_pipeline(env, flow, method):
    """C: ppq_b200.executor (+ RuntimeCalibrationPass with the device-resident observers, or the arena calibrator: one multi-tensor launch
    per forward) on the equivalent torch module vs the real pipeline on the same GPU: same observed set, bit-identical scales, then the
    same aligned / baked / quantised forward."""
    from ppq_b200.calibration import RuntimeCalibrationPass
    from ppq_b200.executor import calibrate_arena
    want = reference_run(env, 'ours', method)
    ex, batches = our_executor(env)
    if flow == 'hooks':
        RuntimeCalibrationPass(method=method).optimize(ex, batches, ex, calib_steps=len(batches))
    else:
        calibrate_arena(ex, batches, method=method, deferred=(True if flow == 'arena-deferred' else 'auto'))
    check_against(ex, env, want['calibrated'], f'{flow}/{method}/calibrated')
    ex.align_quantization()
    ex.bake_parameters()
    check_against(ex, env, want['final'], f'{flow}/{method}/final')
    for o in env['spec']:
        if o['op'] in ('Conv', 'Gemm'):
            assert np.array_equal(bits(getattr(ex.model, o['name']).weight.data.cpu().numpy()), bits(want['baked'][o['name'] + '.w'])), o['name']
    out = ex.forward(batches[0]).cpu().numpy()
    assert np.array_equal(bits(out), bits(want['output'])), np.abs(out - want['output']).max()


@pytest.mark.parametrize('method', ['minmax', 'percentile'])
def test_gpu_pipeline_agrees_with_the_cpu_path_fixture(env, method):
    """D: CPU-path fixture vs the same reference pipeline on the GPU with our kernels.  Weights: bit-equal.  Activations differ by conv
    rounding (cuDNN vs CPU) only: scales within 1e-4 relative; the percentile observer additionally selects a neighbouring order statistic
    on the CPU path (int() truncation vs round-to-nearest index, SURVEY appendix B)."""
    z, entry = env['z'], env['meta']['methods'][method]
    got = reference_run(env, 'ours', method)
    for r, g in zip(entry['calibrated'], got['calibrated']):
        assert (r['op'], r['var'], r['state'], r['dominator']) == (g['op'], g['var'], g['state'], g['dominator'])
        if r['state'] == 'FP32': continue
        if r['var'].endswith('.w') or (r['var'] == 'x' and method == 'minmax'):
            assert np.array_equal(bits(z[r['scale']]), bits(g['scale'])), (r['op'], r['var'])
        else:
            np.testing.assert_allclose(g['scale'], z[r['scale']], rtol=0.15 if method == 'percentile' else 1e-4)   # percentile: the next order statistic of a tail
    np.testing.assert_allclose(got['output'], z[f'{method}.output'], atol=0.08 if method == 'minmax' else 0.5)   # a few quantisation steps of the last layer


def test_parameter_baking_states_values_and_no_requantisation(env):
    """ParameterBakingPass semantics (ppq/IR/quantize.py:98-111, optim/baking.py:34-47): ACTIVATED -> BAKED, PASSIVE -> PASSIVE_BAKED, the
    baked value IS the fake-quantised value, and later forwards use it as is (no weight fake-quant launch, the parameter is not touched)."""
    from ppq_b200.core import QuantizationStates as S
    from ppq_b200.qfunction import PPQuantFunction
    ex, batches = our_executor(env)
    ops = dict(ex.quantable_operations())
    ops['conv3#0'].weight_cfg.master_by = ops['conv2#0'].weight_cfg        # a passive parameter config: shares conv2's per-channel scales (16 channels each)
    assert ops['conv3#0'].weight_cfg.state == S.PASSIVE and ops['conv3#0'].weight_cfg.scale is ops['conv2#0'].weight_cfg.scale
    weighted = {n: op for n, op in ops.items() if op.weight_cfg is not None}
    fp32 = {n: op.module.weight.data.clone() for n, op in weighted.items()}
    want = {n: PPQuantFunction(op.module.weight.data, op.weight_cfg).clone() for n, op in weighted.items()}
    assert len(ex._quantize_all_weights()) == len(weighted)                # before baking: every ACTIVATED / PASSIVE weight is re-quantised per forward (one launch)
    ex._restore_weights()
    ex.bake_parameters()
    for n, op in weighted.items():
        assert op.weight_cfg.state == (S.PASSIVE_BAKED if n == 'conv3#0' else S.BAKED), (n, op.weight_cfg.state)
        assert np.array_equal(bits(op.module.weight.data.cpu().numpy()), bits(want[n].cpu().numpy())), n
    assert ex._quantize_all_weights() == {}                                # nothing left to quantise per forward
    ptrs = {n: op.module.weight.data_ptr() for n, op in weighted.items()}
    ex.forward(batches[0])
    for n, op in weighted.items():
        assert op.module.weight.data_ptr() == ptrs[n] and np.array_equal(bits(op.module.weight.data.cpu().numpy()), bits(want[n].cpu().numpy())), n
    ex.bake_parameters()                                                   # idempotent: BAKED configs are skipped
    for n, op in weighted.items():
        assert np.array_equal(bits(op.module.weight.data.cpu().numpy()), bits(want[n].cpu().numpy())), n
    # dequantize() / restore_quantize_state() (IR/quantize.py:118-160): the fp32 weights come back from `stored_value`, every config reads FP32
    ex.dequantize()
    for n, op in weighted.items():
        assert op.weight_cfg.state == S.FP32 and op.output_cfg.state == S.FP32
        assert np.array_equal(bits(op.module.weight.data.cpu().numpy()), bits(fp32[n].cpu().numpy())), n
    ex.restore_quantize_state()
    for n, op in weighted.items():
        assert op.weight_cfg.state == (S.PASSIVE_BAKED if n == 'conv3#0' else S.BAKED)
        assert np.array_equal(bits(op.module.weight.data.cpu().numpy()), bits(want[n].cpu().numpy())), n


def test_graphwise_error_analyse_equals_the_reference_function(env):
    """The evaluation loop (SURVEY 8f-3): the reference's own graphwise_error_analyse on its quantised graph (our kernels installed) vs ours on the
    equivalent module with bit-identical configs -- same operations, same seeded sample of 4096 elements per image, same SNR."""
    import ppq_b200.install as inst
    from ppq_b200.executor import calibrate_arena, graphwise_error_analyse
    name = f"{env['fixture']}:analyse:kl"
    if env['ppq'] is None:
        want = stored_run(name)
    else:
        inst.install(replace_observers=False)
        try:
            want = netspec.run_reference_pipeline(env['ppq'], env['spec'], env['params'], env['data'], 'kl', device='cuda', cuda_kernel=True, analyse=True)
        finally:
            inst.uninstall()
        record_run(name, want)
    ex, batches = our_executor(env)
    calibrate_arena(ex, batches, method='kl')
    ex.align_quantization(); ex.bake_parameters()
    check_against(ex, env, want['final'], 'analyse/final')
    got = graphwise_error_analyse(ex, batches, fetchs=4096)
    assert sorted(got) == sorted(k + '#0' for k in want['graphwise']), (sorted(got), sorted(want['graphwise']))
    for k, v in want['graphwise'].items():
        assert abs(got[k + '#0'] - v) <= 1e-6 + 2e-4 * abs(v), (k, got[k + '#0'], v)
    full = graphwise_error_analyse(ex, batches)                            # whole tensors, every operation: same order of magnitude, all below the 0.1 bar
    assert len(full) == len(ex.quantable_operations()) and all(0 <= e < 0.1 for e in full.values())


@pytest.mark.parametrize('method', ['kl', 'percentile'])
def test_second_graph_concat_alignment_and_sigmoid_fusion(env_cat, method):
    """A + C on the Concat graph: the reference pipeline is identical under both native extensions, and our executor (arena flow, then Concat
    'Align to Output' + baking) reproduces its configs, baked weights and quantised output bit for bit."""
    from ppq_b200.executor import calibrate_arena
    env = env_cat
    assert_same(reference_run(env, 'ref', method), reference_run(env, 'ours', method), f'tinycat ref-ext vs ours [{method}]')
    want = reference_run(env, 'ours', method)
    ex, batches = our_executor(env)
    calibrate_arena(ex, batches, method=method)
    check_against(ex, env, want['calibrated'], f'tinycat/{method}/calibrated')
    ex.align_quantization(); ex.bake_parameters()
    check_against(ex, env, want['final'], f'tinycat/{method}/final')
    out = ex.forward(batches[0]).cpu().numpy()
    assert np.array_equal(bits(out), bits(want['output'])), np.abs(out - want['output']).max()
