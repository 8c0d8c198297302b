"""Layerwise error analysis without a GPU: the exact-moment oracle against rational arithmetic, the measures derived from moments against the
reference's formulas, torch.cosine_similarity's treatment of zero and tiny rows, the C ABI's argument checks, and the executor's
single-operation state switch."""
import ctypes
import math
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

import layerwise_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fraction_moments(p, r):
    out = []
    for a, b in zip(np.asarray(p, np.float32).reshape(len(p), -1), np.asarray(r, np.float32).reshape(len(r), -1)):
        fa, fb = [Fraction(float(v)) for v in a], [Fraction(float(v)) for v in b]
        out.append([float(sum(((x - y) ** 2 for x, y in zip(fa, fb)), Fraction(0))), float(sum((y * y for y in fb), Fraction(0))),
                    float(sum((x * x for x in fa), Fraction(0))), float(sum((x * y for x, y in zip(fa, fb)), Fraction(0)))])
    return np.array(out)


def rows_like(kind, rng, rows, n):
    if kind == 'fp32': x = rng.standard_normal((rows, n)) * np.exp(rng.uniform(-20, 20, (rows, n)))
    elif kind == 'fp16': x = torch.from_numpy(rng.standard_normal((rows, n)) * 30).half().float().numpy()
    elif kind == 'bf16': x = torch.from_numpy(rng.standard_normal((rows, n)) * 1e10).bfloat16().float().numpy()
    elif kind == 'huge': x = rng.standard_normal((rows, n)) * 1e19                     # an fp32 sum of squares would overflow
    elif kind == 'wide': x = rng.choice([1e-30, 1.0, 3e7, -2e-20, 1e30], (rows, n))   # p - r not exact in fp64
    return x.astype(np.float32)


@pytest.mark.parametrize('kind', ['fp32', 'fp16', 'bf16', 'huge', 'wide'])
@pytest.mark.parametrize('n', [1, 3, 97])
def test_exact_moments_are_the_correctly_rounded_rational_sums(kind, n):
    rng = np.random.default_rng(n * 7 + len(kind))
    p, r = rows_like(kind, rng, 4, n), rows_like(kind, rng, 4, n)
    p[1] = r[1]                                                             # identical rows
    r[2] = 0.0                                                              # zero reference
    p[3] = 0.0; r[3] = 0.0                                                  # all-zero row
    got, want = lo.exact_moments(p, r), fraction_moments(p, r)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (got, want)


def test_exact_moments_follow_ieee_for_special_values():
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    p = np.array([[1, inf, 2], [1, 2, 3], [inf, 1, 1], [nan, 1, 1], [inf, 0, 1]], np.float32)
    r = np.array([[1, 1, 2], [1, 2, -inf], [inf, 1, 1], [1, 1, 1], [1, 1, 1]], np.float32)
    m = lo.exact_moments(p, r)
    assert np.isposinf(m[0]).tolist() == [True, False, True, True] and m[0, 1] == 6.0   # sum r^2 of a finite reference stays finite
    assert np.isposinf(m[1, :2]).all() and m[1, 2] == 14.0 and np.isneginf(m[1, 3])
    assert np.isnan(m[2, 0]) and np.isposinf(m[2, 1:]).all()                           # inf - inf
    assert np.isnan(m[3, [0, 2, 3]]).all() and m[3, 1] == 3.0
    assert np.isposinf(m[4, [0, 2, 3]]).all()
    r5 = np.array([[0, 1, 1]], np.float32)
    assert np.isnan(lo.exact_moments(np.array([[inf, 1, 1]], np.float32), r5)[0, 3])     # inf * 0


def test_long_rows_are_summed_in_exact_partials():
    rng = np.random.default_rng(5)
    n = lo.CHUNK + 3
    p = rng.standard_normal((1, n)).astype(np.float32)
    r = (p + rng.standard_normal((1, n)).astype(np.float32) * 1e-3).astype(np.float32)
    got = lo.exact_moments(p, r)
    ref = [math.fsum(np.float64(p[0]) * np.float64(p[0])), math.fsum(np.float64(p[0]) * np.float64(r[0]))]
    assert abs(got[0, 2] - ref[0]) <= 2 ** -52 * ref[0] and abs(got[0, 3] - ref[1]) <= 2 ** -52 * np.abs(np.float64(p[0]) * r[0]).sum()


def test_measures_from_moments_are_the_reference_formulas_in_exact_arithmetic():
    from ppq_b200.measure import measure_rows
    rng = np.random.default_rng(0)
    p = rng.standard_normal((6, 50)).astype(np.float32); r = (p + 0.1 * rng.standard_normal((6, 50))).astype(np.float32)
    m = torch.from_numpy(lo.exact_moments(p, r))
    P, R = torch.from_numpy(p).double(), torch.from_numpy(r).double()
    want = {'snr': ((P - R) ** 2).sum(1) / ((R ** 2).sum(1) + 1e-7), 'mse': ((P - R) ** 2).mean(1),
            'cosine': torch.cosine_similarity(P, R, dim=-1)}
    for method, w in want.items():
        assert torch.allclose(measure_rows(m, 50, method), w, rtol=1e-13, atol=0), method
    # the fp32 restatements are the reference's values to fp32 accuracy
    fp, fr = torch.from_numpy(p), torch.from_numpy(r)
    assert abs(lo.torch_snr_error(fp, fr).item() - want['snr'].mean().item()) <= 1e-5 * want['snr'].mean().item()
    assert abs(lo.torch_mean_square_error(fp, fr).item() - want['mse'].mean().item()) <= 1e-5 * want['mse'].mean().item()
    assert abs(lo.torch_cosine_similarity(fp, fr).item() - want['cosine'].mean().item()) <= 1e-6


def test_torch_cosine_similarity_clamps_each_norm_to_eps_on_the_cpu():
    """What the installed torch does with zero and tiny rows (ATen cosine_similarity: each norm clamped to eps = 1e-8, then the dot product of
    the normalised rows): a zero row gives 0, never NaN, and a row whose norm is below 1e-8 is divided by 1e-8.  measure_rows(..., 'cosine')
    uses the same rule."""
    from ppq_b200.measure import measure_rows
    x = torch.tensor([[3.0, 4.0], [0.0, 0.0], [3e-9, 4e-9], [1e-20, 0.0]], dtype=torch.float64)
    y = torch.tensor([[3.0, 4.0], [1.0, 2.0], [3e-9, 4e-9], [1.0, 0.0]], dtype=torch.float64)
    got = torch.cosine_similarity(x, y, dim=-1)
    assert got[0] == 1.0 and got[1] == 0.0
    assert abs(got[2].item() - (25e-18 / (1e-8 * 1e-8))) < 1e-12                     # both norms 5e-9 < eps
    assert abs(got[3].item() - 1e-20 / 1e-8) < 1e-25
    m = torch.from_numpy(lo.exact_moments(x.float().numpy(), y.float().numpy()))
    assert torch.allclose(measure_rows(m, 2, 'cosine'), torch.cosine_similarity(x.float().double(), y.float().double(), dim=-1), rtol=1e-6, atol=0)
    f = torch.cosine_similarity(x.float(), y.float(), dim=-1)                          # the same in fp32
    assert f[1] == 0.0 and not torch.isnan(f).any()


def test_recorder_running_mean_matches_the_host_reduction():
    """layerwise_error_analyse replays MeasureRecorder's arithmetic from the per-update values: same order, same Python doubles."""
    rec = lo.MeasureRecorder('snr')
    vals, weights = [0.1, 0.30000000000000004, 1e-9, 7.0], [4, 1, 4, 3]
    rec.fn = lambda y_pred, y_real: torch.tensor(vals[rec.updates], dtype=torch.float64)
    for w in weights: rec.update(torch.zeros(w, 2), torch.zeros(w, 2))
    m, n = 0.0, 0
    for v, w in zip(vals, weights):
        m = m * n + v * w; n += w; m /= n
    assert m == rec.measure


def test_c_abi_paired_moments_argument_checks():
    from ppq_b200.build import LIB
    if not os.path.exists(LIB): pytest.skip('libppq_b200.so not built')
    L = ctypes.CDLL(LIB)
    L.ppq_b200_multi_paired_moments_workspace_bytes.restype = ctypes.c_int64
    L.ppq_b200_multi_paired_moments_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int64]
    L.ppq_b200_multi_paired_moments_dt.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_int,
                                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    assert L.ppq_b200_multi_paired_moments_workspace_bytes(96, 68 * 2 ** 20) == (96 + 68 * 2 ** 20 // 16384) * 32
    assert L.ppq_b200_multi_paired_moments_workspace_bytes(-1, 0) == 0
    f = L.ppq_b200_multi_paired_moments_dt
    dummy = ctypes.c_void_p(16)
    assert f(None, 0, 4, 4, 0, None, None, None) == 0                                  # empty table: nothing to write
    assert f(dummy, -1, 4, 4, 0, dummy, dummy, None) == 1
    assert f(dummy, 2049, 4, 4, 0, dummy, dummy, None) == 1
    assert f(dummy, 1, -1, 4, 0, dummy, dummy, None) == 1
    assert f(dummy, 1, 4, -4, 0, dummy, dummy, None) == 1
    assert f(dummy, 1, 4, 4, 7, dummy, dummy, None) == 1                               # unknown element type
    assert f(None, 1, 4, 4, 0, dummy, dummy, None) == 1
    assert f(dummy, 1, 4, 4, 0, None, dummy, None) == 1
    assert f(dummy, 1, 4, 4, 0, dummy, None, None) == 1
    assert f(dummy, 1, 4, 4, 0, ctypes.c_void_p(24), dummy, None) == 1                 # out not 16-byte aligned


def _fake_baked_executor():
    """A CPU executor with every config given a state and every weight 'baked' by hand (no kernel runs): enough for the state switch."""
    import netspec
    from ppq_b200.core import QuantizationStates as S
    from ppq_b200.executor import TorchExecutor
    spec = netspec.SPECS['tinyres']
    ex = TorchExecutor(netspec.SpecNet(spec, netspec.make_params(spec, 1)), torch.zeros(1, 3, 32, 32), fuse_bn=False)
    for _, op in ex.quantable_operations():
        for c in op.input_cfgs + [op.output_cfg]:
            if c.state == S.INITIAL: c.state = S.ACTIVATED
        if op.weight_cfg is not None:
            op.stored_weight = op.module.weight.data
            op.module.weight.data = op.stored_weight * 0.5
            op.weight_cfg.state = S.BAKED
    return ex


def _snapshot(ex):
    ptr = lambda t: None if t is None else t.data_ptr()                                 # noqa: E731  (`.data` is a new object per access)
    return [(n, [c.state for c in ex._configs_of(op)], ptr(op.module.weight.data) if op.weight_cfg is not None else None,
             ptr(op.stored_weight)) for n, op in ex.quantable_operations()]


def test_quantize_only_switches_one_operation_and_restores_everything():
    from ppq_b200.core import QuantizationStates as S
    ex = _fake_baked_executor()
    before = _snapshot(ex)
    with pytest.raises(RuntimeError, match='dequantize'):
        ex.quantize_only('conv1#0')
    ex.dequantize()
    for name in ['conv1#0', 'conv3#0', 'fc#0']:
        ex.quantize_only(name)
        for (n, states, w, stored), (_, op) in zip(before, ex.quantable_operations()):
            now = [c.state for c in ex._configs_of(op)]
            if n == name:
                assert now == states and op.module.weight.data_ptr() == w and op.stored_weight.data_ptr() == stored
            else:
                assert all(s == S.FP32 for s in now)
                if stored is not None: assert op.module.weight.data_ptr() == stored and op.stored_weight.data_ptr() == w
    ex.quantize_only(None)
    ex.restore_quantize_state()
    after = _snapshot(ex)
    for (n, s0, w0, st0), (_, s1, w1, st1) in zip(before, after):
        assert s0 == s1 and w0 == w1 and st0 == st1, n


# ---------------------------------------------------------------- the reference function's own values (tests/golden/layerwise_ref.npz)
def _fixture():
    import json
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'layerwise_ref.npz'))
    return z, json.loads(bytes(z['meta']).decode())


def _cpu_pipeline(net, meta):
    """oracle/cpu_pipeline.py (pinned bit for bit against the reference pipeline's CPU path) calibrated with minmax, aligned and baked, with
    the fp32 and the baked weight of every operation kept, so that one operation at a time can run quantised."""
    import netspec
    from oracle.cpu_pipeline import CpuPipeline
    spec = netspec.SPECS[net]
    batches = [torch.from_numpy(x) for x in netspec.make_data(net, meta['data_seed'], meta['steps'], meta['batch'])]
    pipe = CpuPipeline(netspec.SpecNet(spec, netspec.make_params(spec, meta['param_seed'])), batches[0], fuse_bn=False)
    pipe.quantize_parameters(); pipe.calibrate(batches, 'minmax'); pipe.align()
    fp32 = {op.name: op.module.weight.data for op in pipe.ops if op.w is not None}
    pipe.bake()
    baked = {op.name: op.module.weight.data for op in pipe.ops if op.w is not None}
    states = {id(c): c.state for op in pipe.ops for c in op.ins + [op.out] + ([op.w] if op.w is not None else [])}

    def only(name):
        """QuantableOperation.dequantize() of every operation, then restore_quantize_state() of `name` (IR/quantize.py:118-160)."""
        for op in pipe.ops:
            for c in op.ins + [op.out] + ([op.w] if op.w is not None else []): c.state = states[id(c)] if op.name == name else 'FP32'
            if op.w is not None: op.module.weight.data = baked[op.name] if op.name == name else fp32[op.name]
    return pipe, batches, only


@pytest.mark.parametrize('net', ['tinyres', 'tinycat'])
def test_restated_measures_on_the_cpu_pipeline_equal_the_reference_function(net):
    """layerwise.py:73-134 restated with the fp32 torch measures and the recorder of layerwise_oracle, run on the CPU pipeline with an
    operation-level dequantise, reproduces the reference function's values bit for bit -- for every measure, steps=8 and steps=1."""
    z, meta = _fixture()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)                                                            # the fixture's reductions ran on one thread
    try:
        _check_restated_loop(net, z, meta)
    finally:
        torch.set_num_threads(threads)


def _check_restated_loop(net, z, meta):
    from ppq_b200.executor import COMPUTING_OP
    pipe, batches, only = _cpu_pipeline(net, meta)
    names = [op.name for op in pipe.ops if op.kind in COMPUTING_OP]
    for run in meta['nets'][net]['runs']:
        assert [n + '#0' for n in run['ops']] == names
        recorders = {n: lo.MeasureRecorder(run['method']) for n in names}
        for n in names:
            for idx, x in enumerate(batches[:run['batches']]):
                only(None); fp = pipe.forward(x)
                only(n); qt = pipe.forward(x)
                recorders[n].update(y_pred=qt, y_real=fp)
                if idx >= run['steps']: break
        got = np.array([recorders[n].measure for n in names])
        assert np.array_equal(got.view(np.uint64), z[run['values']].view(np.uint64)), (net, run['method'], run['steps'], got, z[run['values']])


def test_live_reference_function_on_the_cpu_graph():
    """Where the reference checkout is importable: its layerwise_error_analyse, run now on the graph its own pipeline quantised, still gives the
    committed values."""
    import refppq
    if not refppq.available(): pytest.skip('reference checkout not available')
    ppq = refppq.load()
    import importlib.util
    spec = importlib.util.spec_from_file_location('make_layerwise_golden', os.path.join(ROOT, 'tests', 'golden', 'make_layerwise_golden.py'))
    gen = importlib.util.module_from_spec(spec); spec.loader.exec_module(gen)
    z, meta = _fixture()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    arrays, fresh = {}, {'nets': {}}
    try:
        gen.generate(ppq, 'tinyres', arrays, fresh)
    finally:
        torch.set_num_threads(threads)
    for run in fresh['nets']['tinyres']['runs']:
        assert np.array_equal(arrays[run['values']].view(np.uint64), z[run['values']].view(np.uint64)), run
