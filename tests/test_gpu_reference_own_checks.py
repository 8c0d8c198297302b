"""The reference's OWN Python surface on the GPU with ppq_b200 plugged in (VERDICT r1 item 1d): after `ppq_b200.install.install()` the real package's
`ppq.core.CUDA` wrappers, `PPQLinearQuantFunction`, `PPQFloatingQuantFunction` and `ppq.lib.Observer` are driven on CUDA tensors and checked

  * the way the reference's tests/test_cuda_kernel.py checks its kernels (re-stated here: same shapes, symmetric / asymmetric offsets, same pass
    criteria: fake-quant and grad_x bit-equal to the torch formulation, grad_s within its SNR bar, 50-bin histogram within 100 counts of histc),
  * against the reference's own torch path for the same call (`USING_CUDA_KERNEL = False`) and against its own CUDA extension (oracle/_ref).

Without the package (tests/refppq.py) the checks drive ppq_b200's mirror of that surface against the reference results recorded in
tests/golden/ref_own_checks.json.gz (PPQ_RECORD_REFERENCE=<dir> rewrites them).
"""
import atexit
import contextlib
import gzip
import hashlib
import json
import os
import types
from math import sqrt

import pytest
import torch

import refppq
from conftest import GOLDEN

pytestmark = pytest.mark.gpu
Q_MIN, Q_MAX = 0, 255
RECORD = os.path.join(GOLDEN, 'ref_own_checks.json.gz')
_recorded = {}


def digest(t):
    return hashlib.sha1(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()[:20]


def reference_result(key, compute):
    """What the reference computed for `key`: live (recorded with PPQ_RECORD_REFERENCE) where the package is present, stored otherwise."""
    if compute is None:
        with gzip.open(RECORD, 'rt') as f:
            stored = json.load(f)
        assert key in stored, f'no recorded reference result {key} in {RECORD}'
        return stored[key]
    value = compute()
    out_dir = os.environ.get('PPQ_RECORD_REFERENCE')
    if out_dir:
        if not _recorded:
            def write():
                os.makedirs(out_dir, exist_ok=True)
                with gzip.open(os.path.join(out_dir, 'ref_own_checks.json.gz'), 'wt') as f:
                    json.dump(_recorded, f, sort_keys=True)
            atexit.register(write)
        _recorded[key] = value
    return value


def mirror():
    """ppq_b200's restatement of the reference surface these tests drive."""
    import ppq_b200.core as core
    import ppq_b200.ffi as ffi
    import ppq_b200.observer as obs
    import ppq_b200.qfunction as qf

    def ppq_tensor_round(t, policy):
        assert policy == core.RoundingPolicy.ROUND_HALF_EVEN
        return torch.round(t)

    def torch_snr_error(y_pred, y_real):                                   # restatement of ppq.torch_snr_error, reduction="mean"
        noise = torch.pow(y_pred - y_real, 2).sum(dim=-1)
        signal = torch.pow(y_real, 2).sum(dim=-1)
        return (noise / signal).mean()
    return types.SimpleNamespace(
        live=False, CUDA=ffi.CUDA, RoundingPolicy=core.RoundingPolicy, QuantizationStates=core.QuantizationStates,
        ppq_tensor_round=ppq_tensor_round, torch_snr_error=torch_snr_error, ENABLE_CUDA_KERNEL=contextlib.nullcontext,
        PPQ_CONFIG=types.SimpleNamespace(USING_CUDA_KERNEL=False),
        PFL=types.SimpleNamespace(LinearQuantizationConfig=core.LinearQuantizationConfig, FloatingQuantizationConfig=core.FloatingQuantizationConfig,
                                  Observer=obs.Observer),
        PPQLinearQuantFunction=qf.PPQLinearQuantFunction, PPQFloatingQuantFunction=qf.PPQFloatingQuantFunction)


@pytest.fixture(scope='module')
def ppq():
    if not torch.cuda.is_available(): pytest.skip('no CUDA device')
    pkg = refppq.load()
    if pkg is None:
        yield mirror()
        return
    import ppq_b200.install as inst
    inst.install(replace_observers=False)
    import ppq.core.ffi as ffi
    import ppq.lib as PFL
    from ppq import QuantizationStates, RoundingPolicy, ppq_tensor_round, torch_snr_error
    from ppq.api.interface import ENABLE_CUDA_KERNEL
    from ppq.core import CUDA, PPQ_CONFIG
    from ppq.quantization.qfunction.floating import PPQFloatingQuantFunction
    from ppq.quantization.qfunction.linear import PPQLinearQuantFunction
    from ppq_b200.ffi import extension
    assert ffi.CUDA_COMPLIER.CUDA_EXTENSION is extension()
    yield types.SimpleNamespace(
        live=True, CUDA=CUDA, RoundingPolicy=RoundingPolicy, QuantizationStates=QuantizationStates, ppq_tensor_round=ppq_tensor_round,
        torch_snr_error=torch_snr_error, ENABLE_CUDA_KERNEL=ENABLE_CUDA_KERNEL, PPQ_CONFIG=PPQ_CONFIG, PFL=PFL,
        PPQLinearQuantFunction=PPQLinearQuantFunction, PPQFloatingQuantFunction=PPQFloatingQuantFunction)
    inst.uninstall()


SHAPES_T = [([1, 1, 1, 1], True), ([1, 1, 1, 1], False), ([5, 12, 13, 4], True), ([1, 7, 15, 41], False), ([50, 120, 130, 4], True),
            ([12, 74, 15, 411], False), ([50, 7, 130, 1], True), ([12, 4, 15, 3], False), ([5011, 7, 7, 1], True), ([122552, 1, 10, 4], False),
            ([10, 10, 124, 47], True), ([19, 42, 150, 3], False)]
SHAPES_C = [(s, sym, 1) for s, sym in SHAPES_T[:8]] + [([5011, 7, 7, 1], True, 0), ([122552, 1, 10, 4], False, 0), ([10, 10, 124, 47], True, 3),
                                                       ([19, 42, 150, 3], False, 3)]


def offsets(sym, n):
    return torch.zeros(n).cuda() if sym else torch.randint(low=0, high=255, size=[n]).float().cuda()


def test_linear_quantize_t_and_c_the_way_the_reference_tests_them(ppq):
    """tests/test_cuda_kernel.py:17-63 re-stated: ppq.core.CUDA.LinearQuantize_T / _C == round(t / s) + o, clip, dequantise in torch, bit for bit."""
    RoundingPolicy, ppq_tensor_round, CUDA = ppq.RoundingPolicy, ppq.ppq_tensor_round, ppq.CUDA
    torch.manual_seed(0)
    policy = RoundingPolicy.ROUND_HALF_EVEN
    for size, sym in SHAPES_T:
        for _ in range(3):
            t = torch.rand(size=size).cuda() * 32
            s, o = torch.rand(size=[1]).cuda(), offsets(sym, 1)
            want = ((ppq_tensor_round(t / s, policy=policy) + o).clip(Q_MIN, Q_MAX) - o) * s
            got = CUDA.LinearQuantize_T(t, s, o, Q_MIN, Q_MAX, policy.value)
            assert (want - got).abs().max() == 0, (size, sym)
    for size, sym, c in SHAPES_C:
        for _ in range(3):
            t = torch.rand(size=size).cuda() * 32
            s, o = torch.rand(size=[t.shape[c]]).cuda(), offsets(sym, t.shape[c])
            shape = [1 if axis != c else -1 for axis in range(t.ndim)]
            want = ((ppq_tensor_round(t / s.view(shape), policy=policy) + o.view(shape)).clip(Q_MIN, Q_MAX) - o.view(shape)) * s.view(shape)
            got = CUDA.LinearQuantize_C(t, s, o, c, Q_MIN, Q_MAX, policy.value)
            assert (want - got).abs().max() == 0, (size, sym, c)


def test_linear_quantize_backward_the_way_the_reference_tests_it(ppq):
    """tests/test_cuda_kernel.py:66-138 re-stated: grad_x bit-equal, grad_s within the reference's SNR bar (1e-5 unless the gradient is tiny)."""
    RoundingPolicy, ppq_tensor_round, torch_snr_error, CUDA = ppq.RoundingPolicy, ppq.ppq_tensor_round, ppq.torch_snr_error, ppq.CUDA
    torch.manual_seed(1)
    policy = RoundingPolicy.ROUND_HALF_EVEN

    def grads(value, dy, scale, offset, axis):
        """Straight-through gradient of fake-quant w.r.t. the input and LSQ-style gradient w.r.t. the scale, normalised by sqrt(numel * levels)."""
        q = ppq_tensor_round(value / scale, policy=policy) + offset
        below, above = q < Q_MIN, q > Q_MAX
        inside = ~(below | above)
        dx = dy * inside
        per_elem = inside * (((q - offset) * scale - value) / scale) + above * (Q_MAX - offset) + below * (Q_MIN - offset)
        ds = per_elem * dy
        ds = ds.sum() if axis is None else ds.movedim(axis, 0).flatten(1).sum(dim=1)
        return dx, ds / sqrt(value.numel() * (Q_MAX - Q_MIN))               # the whole tensor's element count, per channel too (test_cuda_kernel.py:118)

    def check_scale_grad(got, want, tag):
        snr = torch_snr_error(got.reshape([1, -1]), want.reshape([1, -1])).item()
        assert snr <= 1e-5 or got.abs().max().item() <= 1, tag + (snr,)

    for size, sym in [([1, 1, 1, 1], True), ([5, 12, 13, 4], True), ([1, 7, 15, 41], False), ([5, 12, 2130, 4], True), ([12, 74, 315, 41], False),
                      ([501, 7, 73, 1], True), ([1222, 12, 10, 4], False), ([19, 42, 120, 3], False)]:
        t = torch.rand(size=size).cuda() * 50
        s, o, dy = torch.rand(size=[1]).cuda(), offsets(sym, 1), torch.rand(size=size).cuda()
        gx, gs = CUDA.LinearQuantize_T_B(t, s, o, dy, Q_MIN, Q_MAX, policy.value)
        rx, rs = grads(t, dy, s, o, None)
        assert (rx.flatten() - gx.flatten()).abs().max() == 0, size
        check_scale_grad(gs, rs, (size, 'T'))
    for size, sym, c in [([1, 1, 1, 1], True, 1), ([5, 12, 14, 12], True, 1), ([1, 7, 15, 41], False, 1), ([12, 74, 15, 41], False, 1),
                         ([501, 7, 7, 1], True, 0), ([1222, 1, 10, 4], False, 0), ([10, 10, 14, 47], True, 3), ([19, 42, 10, 3], False, 3)]:
        t = torch.rand(size=size).cuda() * 50
        s, o, dy = torch.rand(size=[t.shape[c]]).cuda(), offsets(sym, t.shape[c]), torch.rand(size=size).cuda()
        shape = [1 if axis != c else -1 for axis in range(t.ndim)]
        gx, gs = CUDA.LinearQuantize_C_B(t, s, o, dy, Q_MIN, Q_MAX, c, policy.value)
        rx, rs = grads(t, dy, s.view(shape), o.view(shape), c)
        assert (rx.flatten() - gx.flatten()).abs().max() == 0, (size, c)
        check_scale_grad(gs, rs, (size, c))


def test_histogram_the_way_the_reference_tests_it(ppq):
    """tests/test_cuda_kernel.py:198-208 re-stated: 50-bin Histogram_T of |t| at scale 0.01 within 100 counts of torch.histc per bin."""
    CUDA = ppq.CUDA
    torch.manual_seed(2)
    for _ in range(3):
        t = torch.rand(size=[128, 3, 224, 224]).cuda()
        hist = torch.histc(torch.abs(t), bins=50, min=0, max=0.5)
        got = CUDA.Histogram_T(t, torch.zeros(size=[50]).cuda().int(), 0.01)
        assert torch.abs(hist - got).max().item() < 100


@pytest.mark.parametrize('per_channel', [False, True])
def test_reference_linear_quant_function_cuda_path_equals_its_torch_path(ppq, per_channel):
    """PPQLinearQuantFunction (qfunction/linear.py:200-215) on CUDA tensors: with our kernels (ENABLE_CUDA_KERNEL) == the reference's torch
    formulation (USING_CUDA_KERNEL False) == the reference's own CUDA extension, forward and backward, all 8 rounding policies forward."""
    PFL, QuantizationStates, RoundingPolicy = ppq.PFL, ppq.QuantizationStates, ppq.RoundingPolicy
    ENABLE_CUDA_KERNEL, PPQ_CONFIG, PPQLinearQuantFunction = ppq.ENABLE_CUDA_KERNEL, ppq.PPQ_CONFIG, ppq.PPQLinearQuantFunction
    torch.manual_seed(3)
    x = (torch.randn(6, 16, 17, 9).cuda() * 3).requires_grad_(True)
    dy = torch.randn_like(x)
    for rounding in RoundingPolicy:
        cfg = PFL.LinearQuantizationConfig(symmetrical=not per_channel, channel_axis=1 if per_channel else None, quant_min=-128 if not per_channel else 0,
                                           quant_max=127 if not per_channel else 255, rounding=rounding)
        n = 16 if per_channel else 1
        cfg.scale = (torch.rand(n).cuda() * 0.1 + 0.01)
        cfg.offset = torch.zeros(n).cuda() if not per_channel else torch.randint(0, 255, [n]).float().cuda()
        cfg.state = QuantizationStates.ACTIVATED
        assert PPQ_CONFIG.USING_CUDA_KERNEL is False
        with ENABLE_CUDA_KERNEL():
            y_ours = PPQLinearQuantFunction(x, cfg)
            (g_ours,) = torch.autograd.grad(y_ours, x, dy)
        key = f'linear:{per_channel}:{rounding.name}'
        if rounding == RoundingPolicy.ROUND_HALF_EVEN:                     # the policy the reference's own test compares (its torch path
            def torch_path():                                              # spells the others as fp32 floor / ceil formulas, NEAR_INT not at all)
                y_torch = PPQLinearQuantFunction(x, cfg)
                (g_torch,) = torch.autograd.grad(y_torch, x, dy)
                return [digest(y_torch), digest(g_torch)]
            assert [digest(y_ours), digest(g_ours)] == reference_result(key + ':torch', torch_path if ppq.live else None)
        ref = refppq.reference_cuda_extension() if ppq.live else None

        def reference_extension():
            with refppq.use_extension(ref):
                PPQ_CONFIG.USING_CUDA_KERNEL = True
                try:
                    y_ref = PPQLinearQuantFunction(x, cfg)
                    (g_ref,) = torch.autograd.grad(y_ref, x, dy)
                finally: PPQ_CONFIG.USING_CUDA_KERNEL = False
            return [digest(y_ref), digest(g_ref)]
        if ref is not None or not ppq.live:
            assert [digest(y_ours), digest(g_ours)] == reference_result(key + ':ref', reference_extension if ppq.live else None), rounding


def test_reference_floating_quant_function_with_our_kernels(ppq):
    """PPQFloatingQuantFunction (qfunction/floating.py:95-125) has no torch path: ours vs the reference's own CUDA extension through the same
    function, per tensor and per channel (forward: the reference's backward returns one gradient too many for autograd, floating.py:48-49)."""
    PFL, QuantizationStates, ENABLE_CUDA_KERNEL, PPQ_CONFIG = ppq.PFL, ppq.QuantizationStates, ppq.ENABLE_CUDA_KERNEL, ppq.PPQ_CONFIG
    PPQFloatingQuantFunction = ppq.PPQFloatingQuantFunction
    ref = refppq.reference_cuda_extension() if ppq.live else None
    if ppq.live and ref is None: pytest.skip('oracle/_ref/PPQ_Cuda_Impls_ref.so not built')
    torch.manual_seed(4)
    x = torch.randn(4, 24, 33).cuda() * 40
    for axis in (None, 1):
        cfg = PFL.FloatingQuantizationConfig(channel_axis=axis)
        n = 1 if axis is None else 24
        cfg.scale, cfg.offset, cfg.state = torch.rand(n).cuda() + 0.5, torch.zeros(n).cuda(), QuantizationStates.ACTIVATED
        if axis is not None: cfg.channel_axis = axis
        with ENABLE_CUDA_KERNEL():
            y_ours = PPQFloatingQuantFunction(x, cfg)

        def reference_extension():
            with refppq.use_extension(ref):
                PPQ_CONFIG.USING_CUDA_KERNEL = True
                try: return digest(PPQFloatingQuantFunction(x, cfg))
                finally: PPQ_CONFIG.USING_CUDA_KERNEL = False
        assert digest(y_ours) == reference_result(f'floating:{axis}', reference_extension if ppq.live else None), axis
    if ppq.live:
        with pytest.raises(PermissionError):
            PPQFloatingQuantFunction(x, cfg)                                # outside ENABLE_CUDA_KERNEL the reference refuses, with or without us


@pytest.mark.parametrize('algo', ['minmax', 'percentile', 'kl', 'mse'])
def test_reference_observers_through_ppq_lib_with_our_kernels(ppq, algo):
    """ppq.lib.Observer (lib/quant.py:47-56) builds the reference's own observer classes; observe() + render under ENABLE_CUDA_KERNEL call
    Quantile / Histogram_T / compute_mse_loss of whichever extension ppq.core.ffi serves: ours and the reference's give the same scale."""
    PFL, ENABLE_CUDA_KERNEL, PPQ_CONFIG = ppq.PFL, ppq.ENABLE_CUDA_KERNEL, ppq.PPQ_CONFIG
    ref = refppq.reference_cuda_extension() if ppq.live else None
    if ppq.live and ref is None: pytest.skip('oracle/_ref/PPQ_Cuda_Impls_ref.so not built')
    torch.manual_seed(5)
    batches = [torch.relu(torch.randn(8, 32, 28, 28).cuda()) * (1 + 0.1 * k) for k in range(4)]

    def run():
        cfg = PFL.LinearQuantizationConfig(symmetrical=True, calibration=algo)
        ob = PFL.Observer(quant_config=cfg)
        phases = 2 if algo in ('kl', 'mse') else 1
        for _ in range(phases):
            for b in batches: ob.observe(b)
            ob.render_quantization_config()
        return cfg.scale.clone(), cfg.offset.clone()

    with ENABLE_CUDA_KERNEL():
        s_ours, o_ours = run()

    def reference_extension():
        with refppq.use_extension(ref):
            PPQ_CONFIG.USING_CUDA_KERNEL = True
            try: s_ref, o_ref = run()
            finally: PPQ_CONFIG.USING_CUDA_KERNEL = False
        return [s_ref.cpu().reshape(-1).tolist(), o_ref.cpu().reshape(-1).tolist()]
    s_ref, o_ref = reference_result(f'observer:{algo}', reference_extension if ppq.live else None)
    assert s_ours.cpu().reshape(-1).tolist() == s_ref and o_ours.cpu().reshape(-1).tolist() == o_ref, (algo, s_ours, s_ref)
