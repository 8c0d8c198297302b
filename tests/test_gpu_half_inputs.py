"""fp16 / bf16 inputs: every kernel that takes a half tensor against the fp32 kernel on its exact upcast X = x.float().

The fp32 kernels are pinned to the oracle and the reference elsewhere, so the contract is checked against them:
  * collectors (min/max, histograms, quantiles): bit for bit what the fp32 collector returns on X;
  * fake-quant (LT, LC, FT, FC): the input's dtype and layout, value fp32_kernel(X).to(dtype), bitwise except NaN == NaN;
  * toInt: equal to toInt(X).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HALF = [torch.float16, torch.bfloat16]
SIZES = [1, 7, 8, 9, 4095, (1 << 20) + 3]


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


def specials(dtype):
    fi = torch.finfo(dtype)
    sub = torch.tensor(1, dtype=torch.int16).view(dtype).item()                               # smallest subnormal
    return [0.0, -0.0, float('inf'), float('-inf'), fi.max, -fi.max, fi.tiny, -fi.tiny, sub, -sub, 3 * sub, 0.5, -0.5, 1.5, 2.5]


def make(n, dtype, seed=0, nan=True, extra=8):
    """n elements of dtype at a storage offset of `extra` elements from a larger buffer's start (the caller slices)."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(n + extra, generator=g) * 3
    x[::5] = torch.round(x[::5] * 16) / 16                              # many exact ties of x / 0.0625
    sp = specials(dtype) + ([float('nan')] if nan else [])
    for i, v in enumerate(sp):
        x[(i * 37) % (n + extra)] = v
    return x.to(dtype).cuda()


def assert_same_half(got, want32, dtype, msg=''):
    """got (half) == want32.to(dtype) bitwise, NaN matches NaN."""
    assert got.dtype == dtype, (got.dtype, msg)
    want = want32.to(dtype)
    assert got.shape == want.shape and got.stride() == want.stride(), (got.stride(), want.stride(), msg)
    g, w = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    ok = (g == w) | (got.contiguous().isnan() & want.contiguous().isnan())
    if not bool(ok.all()):
        bad = torch.nonzero(~ok.flatten())[0].item()
        raise AssertionError(f'{msg}: {(~ok).sum().item()} differ, first at {bad}: {got.flatten()[bad].item()} vs {want.flatten()[bad].item()}')


def assert_bits(got, want, msg=''):
    assert got.dtype == want.dtype, msg
    a, b = got.cpu().numpy(), want.cpu().numpy()
    if a.dtype == np.float32: a, b = a.view(np.uint32), b.view(np.uint32)
    assert np.array_equal(a, b), msg


def t1(v):
    return torch.tensor([v], dtype=torch.float32, device='cuda')


# ------------------------------------------------------------------------------------------------ element-wise, per tensor
# 0.0625 puts every x of the ::5 grid on an exact tie; 1 + 2^-8 / 1 + 2^-11 make q * s fall on a tie of the cast back to bf16 / fp16.
LT_SCALES = [0.0625, 0.1, 1.00390625, 1.00048828125]


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('mode', range(8))
def test_lt_every_size_offset_and_mode(ext, dtype, mode):
    base = make(SIZES[-1], dtype, seed=mode)
    for n in SIZES:
        for off in (range(8) if n < 4096 else (0, 3)):
            x = base[off:off + n]
            for s in LT_SCALES:
                for lo, hi, o in ((-128, 127, 0.0), (0, 255, 7.0)):
                    y = ext.QuantizeTensor_LT_Half(x, t1(s), t1(o), lo, hi, mode)
                    assert_same_half(y, ext.QuantizeTensor_LT(x.float(), t1(s), t1(o), lo, hi, mode), dtype, f'LT n={n} off={off} s={s} o={o}')


@pytest.mark.parametrize('dtype', HALF)
def test_lt_channels_last_keeps_the_layout(ext, dtype):
    x = make(2 * 16 * 5 * 6, dtype)[:2 * 16 * 5 * 6].view(2, 16, 5, 6).to(memory_format=torch.channels_last)
    y = ext.QuantizeTensor_LT_Half(x, t1(0.05), t1(0), -128, 127, 0)
    assert y.is_contiguous(memory_format=torch.channels_last)
    assert_same_half(y, ext.QuantizeTensor_LT(x.float(), t1(0.05), t1(0), -128, 127, 0), dtype, 'LT channels_last')


LC_SPECS = [((4, 6, 5, 3), 0), ((4, 6, 5, 3), 1), ((4, 6, 5, 3), 3), ((4, 6, 5, 3), -1), ((4, 6, 5, 3), -3), ((3, 16, 8), 1),
            ((2, 3, 7), 1), ((64, 3, 3, 3), 0), ((32, 128, 3), 1), ((5, 1), 0), ((1, 1), 1), ((300, 1000), 0)]


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('mode', range(8))
def test_lc_axes_offsets_and_modes(ext, dtype, mode):
    for shape, axis in LC_SPECS:
        n = int(np.prod(shape))
        base = make(n, dtype, seed=n + mode)
        C = shape[axis]
        s = (torch.rand(C, generator=torch.Generator().manual_seed(C)) * 0.2 + 0.01).cuda()
        s[0] = 0.0625
        o = torch.round(torch.rand(C, generator=torch.Generator().manual_seed(C + 1)) * 8).cuda()
        for off in (0, 1, 3, 7):
            x = base[off:off + n].view(shape)
            y = ext.QuantizeTensor_LC_Half(x, s, o, 0, 255, axis, mode)
            assert_same_half(y, ext.QuantizeTensor_LC(x.float(), s, o, 0, 255, axis, mode), dtype, f'LC {shape} axis={axis} off={off}')


@pytest.mark.parametrize('dtype', HALF)
def test_lc_channels_last(ext, dtype):
    x = make(2 * 8 * 5 * 6, dtype)[:2 * 8 * 5 * 6].view(2, 8, 5, 6).to(memory_format=torch.channels_last)
    s = torch.linspace(0.01, 0.2, 8, device='cuda')
    y = ext.QuantizeTensor_LC_Half(x, s, torch.zeros(8, device='cuda'), -128, 127, 1, 0)
    assert_same_half(y, ext.QuantizeTensor_LC(x.float(), s, torch.zeros(8, device='cuda'), -128, 127, 1, 0), dtype, 'LC channels_last')


FP_FORMATS = [(4, 3, -448.0, 448.0), (5, 2, -57344.0, 57344.0), (4, 3, -300.0, 300.0), (2, 1, -6.0, 6.0)]


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('mode', range(8))
def test_ft_fc_formats_and_modes(ext, dtype, mode):
    base = make(SIZES[-1], dtype, seed=100 + mode)
    for E, M, lo, hi in FP_FORMATS:
        for n in SIZES:
            for off in ((0, 1, 5) if n < 4096 else (0,)):
                x = base[off:off + n]
                for s in (1.0, 0.5, 0.1):
                    y = ext.QuantizeTensor_FT_Half(x, t1(s), t1(0), E, M, lo, hi, mode)
                    assert_same_half(y, ext.QuantizeTensor_FT(x.float(), t1(s), t1(0), E, M, lo, hi, mode), dtype, f'FT E{E}M{M} n={n} off={off} s={s}')
        for shape, axis in LC_SPECS[:8]:
            n = int(np.prod(shape))
            x = base[3:3 + n].view(shape)
            C = shape[axis]
            s = torch.linspace(0.25, 2.0, C, device='cuda')
            y = ext.QuantizeTensor_FC_Half(x, s, torch.zeros(C, device='cuda'), E, M, lo, hi, axis, mode)
            assert_same_half(y, ext.QuantizeTensor_FC(x.float(), s, torch.zeros(C, device='cuda'), E, M, lo, hi, axis, mode), dtype,
                             f'FC E{E}M{M} {shape} axis={axis}')


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('mode', [0, 1, 5, 7])
def test_toint_tensor_and_channel(ext, dtype, mode):
    base = make(SIZES[-1], dtype, seed=200 + mode)
    for n in SIZES:
        for off in ((0, 1, 4, 7) if n < 4096 else (0, 3)):
            x = base[off:off + n]
            for lo, hi, o, bits in ((-128, 127, 0.0, 8), (0, 255, 9.0, 8), (-2 ** 31, 2 ** 31 - 1, 0.0, 32)):
                got = ext.QuantizeTensor_toInt(x, t1(0.0625), t1(o), lo, hi, -1000, mode, bits)
                assert torch.equal(got, ext.QuantizeTensor_toInt(x.float(), t1(0.0625), t1(o), lo, hi, -1000, mode, bits)), (n, off, bits)
    for shape, axis in LC_SPECS:
        n = int(np.prod(shape))
        x = base[1:1 + n].view(shape)
        C = shape[axis]
        s = torch.linspace(0.01, 0.3, C, device='cuda')
        for bits in (8, 32):
            got = ext.QuantizeTensor_toInt(x, s, torch.zeros(C, device='cuda'), -128, 127, axis, mode, bits)
            assert torch.equal(got, ext.QuantizeTensor_toInt(x.float(), s, torch.zeros(C, device='cuda'), -128, 127, axis, mode, bits)), (shape, axis)


# ------------------------------------------------------------------------------------------------ collectors
def minmax_of(ext, x):
    mm = torch.empty(2, device='cuda')
    ext.MinMax_Init(mm[0:1], mm[1:2])
    ext.MinMax_T(x, mm)
    return mm


@pytest.mark.parametrize('dtype', HALF)
def test_minmax_t_and_c(ext, dtype):
    for nan in (False, True):
        base = make(SIZES[-1], dtype, seed=7, nan=nan)
        for n in SIZES:
            for off in ((0, 1, 2, 5, 7) if n < 4096 else (0, 3)):
                x = base[off:off + n]
                assert_bits(minmax_of(ext, x), minmax_of(ext, x.float()), f'MinMax_T n={n} off={off} nan={nan}')
        for shape, axis in LC_SPECS:
            n = int(np.prod(shape))
            x = base[5:5 + n].view(shape)
            C = shape[axis]
            res = []
            for v in (x, x.float()):
                lo, hi = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
                ext.MinMax_Init(lo, hi)
                ext.MinMax_C(v, axis, lo, hi)
                res.append((lo, hi))
            assert_bits(res[0][0], res[1][0], f'MinMax_C min {shape} {axis}')
            assert_bits(res[0][1], res[1][1], f'MinMax_C max {shape} {axis}')


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('bins', [2048, 4096, 12287, 16384])
def test_histograms(ext, dtype, bins):
    base = make(SIZES[-1], dtype, seed=bins, nan=False)
    base[base.isinf()] = 0
    relu = torch.clamp(base, min=0)
    for src in (base, relu):
        for n in SIZES:
            for off in ((0, 1, 6) if n < 4096 else (0, 5)):
                x = src[off:off + n]
                for clip in (True, False):
                    hs = torch.tensor([3.0 / bins], device='cuda')
                    h = [torch.zeros(bins, dtype=torch.int32, device='cuda') for _ in range(2)]
                    ext.Histogram_T_DeviceScale(x, hs, clip, h[0])
                    ext.Histogram_T_DeviceScale(x.float(), hs, clip, h[1])
                    assert torch.equal(h[0], h[1]), f'dscale n={n} off={off} clip={clip}'
                    h = [torch.zeros(bins, dtype=torch.int32, device='cuda') for _ in range(2)]
                    ext.Histogram_Asymmetric_T_Half(-2.5, 4.0, x, clip, h[0])
                    ext.Histogram_Asymmetric_T(-2.5, 4.0, x.float(), clip, h[1])
                    assert torch.equal(h[0], h[1]), f'asym n={n} off={off} clip={clip}'


@pytest.mark.parametrize('dtype', HALF)
def test_quantile_single_and_guess(ext, dtype):
    for n in SIZES + [(9 << 20) + 5]:
        base = make(n, dtype, seed=n % 1000, nan=False)
        for src in (base, torch.clamp(base, min=0)):
            for off in ((0, 1, 7) if n < 4096 else (0, 3)):
                x = src[off:off + n]
                for q in (0.9999, 0.999, 0.5):
                    assert_bits(ext.Quantile_T_Half(x, q), ext.Quantile_T(x.float(), q), f'quantile n={n} off={off} q={q}')
    # the guess form over consecutive batches of one activation: the same answers as the fp32 guess form on the upcasts
    g16, g32 = ext.Quantile_Guess_Init(1, base), ext.Quantile_Guess_Init(1, base.float())
    for b in range(4):
        x = make((1 << 20) + 11, dtype, seed=50 + b, nan=False)[1:]
        assert_bits(ext.Quantile_T_Guess(x, 0.9999, g16), ext.Quantile_T_Guess(x.float(), 0.9999, g32), f'guess batch {b}')
    assert ext.Quantile_T_Half(make(9, dtype, nan=True), 0.9).dtype == torch.float32


# ------------------------------------------------------------------------------------------------ host mirror
def _cfg(kind, sym):
    from ppq_b200 import LinearQuantizationConfig
    return LinearQuantizationConfig(symmetrical=sym, quant_min=-128 if sym else 0, quant_max=127 if sym else 255, calibration=kind)


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('kind,sym', [('minmax', True), ('minmax', False), ('kl', True), ('percentile', True), ('percentile', False),
                                      ('mse', True), ('mse', False)])
def test_observers_match_the_upcast(ext, dtype, kind, sym):
    """Each observer calibrated on half batches gives the scale and offset it gives on their fp32 upcasts; the fake-quant forward with that
    config is the fp32 kernel on the upcast, cast back."""
    from ppq_b200.observer import Observer
    from ppq_b200.qfunction import PPQuantFunction
    batches = [make(3 * 64 * 17 * 17, dtype, seed=300 + i, nan=False)[i + 1:i + 1 + 3 * 64 * 17 * 17].view(3, 64, 17, 17) for i in range(3)]
    for b in batches: b[b.isinf()] = 0
    got = []
    for cast in (lambda t: t, lambda t: t.float()):
        cfg = _cfg(kind, sym)
        ob = Observer(cfg)
        for b in batches: ob.observe(cast(b))
        ob.render_quantization_config()
        if kind in ('kl', 'mse'):
            for b in batches: ob.observe(cast(b))
            ob.render_quantization_config()
        got.append(cfg)
    assert_bits(got[0].scale, got[1].scale, f'{kind} sym={sym} scale')
    assert_bits(got[0].offset, got[1].offset, f'{kind} sym={sym} offset')
    y = PPQuantFunction(batches[0], got[0])
    assert_same_half(y, ext.QuantizeTensor_LT(batches[0].float(), got[0].scale.view(1), got[0].offset.view(1), got[0].quant_min,
                                              got[0].quant_max, 0), dtype, f'{kind} forward')


@pytest.mark.parametrize('dtype', HALF)
def test_qfunction_per_channel_dynamic_float_and_toint(ext, dtype):
    from ppq_b200 import FloatingQuantizationConfig, LinearQuantizationConfig, QuantizationStates
    from ppq_b200.qfunction import PPQLinearQuant_toInt, PPQuantFunction
    w = make(64 * 3 * 3 * 3, dtype, seed=9, nan=False)[:64 * 27].view(64, 3, 3, 3)
    w[w.isinf()] = 1
    s = torch.linspace(0.01, 0.3, 64, device='cuda')
    cfg = LinearQuantizationConfig(channel_axis=0)
    cfg.scale, cfg.offset, cfg.state = s, torch.zeros(64, device='cuda'), QuantizationStates.ACTIVATED
    assert_same_half(PPQuantFunction(w, cfg), ext.QuantizeTensor_LC(w.float(), s, cfg.offset, -128, 127, 0, 0), dtype, 'per-channel')
    assert torch.equal(PPQLinearQuant_toInt(w, cfg), PPQLinearQuant_toInt(w.float(), cfg))
    # gradients pass straight through in the input's dtype
    wg = w.clone().requires_grad_(True)
    PPQuantFunction(wg, cfg).sum().backward()
    assert wg.grad.dtype == dtype and bool((wg.grad == 1).all())
    dyn = LinearQuantizationConfig(dynamic=True)
    dyn.state = QuantizationStates.ACTIVATED
    assert_same_half(PPQuantFunction(w, dyn), PPQuantFunction(w.float(), dyn), dtype, 'dynamic')
    fcfg = FloatingQuantizationConfig()
    fcfg.scale, fcfg.offset, fcfg.state = torch.tensor(0.5, device='cuda'), torch.tensor(0.0, device='cuda'), QuantizationStates.ACTIVATED
    assert_same_half(PPQuantFunction(w, fcfg), ext.QuantizeTensor_FT(w.float(), t1(0.5), t1(0), 4, 3, -448.0, 448.0, 0), dtype, 'FP8')


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize('dtype', HALF)
def test_half_input_refusals(ext, dtype):
    from ppq_b200.qfunction import CuLSQ_LC, CuLSQ_LT
    x = torch.ones(16, 4, device='cuda', dtype=dtype)
    s, o = t1(0.1), t1(0)
    for call in (lambda: ext.QuantizeTensor_LT(x, s, o, -128, 127, 0),
                 lambda: ext.QuantizeTensor_LT_B(x, s, o, x, -128, 127, 0),
                 lambda: ext.QuantizeTensor_FT_B(x, s, o, x, 4, 3, -448.0, 448.0, 0),
                 lambda: ext.TensorClip_T(x, x, s),
                 lambda: ext.RoundingLoss_LT(x, s, o, -128, 127, 0),
                 lambda: ext.Histogram_C(x, 1, 0.1, True, torch.zeros(4, 16, dtype=torch.int32, device='cuda')),
                 lambda: ext.Isotone_T(x),
                 lambda: ext.Quantile_T(x, 0.9)):
        with pytest.raises(RuntimeError, match='Invalid dtype of Input tensor'):
            call()
    with pytest.raises(RuntimeError, match=r'Expect to be FP16 or BF16'):
        ext.QuantizeTensor_LT_Half(x.float(), s, o, -128, 127, 0)
    with pytest.raises(TypeError):
        CuLSQ_LT.apply(x, s, o, -128, 127, 0)
    with pytest.raises(TypeError):
        CuLSQ_LC.apply(x, torch.ones(16, device='cuda'), torch.zeros(16, device='cuda'), 0, -128, 127, 0)


# ------------------------------------------------------------------------------------------------ networks
class _Tap:
    """Records what the executor hands every quantable operation: (fp inputs, fake-quantised inputs, configs) and the outputs."""

    def __init__(self, store, name): self.store, self.name = store, name
    def pre_forward_hook(self, inputs, quant_inputs, quant_configs): self.store[self.name] = [list(zip(inputs, quant_inputs, quant_configs))]
    def post_forward_hook(self, outputs, quant_outputs, quant_configs): self.store[self.name].append((outputs[0], quant_outputs[0], quant_configs[0]))


def _expected_fake_quant(ext, x, cfg):
    """The fp32 kernel on the upcast with the config's (fp32) scale and offset."""
    from ppq_b200.core import QuantizationProperty as P
    if cfg.policy.has_property(P.PER_CHANNEL):
        return ext.QuantizeTensor_LC(x.float(), cfg.scale.float(), cfg.offset.float(), cfg.quant_min, cfg.quant_max, cfg.channel_axis, 0)
    return ext.QuantizeTensor_LT(x.float(), cfg.scale.float().reshape(1), cfg.offset.float().reshape(1), cfg.quant_min, cfg.quant_max, 0)


def _check_quantised_forward(ext, ex, x, dtype):
    from ppq_b200.core import QuantizationStates as S
    store = {}
    ex.forward(x, hooks={n: _Tap(store, n) for n, _ in ex.quantable_operations()})
    checked = 0
    for name, rec in store.items():
        for fp, q, cfg in rec[0] + rec[1:]:
            if cfg is None or cfg.state not in (S.ACTIVATED, S.PASSIVE) or q is fp: continue
            assert fp.dtype == dtype and q.dtype == dtype, (name, fp.dtype, q.dtype)
            assert_same_half(q, _expected_fake_quant(ext, fp, cfg), dtype, f'{name} {cfg.state}')
            checked += 1
    assert checked > 0
    return checked


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('method', ['minmax', 'percentile', 'kl', 'mse'])
def test_half_network_calibrate_quantise_bake_and_analyse(ext, dtype, method):
    """A netspec network cast to fp16 / bf16 through the hook calibration flow: quantize_parameters -> RuntimeCalibrationPass -> alignment ->
    quantised forward (weights fake-quantised one launch per weight, never through the fp32-only table kernel) -> bake -> forward ->
    graphwise_error_analyse.  Every fake-quantised weight and activation is the fp32 kernel on its upcast, cast back; every weight scale is the
    fp32 observer's on the upcast weight."""
    import netspec
    from ppq_b200.calibration import RuntimeCalibrationPass
    from ppq_b200.core import QuantizationStates as S
    from ppq_b200.executor import TorchExecutor, graphwise_error_analyse
    from ppq_b200.observer import TorchMinMaxObserver
    for name in ('tinyres', 'tinycat'):
        spec = netspec.SPECS[name]
        model = netspec.SpecNet(spec, netspec.make_params(spec, 3)).cuda().to(dtype)
        batches = [torch.from_numpy(b).cuda().to(dtype) for b in netspec.make_data(name, 4, 8, 4)]
        ex = TorchExecutor(model, batches[0], fuse_bn=False)
        ex.quantize_parameters()
        for n, op in ex.quantable_operations():
            if op.weight_cfg is None: continue
            w = op.module.weight.data
            assert w.dtype == dtype
            ref = type(op.weight_cfg)(policy=op.weight_cfg.policy, rounding=op.weight_cfg.rounding, num_of_bits=op.weight_cfg.num_of_bits,
                                      quant_min=op.weight_cfg.quant_min, quant_max=op.weight_cfg.quant_max, observer_algorithm='minmax',
                                      channel_axis=op.weight_cfg.channel_axis)
            ob = TorchMinMaxObserver(None, ref)
            ob.observe(w.float()); ob.render_quantization_config()
            assert_bits(op.weight_cfg.scale, ref.scale, f'{n} weight scale')
        RuntimeCalibrationPass(method=method).optimize(graph=ex, dataloader=batches, executor=ex, calib_steps=8)
        ex.align_quantization()
        cfgs = [c for _, op in ex.quantable_operations() for c in op.input_cfgs + [op.output_cfg]]
        assert all(c.state != S.INITIAL for c in cfgs), name
        assert all(bool(torch.isfinite(c.scale).all()) for c in cfgs if c.state == S.ACTIVATED), name
        n_before = _check_quantised_forward(ext, ex, batches[1], dtype)
        ex.bake_parameters()
        for n, op in ex.quantable_operations():
            if op.weight_cfg is None: continue
            assert op.weight_cfg.state == S.BAKED
            assert_same_half(op.module.weight.data, _expected_fake_quant(ext, op.stored_weight, op.weight_cfg), dtype, f'{n} baked')
        assert _check_quantised_forward(ext, ex, batches[2], dtype) > 0 and n_before > 0
        snr = graphwise_error_analyse(ex, batches[:2])
        assert snr and all(np.isfinite(v) for v in snr.values()), snr


@pytest.mark.parametrize('dtype', HALF)
def test_fp32_only_table_paths_refuse_half_before_a_launch(ext, dtype):
    """The descriptor tables carry raw pointers to fp32 data: their builders refuse anything else, so no half tensor reaches a table kernel."""
    import netspec
    from ppq_b200.calibration import ArenaCalibrator, MultiWeightQuantizer
    from ppq_b200.executor import TorchExecutor, calibrate_arena
    w = torch.randn(8, 4, device='cuda').to(dtype)
    with pytest.raises(TypeError, match='fp32'):
        MultiWeightQuantizer([w, w], [torch.ones(8, device='cuda')] * 2, [torch.zeros(8, device='cuda')] * 2)
    with pytest.raises(RuntimeError, match='fp32'):
        ArenaCalibrator(1, 'cuda', method='minmax').observe([w])
    spec = netspec.SPECS['tinyres']
    model = netspec.SpecNet(spec, netspec.make_params(spec, 3)).cuda().to(dtype)
    x = torch.rand(2, 3, 32, 32, device='cuda').to(dtype)
    ex = TorchExecutor(model, x, fuse_bn=False)
    with pytest.raises(TypeError, match='RuntimeCalibrationPass'):
        calibrate_arena(ex, [x], method='minmax')
