"""Calibration beyond symmetric INT8: every scale search on the device against the oracle chain, bit for bit on the fp32 scale and offset.

Configs: symmetric INT8 (control), asymmetric 0..255, symmetric 4-bit and asymmetric 0..15, power-of-two (both), the minimum-scale override
and the KL bin override.  Data: randn, post-ReLU, all-negative, all-zero, a constant, a single element, a range that clamps to the minimum
scale, +-3e38, +-inf and NaN.  Both calibration flows are checked: the hook path (RuntimeCalibrationPass, one observer per config) and the
arena path (calibrate_arena, one ArenaCalibrator for all tensors).

Expected values come from the oracle (pinned on the reference: tests/test_oracle_pinning.py, tests/test_cpu_live_reference.py):
histogram_t / histogram_asym_t -> kl_search / mse_search, quantile_t + the fp32 mean of the batches -> minmax_to_scale_offset, and
minmax_t / minmax_c -> minmax_to_scale_offset.  Where the reference raises (int(nan) for an asymmetric offset, the power-of-two of a NaN or
inf scale) the device returns the IEEE result -- a NaN or +inf scale, a NaN offset -- and the oracle's `ieee=True` says so (DESIGN.md §2).
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BATCHES = 8


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


def f32(v):
    return np.asarray(v, dtype=np.float32).reshape(-1)


def assert_same(got, want, msg):
    """fp32 bit equality, except that every NaN equals every NaN and +0 equals -0 (an offset of -0.0 is rint(-0.0 / scale))."""
    g, w = f32(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got), f32(want)
    ok = (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w)) | ((g == 0) & (w == 0))
    if not ok.all():
        i = int(np.flatnonzero(~ok)[0])
        raise AssertionError(f'{msg}: {int((~ok).sum())} of {g.size} differ, first at {i}: {g[i]!r} vs {w[i]!r}')


def py_max(a, b):
    return max(a, b)                                       # written out so the argument order of range.py is visible at the call sites


# ------------------------------------------------------------------------------------------------ configs and data
MIN_SCALE = 'OBSERVER_MIN_SCALE_MANUL_OVERRIDE'
KL_BINS = 'OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE'
CONFIGS = {
    'int8_sym': dict(sym=True, qmin=-128, qmax=127, bits=8),
    'uint8_asym': dict(sym=False, qmin=0, qmax=255, bits=8),
    'int4_sym': dict(sym=True, qmin=-8, qmax=7, bits=4),
    'uint4_asym': dict(sym=False, qmin=0, qmax=15, bits=4),
    'pow2_sym': dict(sym=True, qmin=-128, qmax=127, bits=8, pow2=True),
    'pow2_asym': dict(sym=False, qmin=0, qmax=255, bits=8, pow2=True),
    'min_scale_1e-3': dict(sym=True, qmin=-128, qmax=127, bits=8, detail={MIN_SCALE: 1e-3}),
    'min_scale_2^-20_pow2_asym': dict(sym=False, qmin=0, qmax=255, bits=8, pow2=True, detail={MIN_SCALE: 2.0 ** -20}),
    'kl_bins_1024': dict(sym=True, qmin=-128, qmax=127, bits=8, detail={KL_BINS: 1024}),
    'kl_bins_16384': dict(sym=True, qmin=-128, qmax=127, bits=8, detail={KL_BINS: 16384}),
}
DATA = ('randn', 'relu', 'negative', 'zero', 'constant', 'single', 'tiny', 'huge', 'inf', 'nan')


def batches_of(kind: str, seed: int):
    r = np.random.RandomState(seed)
    shape = (1, 1, 1, 1) if kind == 'single' else (2, 3, 7, 9)
    out = []
    for b in range(BATCHES):
        x = r.standard_normal(shape).astype(np.float32) * np.float32(1 + b % 3)
        if kind == 'relu': x = np.maximum(x, 0)
        elif kind == 'negative': x = -np.abs(x) - np.float32(0.25)
        elif kind == 'zero': x[:] = 0
        elif kind == 'constant': x[:] = np.float32(0.7)
        elif kind == 'tiny': x *= np.float32(1e-12)                          # 2 * max / 255 < 1e-8: the scale clamps to the minimum
        elif kind == 'huge': x = np.where(x > 0, np.float32(3e38), np.float32(-3e38)) * np.float32(0.5 + 0.5 * (b % 2))
        elif kind == 'inf':
            if b in (2, 5): x.reshape(-1)[r.randint(x.size)] = np.inf
            if b == 5: x.reshape(-1)[r.randint(x.size)] = -np.inf
        elif kind == 'nan':
            if b == 3: x.reshape(-1)[r.randint(x.size)] = np.nan
        out.append(np.ascontiguousarray(x, np.float32))
    return out


class Net(torch.nn.Module):
    """x -> LeakyReLU -> Sigmoid: three observed activations (the input, the LeakyReLU output, the Sigmoid output), nothing that mixes
    elements, so the degenerate inputs reach the observers as they are.  The parameter only tells calibrate_arena which device to use."""

    def __init__(self):
        super().__init__()
        self.leaky, self.sig = torch.nn.LeakyReLU(0.5), torch.nn.Sigmoid()
        self.anchor = torch.nn.Parameter(torch.zeros(1))

    def forward(self, x):
        return self.sig(self.leaky(x))


def executor_with(cfg_spec: dict):
    from ppq_b200 import LinearQuantizationConfig
    from ppq_b200.executor import TorchExecutor
    ex = TorchExecutor(Net().cuda(), torch.zeros(2, 3, 7, 9, device='cuda'))
    proto = LinearQuantizationConfig(symmetrical=cfg_spec['sym'], power_of_2=cfg_spec.get('pow2', False), quant_min=cfg_spec['qmin'],
                                     quant_max=cfg_spec['qmax'], num_of_bits=cfg_spec['bits'])
    for c in ex.observed_configs():
        c.policy, c.quant_min, c.quant_max, c.num_of_bits = proto.policy, proto.quant_min, proto.quant_max, proto.num_of_bits
        c.detail = dict(cfg_spec.get('detail', {}))
    return ex


def observed_tensors(data):
    """Per observed slot, the host copies of the tensors the observers see, batch by batch (the forward's own collect list)."""
    ex = executor_with(CONFIGS['int8_sym'])
    per_slot = None
    for x in data:
        _, ts = ex.forward(x, collect=True)
        if per_slot is None: per_slot = [[] for _ in ts]
        for k, t in enumerate(ts): per_slot[k].append(t.cpu().numpy().copy())
    return per_slot


def expected(oracle, algo: str, spec: dict, xs):
    """Oracle chain for one observed tensor (its batches `xs`): (scale, offset) as the device must render them."""
    sym, qmin, qmax, bits_, pow2 = spec['sym'], spec['qmin'], spec['qmax'], spec['bits'], spec.get('pow2', False)
    thr = spec.get('detail', {}).get(MIN_SCALE, 1e-8)
    mm = [oracle.minmax_t(x) for x in xs]
    if any(math.isnan(float(lo)) for lo, _ in mm):
        vmin = vmax = math.nan                                      # the collectors poison both slots on NaN (and so does the reference's torch.min)
    else:
        vmin, vmax = min(float(lo) for lo, _ in mm), max(float(hi) for _, hi in mm)
    if algo == 'minmax':
        return oracle.minmax_to_scale_offset(vmin, vmax, qmin, qmax, sym, pow2, thr, ieee=True)
    if algo == 'percentile':
        pairs = torch.tensor(np.stack([oracle.quantile_t(x, 0.9999) for x in xs]), dtype=torch.float32, device='cuda')
        mean = pairs.mean(dim=0).cpu()                             # range.py:369: the fp32 mean over [batches, 2] on the tensors' device
        return oracle.minmax_to_scale_offset(float(mean[1]), float(mean[0]), qmin, qmax, sym, pow2, thr, ieee=True)
    bins = spec.get('detail', {}).get(KL_BINS, 4096) if algo == 'kl' else 2048
    hs = (py_max(abs(vmax), abs(vmin)) if sym else (vmax - vmin)) / bins
    hist = np.zeros(bins, np.int32)
    for x in xs:
        if sym: oracle.histogram_t(x, np.float32(hs), hist=hist)
        else: oracle.histogram_asym_t(x, vmin, vmax, hist=hist)
    if algo == 'kl':
        return oracle.kl_search(hist, hs, bits_, pow2, thr, ieee=True)
    return oracle.mse_search(hist, hs, vmin, qmin, qmax, sym, pow2, 8, None, thr, ieee=True)


CASES = [(name, algo) for name in CONFIGS for algo in ('minmax', 'percentile', 'kl', 'mse') if not name.startswith('kl_bins') or algo == 'kl']


@pytest.mark.parametrize('name,algo', CASES, ids=[f'{n}-{a}' for n, a in CASES])
def test_configs_through_hook_and_arena_paths(ext, oracle, name, algo):
    """Both calibration flows render every observed config of the network to the oracle chain's scale and offset, bit for bit, for every
    data kind; asymmetric KL raises PermissionError in both, as upstream; the arena refuses what its symmetric multi-tensor histogram
    cannot serve (asymmetric MSE, more than 12287 bins) before it sees a batch."""
    from ppq_b200.calibration import RuntimeCalibrationPass
    from ppq_b200.core import QuantizationStates
    from ppq_b200.executor import calibrate_arena
    spec = CONFIGS[name]
    arena_refuses = (algo == 'mse' and not spec['sym']) or spec.get('detail', {}).get(KL_BINS, 0) > 12287
    for j, kind in enumerate(DATA):
        if kind == 'nan' and algo == 'percentile': continue        # the select's NaN order is defined by neither the oracle nor a recording
        host = batches_of(kind, 1000 + 17 * j)
        data = [torch.from_numpy(x).cuda() for x in host]
        ex_hook, ex_arena = executor_with(spec), executor_with(spec)
        if algo == 'kl' and not spec['sym']:
            with pytest.raises(PermissionError):
                RuntimeCalibrationPass(method='kl').optimize(graph=ex_hook, dataloader=data, executor=ex_hook, calib_steps=BATCHES)
            with pytest.raises(PermissionError):
                calibrate_arena(ex_arena, data, method='kl')
            return
        RuntimeCalibrationPass(method=algo).optimize(graph=ex_hook, dataloader=data, executor=ex_hook, calib_steps=BATCHES)
        cfgs = ex_hook.observed_configs_all()
        assert all(c.state == QuantizationStates.ACTIVATED for c in cfgs)
        per_slot = observed_tensors(data)
        assert len(per_slot) == len(cfgs) == 3
        want = [expected(oracle, algo, spec, xs) for xs in per_slot]
        for k, (c, (ws, wo)) in enumerate(zip(cfgs, want)):
            assert_same(c.scale, ws, f'hook {name} {algo} {kind} slot {k} scale')
            assert_same(c.offset, wo, f'hook {name} {algo} {kind} slot {k} offset')
        if arena_refuses:
            with pytest.raises(ValueError):
                calibrate_arena(ex_arena, data, method=algo)
            continue
        for deferred in ('auto', False):
            ex_arena = executor_with(spec)
            cal = calibrate_arena(ex_arena, data, method=algo, deferred=deferred)
            for k, (ws, wo) in enumerate(want):
                assert_same(cal.scale[k], ws, f'arena({deferred}) {name} {algo} {kind} slot {k} scale')
                assert_same(cal.offset[k], wo, f'arena({deferred}) {name} {algo} {kind} slot {k} offset')
            assert all(c.state == QuantizationStates.ACTIVATED for c in ex_arena.observed_configs_all())


def test_per_channel_minmax_configs(ext, oracle):
    """Per-channel min-max (hook path; the arena serves per-tensor configs only and says so before the first batch)."""
    from ppq_b200 import LinearQuantizationConfig
    from ppq_b200.executor import calibrate_arena
    from ppq_b200.observer import Observer
    for name, spec in CONFIGS.items():
        if name.startswith('kl_bins'): continue
        thr = spec.get('detail', {}).get(MIN_SCALE, 1e-8)
        for j, kind in enumerate(DATA):
            host = batches_of(kind, 2000 + 31 * j)
            cfg = LinearQuantizationConfig(symmetrical=spec['sym'], power_of_2=spec.get('pow2', False), quant_min=spec['qmin'],
                                           quant_max=spec['qmax'], num_of_bits=spec['bits'], channel_axis=1)
            cfg.detail = dict(spec.get('detail', {}))
            ob = Observer(cfg)
            for x in host: ob.observe(torch.from_numpy(x).cuda())
            ob.render_quantization_config()
            C = host[0].shape[1]
            lo, hi = np.full(C, np.inf, np.float32), np.full(C, -np.inf, np.float32)
            poisoned = np.zeros(C, bool)
            for x in host:
                a, b = oracle.minmax_c(x, 1)
                poisoned |= np.isnan(a)
                lo, hi = np.minimum(lo, a), np.maximum(hi, b)
            want = [oracle.minmax_to_scale_offset(math.nan if p else float(a), math.nan if p else float(b), spec['qmin'], spec['qmax'],
                                                  spec['sym'], spec.get('pow2', False), thr, ieee=True) for a, b, p in zip(lo, hi, poisoned)]
            assert_same(cfg.scale, [s for s, _ in want], f'{name} {kind} scale')
            assert_same(cfg.offset, [o for _, o in want], f'{name} {kind} offset')
    ex = executor_with(CONFIGS['int8_sym'])
    for c in ex.observed_configs():
        c.policy = LinearQuantizationConfig(channel_axis=1).policy; c.channel_axis = 1
    with pytest.raises(ValueError, match='per-tensor'):
        calibrate_arena(ex, NoBatches(), method='minmax')


class NoBatches:
    """A calibration set that fails the test if anything reads it: the arena must refuse a config before the first batch."""

    def __iter__(self):
        raise AssertionError('calibrate_arena read a batch before refusing the configs')


def test_calibrate_arena_refuses_before_the_first_batch(ext):
    from ppq_b200.executor import calibrate_arena
    with pytest.raises(PermissionError):
        calibrate_arena(executor_with(CONFIGS['uint8_asym']), NoBatches(), method='kl')
    with pytest.raises(ValueError, match='symmetric'):
        calibrate_arena(executor_with(CONFIGS['uint8_asym']), NoBatches(), method='mse')
    with pytest.raises(ValueError, match='12287'):
        calibrate_arena(executor_with(CONFIGS['kl_bins_16384']), NoBatches(), method='kl')
    for a, b, field in (('int8_sym', 'uint8_asym', 'symmetrical'), ('int8_sym', 'int4_sym', 'quant_min'), ('int8_sym', 'pow2_sym', 'power_of_2'),
                        ('int8_sym', 'min_scale_1e-3', 'min_scale'), ('int8_sym', 'kl_bins_1024', 'bins')):
        ex = executor_with(CONFIGS[a])
        odd = executor_with(CONFIGS[b]).observed_configs()[1]
        c = ex.observed_configs()[1]
        c.policy, c.quant_min, c.quant_max, c.num_of_bits, c.detail = odd.policy, odd.quant_min, odd.quant_max, odd.num_of_bits, dict(odd.detail)
        with pytest.raises(ValueError, match=field):
            calibrate_arena(ex, NoBatches(), method='kl' if field == 'bins' else 'minmax')


# ------------------------------------------------------------------------------------------------ power-of-two rounding of the scale
def test_minmax_to_scale_offset_power_of_two_rounding(ext, oracle):
    """CUDA's log2 against math.log2 + Decimal: random ranges over 2^-40..2^40, ranges whose double scale is an exact power of two and their
    1-4 fp32-ulp neighbours, and minimum scales at exact powers of two and +-1 double ulp (where ceil(log2(.)) depends on the last bit)."""
    r = np.random.RandomState(404)
    n = 100000
    lo = (-(2.0 ** r.uniform(-40, 40, n)) * (r.rand(n) < 0.8)).astype(np.float32)
    hi = (2.0 ** r.uniform(-40, 40, n) * (r.rand(n) < 0.9)).astype(np.float32)

    def ulps(v, d):                                                # v moved by d fp32 ulps
        v = np.float32(v)
        for _ in range(abs(d)): v = np.nextafter(v, np.float32(np.inf if d > 0 else -np.inf))
        return v
    adv_lo, adv_hi = [], []
    for k in range(-40, 41):
        # 2 * 127.5 * 2^k / 255 and 255 * 2^k / 255 are exact powers of two in double (and 7.5 / 15 for 4-bit)
        for base_lo, base_hi in ((-128.0, 127.5), (0.0, 127.5), (-127.5, 0.0), (0.0, 255.0), (-255.0, 0.0), (-127.5, 127.5), (-8.0, 7.5), (0.0, 15.0)):
            a, b = np.float32(base_lo * 2.0 ** k), np.float32(base_hi * 2.0 ** k)
            for d in range(-4, 5):
                adv_lo.append(a); adv_hi.append(ulps(b, d))
                adv_lo.append(ulps(a, d)); adv_hi.append(b)
    lo, hi = np.concatenate([lo, np.float32(adv_lo)]), np.concatenate([hi, np.float32(adv_hi)])
    dlo, dhi = torch.from_numpy(lo).cuda(), torch.from_numpy(hi).cuda()
    for sym, qmin, qmax in ((True, -128, 127), (False, 0, 255), (True, -8, 7), (False, 0, 15)):
        s, o = ext.MinMax_To_Scale_Offset(dlo, dhi, 1, qmin, qmax, sym, True, 1e-8)
        want = [oracle.minmax_to_scale_offset(float(a), float(b), qmin, qmax, sym, True, 1e-8) for a, b in zip(lo, hi)]
        assert_same(s, [w[0] for w in want], f'pow2 scale sym={sym} {qmin}..{qmax}')
        assert_same(o, [w[1] for w in want], f'pow2 offset sym={sym} {qmin}..{qmax}')
    # minimum scales at and next to exact powers of two: a zero range clamps to them
    z = torch.zeros(1, device='cuda')
    for k in range(-60, 11):
        p = 2.0 ** k
        for thr in (p, math.nextafter(p, 0.0), math.nextafter(p, math.inf), p * math.sqrt(2.0)):
            for sym, qmin, qmax in ((True, -128, 127), (False, 0, 255)):
                s, o = ext.MinMax_To_Scale_Offset(z, z, 1, qmin, qmax, sym, True, thr)
                ws, wo = oracle.minmax_to_scale_offset(0.0, 0.0, qmin, qmax, sym, True, thr)
                assert_same(s, ws, f'min scale {thr!r}'); assert_same(o, wo, f'min scale {thr!r} offset')


def test_kl_power_of_two_half_up(ext, oracle):
    """KL rounds the exponent half-up: scales landing exactly on 2^k, and next to 2^(k+1/2) (the minimum scale set to the double nearest
    sqrt(2) * 2^k and its neighbours, with a histogram scale small enough that the clamp applies)."""
    r = np.random.RandomState(77)
    hist = np.floor(r.gamma(0.8, 50.0, size=2048) * np.exp(-np.arange(2048) / 400.0)).astype(np.int32)
    H = torch.from_numpy(np.stack([hist] * 3)).cuda()
    _, _, best, _ = oracle.kl_search(hist, 1.0, 8, return_losses=True)
    for k in range(-30, 20):
        # unclamped scale = (best / bins) * hs * (bins / 128) == 2^k exactly for hs = 2^k * 128 / best when that is an fp32
        hs32 = np.float32(2.0 ** k * 128 / best)
        hss = [hs32, np.nextafter(hs32, np.float32(np.inf)), np.nextafter(hs32, np.float32(0))]
        hs = torch.tensor(hss, dtype=torch.float32, device='cuda')
        s, b = ext.KL_Search(H, 2048, hs, None, 8, True, 1e-30)
        assert b.tolist() == [best] * 3
        assert_same(s, [oracle.kl_scale(best, 2048, float(h), 8, True, 1e-30) for h in hss], f'KL pow2 at 2^{k}')
        mid = (2.0 ** k) * math.sqrt(2.0)
        for thr in (mid, math.nextafter(mid, 0.0), math.nextafter(mid, math.inf), math.nextafter(math.nextafter(mid, 0.0), 0.0)):
            tiny = torch.full((3,), 1e-30, dtype=torch.float32, device='cuda')
            s, _ = ext.KL_Search(H, 2048, tiny, None, 8, True, thr)
            assert_same(s, [oracle.kl_scale(best, 2048, 1e-30, 8, True, thr)] * 3, f'KL pow2 near 2^{k}.5: {thr!r}')


def test_non_finite_ranges(ext, oracle):
    """NaN and +-inf ranges through MinMax_To_Scale_Offset and Hist_Scale_From_MinMax: Python's max() order of range.py (a NaN range stays
    NaN instead of clamping to the minimum scale) and the IEEE result where the reference raises."""
    nan, inf = math.nan, math.inf
    pairs = [(nan, nan), (-inf, inf), (-inf, 1.0), (-1.0, inf), (0.0, inf), (-inf, 0.0), (-3e38, 3e38), (nan, 1.0), (-1.0, nan), (0.0, 0.0), (2.0, 5.0)]
    lo = torch.tensor([p[0] for p in pairs], dtype=torch.float32, device='cuda')
    hi = torch.tensor([p[1] for p in pairs], dtype=torch.float32, device='cuda')
    for sym, qmin, qmax in ((True, -128, 127), (False, 0, 255), (True, -8, 7), (False, 0, 15)):
        for pow2 in (False, True):
            s, o = ext.MinMax_To_Scale_Offset(lo, hi, 1, qmin, qmax, sym, pow2, 1e-8)
            want = [oracle.minmax_to_scale_offset(float(np.float32(a)), float(np.float32(b)), qmin, qmax, sym, pow2, 1e-8, ieee=True) for a, b in pairs]
            assert_same(s, [w[0] for w in want], f'scale sym={sym} pow2={pow2}')
            assert_same(o, [w[1] for w in want], f'offset sym={sym} pow2={pow2}')
    mm = torch.stack([lo, hi], dim=1).contiguous()
    for sym in (True, False):
        hs = ext.Hist_Scale_From_MinMax(mm, sym, 4096)
        want = [(py_max(abs(float(np.float32(b))), abs(float(np.float32(a)))) if sym else float(np.float32(b)) - float(np.float32(a))) / 4096
                for a, b in pairs]
        assert_same(hs, want, f'hist scale sym={sym}')


# ------------------------------------------------------------------------------------------------ the search and count kernels on their own
def kl_table(r, bins, n=3):
    hs = []
    for kind in range(n):
        base = r.gamma(0.6 + 0.5 * kind, 40.0, size=bins) * np.exp(-np.arange(bins) / (bins / (1.5 + 2 * kind)))
        if kind == 1: base[bins // 3:] = 0
        if kind == 2: base[r.rand(bins) < 0.6] = 0
        hs.append(np.floor(base).astype(np.int32))
    mm = np.array([[-r.uniform(0.1, 3), r.uniform(0.1, 3)] for _ in range(n)], np.float32)
    return hs, mm


def test_kl_search_bits_bins_pow2_and_min_scale(ext, oracle):
    """KL_Search for bits 2..8 and 256..16384 bins, with and without power-of-two and a minimum-scale override, both kernels, tables of
    several histograms each with its own min/max row.  The argmin may only move on a numerical tie of the losses (DESIGN.md §2 deviation 2)."""
    r = np.random.RandomState(95)
    for bins in (256, 512, 2048, 4096, 8192, 16384):
        for bits_ in range(2, 9):
            if bins >= 8192 and bits_ < 4: continue                 # 2048+ candidates per histogram: the oracle would take minutes
            qb = 2 ** (bits_ - 1)
            hists, mm = kl_table(r, bins)
            H, MM = torch.from_numpy(np.stack(hists)).cuda(), torch.from_numpy(mm).cuda()
            hs_dev = torch.zeros(len(hists), device='cuda')
            ref = [oracle.kl_search(h, 1.0, bits_, return_losses=True) for h in hists]
            for variant in (0, 1):
                ext.set_variant('kl_search', variant)
                try:
                    for pow2 in (False, True):
                        for thr in (1e-8, 2e-3):
                            s, b = ext.KL_Search(H, bins, hs_dev, MM, bits_, pow2, thr)
                            for i, (_, _, wb, losses) in enumerate(ref):
                                hs = py_max(abs(float(mm[i, 1])), abs(float(mm[i, 0]))) / bins
                                got = int(b[i])
                                if got != wb:
                                    assert abs(losses[got // qb - 1] - losses[wb // qb - 1]) <= 1e-12 * max(1.0, abs(losses[wb // qb - 1])), \
                                        (bins, bits_, variant, i, got, wb)
                                    continue
                                assert_same(s[i], oracle.kl_scale(wb, bins, hs, bits_, pow2, thr), f'KL {bins} bins {bits_} bits v{variant} pow2={pow2} {thr}')
                finally:
                    ext.set_variant('kl_search', 0)


def test_kl_search_rejects_bins_the_reference_rejects(ext):
    H = torch.ones(1, 4100, dtype=torch.int32, device='cuda')
    hs = torch.full((1,), 0.01, device='cuda')
    for bits_ in (8, 4, 3):                                        # 4100 % 128, 4100 % 8 != 0; 4100 % 4 == 0 works
        if 4100 % 2 ** (bits_ - 1) == 0: continue
        for variant in (0, 1):
            ext.set_variant('kl_search', variant)
            try:
                with pytest.raises(RuntimeError):
                    ext.KL_Search(H, 4100, hs, None, bits_, False, 1e-8)
            finally:
                ext.set_variant('kl_search', 0)
    s, b = ext.KL_Search(H, 4100, hs, None, 3, False, 1e-8)
    assert int(b[0]) % 4 == 0


def memo_loss(oracle, h):
    """oracle.compute_mse_loss of one histogram, memoised by candidate: the searches of several configs revisit the same candidates."""
    h64, cache = np.ascontiguousarray(h, np.int64), {}

    def loss(_hist, start, step, end):
        key = (start, step, end)
        if key not in cache: cache[key] = oracle.compute_mse_loss(h64, start, step, end)
        return cache[key]
    return loss


def test_mse_search_configs(ext, oracle):
    """MSE_Search: 4- and 8-bit, sym and asym, interval 1 / 8 / 16, bins = the level count, 2048 and 11264, power-of-two on and off, vmin
    below, at and above 0 (asymmetric with vmin > 0: only the min-max fallback candidate survives), random, flat and single-bin
    histograms, the minimum-scale override."""
    r = np.random.RandomState(123)
    for bits_, bins_list in ((4, (16, 2048)), (8, (256, 2048, 11264))):
        for bins in bins_list:
            hists = [(r.gamma(0.6, 300.0, size=bins) * (r.rand(bins) > 0.3)).astype(np.int32), np.full(bins, 7, np.int32), np.zeros(bins, np.int32)]
            hists[2][bins // 5] = 1000
            losses = [memo_loss(oracle, h) for h in hists]
            for sym in (True, False):
                qmin, qmax = (-(2 ** (bits_ - 1)), 2 ** (bits_ - 1) - 1) if sym else (0, 2 ** bits_ - 1)
                if bins < qmax - qmin + 1: continue
                for interval in (1, 8, 16):
                    # asym vmin < 0 close to 0: a few dozen starts survive (the host oracle walks every candidate); a wide negative side
                    # only where that stays a few thousand candidates
                    mms = [(-2.0, 1.5), (0.0, 3.0), (0.4, 3.0)] if sym else \
                        [(-0.02, 3.0), (0.0, 3.0), (0.4, 3.0)] + ([(-2.0, 1.5)] if bins <= 2048 and interval >= 8 else [])
                    H = torch.from_numpy(np.stack([h for h in hists for _ in mms])).cuda()
                    MM = torch.tensor([m for _ in hists for m in mms], dtype=torch.float32, device='cuda')
                    for pow2, thr in ((False, 1e-8), (True, 1e-8), (False, 0.05)):
                        s, o = ext.MSE_Search(H, bins, MM, qmin, qmax, sym, pow2, thr, interval)
                        want = []
                        for h, loss in zip(hists, losses):
                            for lo, hi in mms:
                                lo32, hi32 = float(np.float32(lo)), float(np.float32(hi))
                                hs = (py_max(abs(hi32), abs(lo32)) if sym else (hi32 - lo32)) / bins
                                want.append(oracle.mse_search(h, hs, lo32, qmin, qmax, sym, pow2, interval, loss, thr))
                        tag = f'MSE {bits_} bits {bins} bins sym={sym} interval={interval} pow2={pow2} thr={thr}'
                        assert_same(s, [w[0] for w in want], tag + ' scale')
                        assert_same(o, [w[1] for w in want], tag + ' offset')


def test_mse_search_rejects_bin_counts(ext):
    MM = torch.tensor([[-1.0, 1.0]], device='cuda')
    for bins, qmin, qmax in ((255, -128, 127), (15, 0, 15), (11265, -128, 127), (12288, 0, 255)):
        with pytest.raises(RuntimeError):
            ext.MSE_Search(torch.ones(1, bins, dtype=torch.int32, device='cuda'), bins, MM, qmin, qmax, qmin < 0, False, 1e-8, 8)


def test_histogram_device_scale_above_shared_memory_bins(ext, oracle):
    """Histogram_T_DeviceScale above 12287 bins (global-atomic fallback) == oracle.histogram_t, including a histogram scale of 0 and NaN."""
    r = np.random.RandomState(12288)
    x = (r.standard_normal(200003) * 3).astype(np.float32)
    x[:3] = (np.inf, -np.inf, np.nan)
    xd = torch.from_numpy(x).cuda()
    for bins in (12287, 12288, 16384, 20000):
        for hs in (np.float32(12.0 / bins), np.float32(0.0), np.float32(np.nan), np.float32(1e-30)):
            for clip in (True, False):
                h = torch.zeros(bins, dtype=torch.int32, device='cuda')
                ext.Histogram_T_DeviceScale(xd, torch.tensor([hs], device='cuda'), clip, h)
                assert np.array_equal(h.cpu().numpy(), oracle.histogram_t(x, hs, bins, clip)), (bins, hs, clip)
