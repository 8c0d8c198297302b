"""Live pinning of the CPU oracle against the REAL reference package, imported from /root/reference where that exists (the build
container; skipped elsewhere -- the committed fixtures in tests/golden/ are what travels).  Unlike the fixtures these cases are
generated at run time from a seed: a fixed default keeps the suite deterministic, `PPQ_FUZZ_SEED=random` (or a number) draws a fresh
one -- 26 different seeds ran clean when this was written -- so the oracle cannot be fitted to a fixed vector set.
CPU only: reference CPU / torch path (USING_CUDA_KERNEL = False) against oracle/."""
import math
import os
import sys
import time

import numpy as np
import pytest
import torch

REF = os.environ.get('PPQ_REFERENCE_ROOT', '/root/reference')


@pytest.fixture(scope='module')
def ref():
    if not os.path.isdir(os.path.join(REF, 'ppq')):
        pytest.skip('reference package not present on this machine')
    os.environ['PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION'] = 'python'
    from unittest.mock import MagicMock
    for m in ['onnx', 'onnx.helper', 'onnx.numpy_helper', 'onnx.mapping', 'onnx.checker', 'onnx.shape_inference']:
        sys.modules.setdefault(m, MagicMock())
    if REF not in sys.path: sys.path.insert(0, REF)
    import ppq
    from ppq.core import PPQ_CONFIG
    assert PPQ_CONFIG.USING_CUDA_KERNEL is False
    torch.set_num_threads(1)
    return ppq


@pytest.fixture(scope='module')
def seed():
    env = os.environ.get('PPQ_FUZZ_SEED', '20260923')
    s = time.time_ns() % (2 ** 31) if env == 'random' else int(env)
    print(f'PPQ_FUZZ_SEED={s}')
    return s


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def activated(cfg, scale, offset):
    from ppq.core import QuantizationStates
    cfg.scale, cfg.offset, cfg.state = torch.as_tensor(scale, dtype=torch.float32), torch.as_tensor(offset, dtype=torch.float32), QuantizationStates.ACTIVATED
    return cfg


def test_linear_fake_quant_per_tensor_and_per_channel(ref, oracle, seed):
    from ppq.core import RoundingPolicy
    from ppq.lib import LinearQuantizationConfig
    from ppq.quantization.qfunction.linear import PPQLinearQuant_toInt, PPQLinearQuantFunction
    r = np.random.RandomState(seed)
    modes = [RoundingPolicy.ROUND_HALF_EVEN, RoundingPolicy.ROUND_HALF_UP, RoundingPolicy.ROUND_HALF_DOWN,
             RoundingPolicy.ROUND_HALF_TOWARDS_ZERO, RoundingPolicy.ROUND_HALF_FAR_FORM_ZERO]
    for it in range(24):
        shape = tuple(int(v) for v in r.randint(1, 9, size=r.randint(1, 5)))
        x = (r.standard_normal(shape) * 10 ** r.uniform(-2, 2)).astype(np.float32)
        x.reshape(-1)[:: 7] = np.round(x.reshape(-1)[:: 7] * 2) / 2                     # ties
        sym = bool(r.randint(2)); bits_ = int(r.choice([4, 8]))
        qmin, qmax = (-(1 << (bits_ - 1)), (1 << (bits_ - 1)) - 1) if sym else (0, (1 << bits_) - 1)
        mode = modes[it % len(modes)]
        # per tensor
        s = np.float32(10 ** r.uniform(-3, 0)); o = np.float32(0 if sym else r.randint(qmin, qmax + 1))
        cfg = activated(LinearQuantizationConfig(symmetrical=sym, quant_min=qmin, quant_max=qmax, rounding=mode), s, o)
        want = PPQLinearQuantFunction(torch.from_numpy(x), cfg).numpy()
        got = oracle.linear_quant_t_torchpath(x, s, o, qmin, qmax, mode.value)
        assert np.array_equal(bits(got), bits(want)), (seed, it, 'LT', shape, mode)
        if mode == RoundingPolicy.ROUND_HALF_EVEN:
            got_dev, q_dev = oracle.linear_quant_t(x, s, o, qmin, qmax, 0, return_int=True)  # device semantics agree for integral offsets
            assert np.array_equal(bits(got_dev), bits(want)), (seed, it, 'LT device semantics')
            assert np.array_equal(q_dev, PPQLinearQuant_toInt(torch.from_numpy(x), cfg).numpy().astype(np.int32)), (seed, it, 'toInt')
        # per channel
        if len(shape) >= 2:
            axis = int(r.randint(len(shape))); C = shape[axis]
            sc = (10 ** r.uniform(-3, 0, size=C)).astype(np.float32)
            oc = np.zeros(C, np.float32) if sym else r.randint(qmin, qmax + 1, size=C).astype(np.float32)
            cfgc = activated(LinearQuantizationConfig(symmetrical=sym, quant_min=qmin, quant_max=qmax, rounding=mode, channel_axis=axis), sc, oc)
            wantc = PPQLinearQuantFunction(torch.from_numpy(x), cfgc).numpy()
            gotc = oracle.linear_quant_c_torchpath(x, sc, oc, axis, qmin, qmax, mode.value)
            assert np.array_equal(bits(gotc), bits(wantc)), (seed, it, 'LC', shape, axis, mode)


def test_scalar_rounding_and_scale_offset(ref, oracle, seed):
    from ppq.core import RoundingPolicy
    from ppq.lib import LinearQuantizationConfig
    from ppq.quantization.observer.range import minmax_to_scale_offset
    from ppq.utils.round import ppq_numerical_round, ppq_round_to_power_of_2
    r = np.random.RandomState(seed + 1)
    for mode in (RoundingPolicy.ROUND_HALF_EVEN, RoundingPolicy.ROUND_HALF_UP, RoundingPolicy.ROUND_HALF_DOWN, RoundingPolicy.ROUND_HALF_TOWARDS_ZERO,
                 RoundingPolicy.ROUND_HALF_FAR_FORM_ZERO, RoundingPolicy.ROUND_TO_NEAR_INT, RoundingPolicy.ROUND_UP):
        for v in list(r.uniform(-50, 50, size=40)) + [k + 0.5 for k in range(-6, 6)] + [0.0, -0.0, 1e-9, -1e-9]:
            assert oracle.numerical_round(float(v), mode.value) == ppq_numerical_round(float(v), mode), (seed, mode, v)
    for mode in (RoundingPolicy.ROUND_HALF_UP, RoundingPolicy.ROUND_UP):
        for v in list(10 ** r.uniform(-8, 4, size=60)) + [1.0, 2.0, 0.5, 3.0, 0.75, 1.5]:
            assert oracle.round_to_power_of_2(float(v), mode.value) == ppq_round_to_power_of_2(float(v), mode), (seed, mode, v)
    for it in range(200):
        lo = float(np.float32(r.uniform(-20, 5) * 10 ** r.uniform(-3, 1))); hi = float(np.float32(lo + abs(r.uniform(0, 30)) * 10 ** r.uniform(-3, 1)))
        if it % 17 == 0: lo, hi = 0.0, 0.0                                                # degenerate range -> min scale
        sym = bool(r.randint(2)); pow2 = bool(r.randint(2)); bits_ = int(r.choice([4, 8]))
        qmin, qmax = (-(1 << (bits_ - 1)), (1 << (bits_ - 1)) - 1) if sym else (0, (1 << bits_) - 1)
        cfg = LinearQuantizationConfig(symmetrical=sym, quant_min=qmin, quant_max=qmax, power_of_2=pow2)
        want = minmax_to_scale_offset(lo, hi, cfg)
        got = oracle.minmax_to_scale_offset(lo, hi, qmin, qmax, sym, pow2)
        assert (float(got[0]), float(got[1])) == (float(want[0]), float(want[1])), (seed, it, lo, hi, sym, pow2, bits_)


def test_kl_and_mse_search_on_random_histograms(ref, oracle, seed):
    from ppq.core import QuantizationStates
    from ppq.lib import LinearQuantizationConfig
    from ppq.quantization.observer.range import TorchHistObserver, TorchMSEObserver
    r = np.random.RandomState(seed + 2)
    for it in range(6):
        bins = 4096
        kind = it % 3
        if kind == 0: hist = r.poisson(np.linspace(400, 0.01, bins) ** 1.2).astype(np.int64)
        elif kind == 1: hist = (r.poisson(3.0, size=bins) * (r.rand(bins) < 0.3)).astype(np.int64)       # sparse
        else:
            hist = np.zeros(bins, np.int64); hist[: 64] = r.randint(0, 10 ** 6, size=64); hist[r.randint(64, bins, 20)] = r.randint(1, 50, size=20)
        hs = float(10 ** r.uniform(-5, -1))
        for nbits in (8, 4):
            cfg = LinearQuantizationConfig(symmetrical=True, num_of_bits=nbits, quant_min=-(1 << (nbits - 1)), quant_max=(1 << (nbits - 1)) - 1, calibration='kl')
            ob = TorchHistObserver(watch_on=None, quant_cfg=cfg)
            want = ob.hist_to_scale_offset(histogram=torch.tensor(hist.astype(np.int32)), hist_bins=bins, hist_scale=hs, config=cfg)
            got = oracle.kl_search(hist, hs, nbits)
            assert (float(got[0]), float(got[1])) == (float(want[0]), float(want[1])), (seed, it, nbits, kind)
    for it in range(4):
        bins = 2048
        hist = r.poisson(np.linspace(200, 0.05, bins)).astype(np.int64)
        if it % 2: hist = hist[::-1].copy()
        for sym in (True, False):
            qmin, qmax = (-128, 127) if sym else (0, 255)
            cfg = LinearQuantizationConfig(symmetrical=sym, quant_min=qmin, quant_max=qmax, calibration='mse')
            ob = TorchMSEObserver(watch_on=None, quant_cfg=cfg)
            ob._min, ob._max = (-3.0, 5.0)
            hs = (max(abs(ob._min), abs(ob._max)) if sym else (ob._max - ob._min)) / bins
            want = ob.hist_to_scale_offset(histogram=torch.tensor(hist.astype(np.int32)), hist_bins=bins, hist_scale=hs, config=cfg)
            got = oracle.mse_search(hist, hs, ob._min, qmin, qmax, sym, loss_fn=oracle.mse_loss_python_twin)
            assert (np.float32(got[0]), float(got[1])) == (np.float32(want[0]), float(want[1])), (seed, it, sym)
    assert cfg.state == QuantizationStates.INITIAL


def test_observers_end_to_end(ref, oracle, seed):
    """ppq.lib.Observer (CPU path) on fresh data: min/max per tensor and per channel, percentile (kthvalue indices of the CPU branch), and the
    two-phase KL / MSE observers, whose histogram (torch.histc on the CPU branch) is fed to the oracle's search."""
    from ppq.lib import LinearQuantizationConfig, Observer
    r = np.random.RandomState(seed + 3)
    for it, algo in enumerate(('minmax', 'percentile', 'kl', 'mse', 'minmax', 'mse')):
        sym = (it % 2 == 0) or algo == 'kl'
        relu = bool(r.randint(2))
        shape = (int(r.randint(1, 4)), int(r.randint(2, 9)), int(r.randint(5, 15)), int(r.randint(5, 15)))
        data = [(np.maximum(x, 0) if relu else x) for x in ((r.standard_normal(shape) * 10 ** r.uniform(-1, 1)).astype(np.float32) for _ in range(3))]
        qmin, qmax = (-128, 127) if sym else (0, 255)
        cfg = LinearQuantizationConfig(symmetrical=sym, quant_min=qmin, quant_max=qmax, calibration=algo)
        ob = Observer(cfg)
        for x in data: ob.observe(torch.from_numpy(x))
        ob.render_quantization_config()
        lo = min(float(oracle.minmax_t(x)[0]) for x in data); hi = max(float(oracle.minmax_t(x)[1]) for x in data)
        if algo in ('kl', 'mse'):
            for x in data: ob.observe(torch.from_numpy(x))
            hist, hs = ob._hist.numpy().copy(), float(ob._hist_scale)
            assert (float(ob._min), float(ob._max)) == (lo, hi), (seed, it)
            ob.render_quantization_config()
            s, o = oracle.kl_search(hist, hs, 8) if algo == 'kl' else oracle.mse_search(hist, hs, lo, qmin, qmax, sym, loss_fn=oracle.mse_loss_python_twin)
        elif algo == 'percentile':
            pairs = []
            for x in data:
                v = np.sort(x.reshape(-1)); n = v.size
                pairs.append([v[min(int(n * 0.9999), n - 1)], v[max(0, int(n * (1 - 0.9999)))]])
            m = torch.tensor(np.array(pairs, np.float32)).mean(dim=0)
            s, o = oracle.minmax_to_scale_offset(m[1].item(), m[0].item(), qmin, qmax, sym)
        else:
            s, o = oracle.minmax_to_scale_offset(lo, hi, qmin, qmax, sym)
        assert (np.float32(s), np.float32(o)) == (np.float32(cfg.scale.item()), np.float32(cfg.offset.item())), (seed, it, algo, sym, relu, shape)
    # per-channel symmetric min/max on a weight (ParameterQuantizePass path)
    for axis in (0, 1):
        w = (r.standard_normal((int(r.randint(2, 20)), int(r.randint(2, 20)), 3, 3)) * 0.1).astype(np.float32)
        cfg = LinearQuantizationConfig(symmetrical=True, channel_axis=axis, calibration='minmax')
        ob = Observer(cfg); ob.observe(torch.from_numpy(w)); ob.render_quantization_config()
        lo, hi = oracle.minmax_c(w, axis)
        so = [oracle.minmax_to_scale_offset(float(a), float(b), -128, 127, True) for a, b in zip(lo, hi)]
        assert np.array_equal(np.float32([s for s, _ in so]), cfg.scale.numpy().reshape(-1)), (seed, axis)
        assert np.array_equal(np.float32([o for _, o in so]), cfg.offset.numpy().reshape(-1)), (seed, axis)


def test_search_configs_vs_reference(ref, oracle, seed, monkeypatch):
    """The oracle is the expected value of tests/test_gpu_calibration_configs.py for every calibration config, so it is pinned on the real
    searches for each: power-of-two, 4-bit sym / asym, OBSERVER_MIN_SCALE_MANUL_OVERRIDE, OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE, the MSE
    interval, zero and constant ranges."""
    import ppq.quantization.observer.range as rng
    from ppq.lib import LinearQuantizationConfig
    from ppq.quantization.observer.range import TorchHistObserver, TorchMSEObserver, minmax_to_scale_offset
    r = np.random.RandomState(seed + 4)

    def config(sym, bits_, pow2, min_scale=None, kl_bins=None, algo='minmax'):
        qmin, qmax = (-(1 << (bits_ - 1)), (1 << (bits_ - 1)) - 1) if sym else (0, (1 << bits_) - 1)
        cfg = LinearQuantizationConfig(symmetrical=sym, quant_min=qmin, quant_max=qmax, num_of_bits=bits_, power_of_2=pow2, calibration=algo)
        if min_scale is not None: cfg.detail['OBSERVER_MIN_SCALE_MANUL_OVERRIDE'] = min_scale
        if kl_bins is not None: cfg.detail['OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE'] = kl_bins
        return cfg, qmin, qmax

    # minmax_to_scale_offset: zero, constant and tiny ranges, powers of two at the minimum scale
    ranges = [(0.0, 0.0), (0.7, 0.7), (-0.7, -0.7), (-1e-12, 2e-12), (-127.5, 127.5), (0.0, 255.0 * 2 ** -20)]
    ranges += [(float(np.float32(-abs(a))), float(np.float32(abs(b)))) for a, b in (2.0 ** r.uniform(-30, 30, size=(40, 2)))]
    for lo, hi in ranges:
        for sym in (True, False):
            for bits_ in (4, 8):
                for pow2 in (False, True):
                    for ms in (None, 1e-3, 2.0 ** -20, math.nextafter(2.0 ** -20, 1.0)):
                        cfg, qmin, qmax = config(sym, bits_, pow2, ms)
                        want = minmax_to_scale_offset(lo, hi, cfg)
                        got = oracle.minmax_to_scale_offset(lo, hi, qmin, qmax, sym, pow2, 1e-8 if ms is None else ms)
                        assert (float(got[0]), float(got[1])) == (float(want[0]), float(want[1])), (seed, lo, hi, sym, bits_, pow2, ms)
    # KL: bin override, 4-bit, power of two, minimum scale, flat (constant data) and single-bin (zero range) histograms
    for bins in (1024, 2048):
        hists = [r.poisson(np.linspace(300, 0.01, bins)).astype(np.int64), np.full(bins, 5, np.int64), np.zeros(bins, np.int64)]
        hists[2][0] = 10 ** 5
        for hist in hists:
            for bits_ in (4, 8):
                for pow2, ms, hs in ((False, None, 1e-3), (True, None, 1e-3), (True, None, 2.0 ** -12 * 3), (False, 0.05, 1e-3), (True, 2.0 ** -20, 0.0)):
                    cfg, _, _ = config(True, bits_, pow2, ms, kl_bins=bins, algo='kl')
                    ob = TorchHistObserver(watch_on=None, quant_cfg=cfg)
                    assert ob._hist_bins == bins
                    want = ob.hist_to_scale_offset(histogram=torch.tensor(hist.astype(np.int32)), hist_bins=bins, hist_scale=hs, config=cfg)
                    got = oracle.kl_search(hist, hs, bits_, pow2, 1e-8 if ms is None else ms)
                    assert (float(got[0]), float(got[1])) == (float(want[0]), float(want[1])), (seed, bins, bits_, pow2, ms, hs)
    # MSE: 4-bit, asym / sym, interval, power of two, minimum scale, zero and constant ranges
    bins = 512
    for it in range(3):
        hist = r.poisson(np.linspace(50, 0.05, bins)).astype(np.int64)
        if it == 1: hist = np.full(bins, 3, np.int64)
        if it == 2: hist = np.zeros(bins, np.int64); hist[bins // 4] = 77
        for sym in (True, False):
            for bits_ in (4, 8):
                for interval in (1, 8, 16):
                    for pow2, ms, (lo, hi) in ((False, None, (-3.0, 5.0)), (True, None, (-0.05, 5.0)), (False, 2.0 ** -20, (0.0, 0.0)),
                                               (True, 1e-3, (0.7, 0.7)), (False, None, (0.4, 2.0))):
                        cfg, qmin, qmax = config(sym, bits_, pow2, ms, algo='mse')
                        monkeypatch.setattr(rng, 'OBSERVER_MSE_COMPUTE_INTERVAL', interval)
                        ob = TorchMSEObserver(watch_on=None, quant_cfg=cfg)
                        ob._min, ob._max = lo, hi
                        hs = (max(abs(hi), abs(lo)) if sym else (hi - lo)) / bins
                        want = ob.hist_to_scale_offset(histogram=torch.tensor(hist.astype(np.int32)), hist_bins=bins, hist_scale=hs, config=cfg)
                        got = oracle.mse_search(hist, hs, lo, qmin, qmax, sym, pow2, interval, oracle.mse_loss_python_twin, 1e-8 if ms is None else ms)
                        assert (np.float32(got[0]), float(got[1])) == (np.float32(want[0]), float(want[1])), (seed, it, sym, bits_, interval, pow2, ms, lo, hi)
