"""Every collector launch route against the oracle, exactly, at the edges of each route.

The routes come from the host restatement in tests/test_cpu_collector_routes.py; each case names the kernel, grid, block and shared memory
it is meant to reach, and test_profiled_kernel_is_the_mirrored_route checks them against what the profiler saw, so a case cannot drift off
its route when a threshold changes.  The calls go through the C ABI so that inputs can sit at any element offset.  Every histogram and
min/max output is carved out of a sentinel-filled buffer (a write outside the bins or the slots shows up as a changed guard byte) and is
pre-filled with counts / earlier extremes, so accumulation is checked too.  The expected value is always the oracle, on the fp32 data or on
the exact fp32 upcast of fp16 / bf16 data.

Data: values at fl(k hs) and one ulp either side for k in {0, 1, bins - 1, bins, bins + 1}, quotients one ulp either side of 2^31 (where the
exact division hands over to div.rn), signed zeros, infinities, NaN payloads of both signs, subnormals and +-FLT_MAX.  Scales: an ordinary
one, 0, +inf, NaN, 1e-40, 2^-60 and the float below, 2^60 and the float above, and a negative scale and -0.0 (dropped under clip, bin 0
without it: DESIGN §2, deviation 9).
"""
import contextlib
import ctypes
import json
import os
import re
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_cpu_collector_routes import (BF16, BIG_BINS, F16, F32, HIST_BINS, K_MAX_SMEM_BINS, K_ROW_CHUNK, NEG_SCALES, ROUTE_CASES, SCALE_EDGES, case_id,
                                       channel_geometry, dscale_route, half_split, hist_route, histogram_c_launch, minmax_c_launch,
                                       minmax_t_launch, multi_stream_grid, scale_value)

pytestmark = pytest.mark.gpu

GUARD = 256
V, I, L, Fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
TORCH_DT = {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}
BASE_SCALE = np.float32(0.0371)                                 # not a power of two
ALL_SCALES = ('ordinary',) + SCALE_EDGES + NEG_SCALES


@pytest.fixture(scope='module')
def cabi():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    lib = ctypes.CDLL(os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so'))
    sig = {'ppq_b200_histogram_t': [V, L, Fl, I, V, L, V],
           'ppq_b200_histogram_asym_t_dt': [V, I, L, Fl, Fl, I, V, L, V],
           'ppq_b200_histogram_t_dscale_dt': [V, I, L, V, I, V, L, V],
           'ppq_b200_histogram_c': [V, L, L, I, Fl, I, V, L, V],
           'ppq_b200_minmax_t_dt': [V, I, L, V, V],
           'ppq_b200_minmax_c_dt': [V, I, L, L, I, V, V, V],
           'ppq_b200_multi_histogram_t_dt': [V, I, L, I, V, I, V, L, V],
           'ppq_b200_set_variant': [ctypes.c_char_p, I]}
    for name, args in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, ctypes.c_int
    return lib


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


@pytest.fixture(scope='module')
def sms():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.cuda.get_device_properties(0).multi_processor_count


def stream():
    return V(torch.cuda.current_stream().cuda_stream)


@contextlib.contextmanager
def histogram_variant(cabi, v):
    assert cabi.ppq_b200_set_variant(b'histogram', v) == 0
    try:
        yield
    finally:
        cabi.ppq_b200_set_variant(b'histogram', 0)


_PATTERN = ((np.arange(251) * 37 + 0x5B) & 0xFF).astype(np.uint8)


class Guarded:
    """An output initialised to `init` at byte offset `off` inside a sentinel-filled device buffer."""

    def __init__(self, init, off=0):
        init = np.ascontiguousarray(init)
        self.dtype, self.shape = init.dtype, init.shape
        self.off, self.nbytes = GUARD + off, init.nbytes
        self.init = np.resize(_PATTERN, self.off + self.nbytes + GUARD)
        self.init[self.off:self.off + self.nbytes] = init.reshape(-1).view(np.uint8)
        self.buf = torch.from_numpy(self.init.copy()).cuda()
        self.ptr = self.buf.data_ptr() + self.off

    def read(self, what=''):
        torch.cuda.synchronize()
        b = self.buf.cpu().numpy()
        lo, hi = self.off, self.off + self.nbytes
        assert np.array_equal(b[:lo], self.init[:lo]), f'{what}: a byte before the output changed'
        assert np.array_equal(b[hi:], self.init[hi:]), f'{what}: a byte after the output changed'
        return b[lo:hi].copy().view(self.dtype).reshape(self.shape)


def dev_at(x32, dtype, off):
    """`x32` in `dtype` on the device, its first element `off` elements past an allocation's start.  Returns (keep-alive, pointer, the
    exact fp32 values the kernel reads)."""
    t = torch.from_numpy(np.ascontiguousarray(x32).reshape(-1)).to(TORCH_DT[dtype])
    up = t.float().numpy()
    buf = torch.cat([torch.zeros(off, dtype=t.dtype), t, torch.zeros(8, dtype=t.dtype)]).cuda()
    return buf, buf.data_ptr() + off * t.element_size(), up


def assert_hist(got, want, what):
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got.reshape(-1) != want.reshape(-1))
        raise AssertionError(f'{what}: {bad.size} bins differ, first at {bad[0]}: {got.reshape(-1)[bad[0]]} vs {want.reshape(-1)[bad[0]]}')


# ---- inputs --------------------------------------------------------------------------------------------------------------------------
def _bits(u):
    return np.uint32(u).view(np.float32)


SPECIALS = np.float32([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -1e-40, 3.4028235e38, -3.4028235e38])
NANS = np.array([_bits(0x7FC00000), _bits(0xFFC00000), _bits(0x7FC00123), _bits(0xFFFFFFFF), _bits(0x7F800001), _bits(0xFF800002)], np.float32)


def edge_values(hs, bins):
    """fl(k hs) and its neighbours for the bin edges, both signs, and quotients next to 2^31."""
    a = abs(np.float32(hs))
    if not np.isfinite(a) or a == 0:
        a = BASE_SCALE
    out = []
    for k in (0, 1, bins - 1, bins, bins + 1, 2.0 ** 31 - 128, 2.0 ** 31, 2.0 ** 31 + 256):
        v = np.float32(np.float64(k) * np.float64(a))
        for w in (v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))):
            out += [w, -w]
    return np.array(out, np.float32)


def hist_data(r, n, hs, bins):
    """n values spread over the bins of scale hs, with the edges, the specials and the NaNs strided through them."""
    a = abs(np.float32(hs))
    if not np.isfinite(a) or a == 0 or a < 1e-37:
        a = BASE_SCALE
    x = (r.standard_normal(n) * (float(a) * bins / 2.5)).astype(np.float32)
    sp = np.concatenate([edge_values(hs, bins), SPECIALS, NANS])
    r.shuffle(sp)
    if n <= sp.size:
        return sp[:n].copy() if n < 10 else np.concatenate([sp[:n // 2], x[n // 2:]])
    step = max(1, n // sp.size)
    idx = (np.arange(sp.size) * step + r.randint(0, step, size=sp.size)) % n
    x[idx] = sp
    return x


def prefill(r, shape):
    return r.randint(0, 1000, size=shape).astype(np.int32)


# ---- one call of each entry, guarded -------------------------------------------------------------------------------------------------
def run_hist_t(cabi, oracle, c, r, hs, clip, x32=None):
    n, bins, off = c['n'], c['bins'], c['off']
    x32 = hist_data(r, n, hs, bins) if x32 is None else x32
    keep, xp, up = dev_at(x32, F32, off)
    init = prefill(r, bins)
    g = Guarded(init, 4 * (bins % 3))
    what = f'{case_id(c)} hs {hs!r} clip {clip}'
    with histogram_variant(cabi, c['variant']):
        assert cabi.ppq_b200_histogram_t(xp, n, float(hs), int(clip), g.ptr, bins, stream()) == 0, what
        got = g.read(what)
    assert_hist(got, oracle.histogram_t(up, hs, clip_outliers=clip, hist=init.copy()), what)


def run_hist_asym(cabi, oracle, c, r, vmin, vmax, clip, x32=None):
    n, bins, off, dt = c['n'], c['bins'], c['off'], c['dtype']
    if x32 is None:
        lo, hi = (vmin, vmax) if np.isfinite(vmin) and np.isfinite(vmax) else (-1.0, 1.0)
        mid, half = (np.float64(lo) + np.float64(hi)) / 2, max(abs(np.float64(hi) - np.float64(lo)), 1e-3)
        x32 = (mid + r.standard_normal(n) * half * 0.6).astype(np.float32)           # about a quarter lies outside [vmin, vmax]
        hs = np.float32(np.float32(np.float32(vmax) - np.float32(vmin)) / np.float32(bins))
        sp = np.concatenate([np.float32([vmin, vmax]), np.nextafter(np.float32([vmin, vmax]), np.float32(np.inf)),
                             np.nextafter(np.float32([vmin, vmax]), np.float32(-np.inf)), SPECIALS, NANS,
                             (np.float32(vmin) + np.arange(4) * hs).astype(np.float32)])
        sp = sp[:n]
        x32[np.linspace(0, n - 1, sp.size).astype(int)] = sp
    keep, xp, up = dev_at(x32, dt, off)
    init = prefill(r, bins)
    g = Guarded(init, 4 * (bins % 3))
    what = f'{case_id(c)} range [{vmin!r}, {vmax!r}] clip {clip}'
    with histogram_variant(cabi, c['variant']):
        assert cabi.ppq_b200_histogram_asym_t_dt(xp, dt, n, float(vmin), float(vmax), int(clip), g.ptr, bins, stream()) == 0, what
        got = g.read(what)
    assert_hist(got, oracle.histogram_asym_t(up, vmin, vmax, clip_outliers=clip, hist=init.copy()), what)


def run_dscale(cabi, oracle, c, r, hs, clip):
    n, bins, off, dt = c['n'], c['bins'], c['off'], c['dtype']
    keep, xp, up = dev_at(hist_data(r, n, hs, bins), dt, off)
    sd = torch.tensor([hs], dtype=torch.float32, device='cuda')
    init = prefill(r, bins)
    g = Guarded(init, 4 * (bins % 3))
    what = f'{case_id(c)} hs {hs!r} clip {clip}'
    assert cabi.ppq_b200_histogram_t_dscale_dt(xp, dt, n, sd.data_ptr(), int(clip), g.ptr, bins, stream()) == 0, what
    assert_hist(g.read(what), oracle.histogram_t(up, hs, clip_outliers=clip, hist=init.copy()), what)


def run_hist_c(cabi, oracle, c, r, hs, clip, x32=None):
    shape, axis, bins = c['shape'], c['axis'], c['bins']
    n, (epc, C) = c['n'], channel_geometry(shape, axis)
    x32 = hist_data(r, n, hs, bins) if x32 is None else x32
    keep, xp, up = dev_at(x32, F32, c['off'])
    init = prefill(r, (C, bins))
    g = Guarded(init, 4)
    what = f'{case_id(c)} hs {hs!r} clip {clip}'
    assert cabi.ppq_b200_histogram_c(xp, n, epc, C, float(hs), int(clip), g.ptr, bins, stream()) == 0, what
    assert_hist(g.read(what), oracle.histogram_c(up.reshape(shape), axis, hs, clip_outliers=clip, hist=init.copy()), what)


def same_extreme(got, want, nan_bits):
    """The device value of one min or max slot against the oracle's: equal as floats, or the device's canonical NaN of that slot."""
    if np.isnan(want):
        return int(np.float32(got).view(np.uint32)) == nan_bits
    return got == want


def expect_slot(oracle, data_extreme, prior, which):
    lo, hi = oracle.minmax_t(np.float32([data_extreme, prior]))
    return lo if which == 0 else hi


def minmax_data(r, n):
    x = (r.standard_normal(n) * 3).astype(np.float32)
    sp = np.concatenate([SPECIALS[:2], SPECIALS[4:8]])
    k = min(n, sp.size)
    x[r.choice(n, k, replace=False)] = sp[:k]
    return x


def run_minmax_t(cabi, oracle, c, r, x32=None, prior=(np.inf, -np.inf)):
    n, off, dt = c['n'], c['off'], c['dtype']
    x32 = minmax_data(r, n) if x32 is None else x32
    keep, xp, up = dev_at(x32, dt, off)
    g = Guarded(np.float32(prior), 4)
    what = f'{case_id(c)} prior {prior}'
    assert cabi.ppq_b200_minmax_t_dt(xp, dt, n, g.ptr, stream()) == 0, what
    got = g.read(what)
    lo, hi = oracle.minmax_t(up)
    assert same_extreme(got[0], expect_slot(oracle, lo, prior[0], 0), 0xFFC00000), (what, got, lo, hi)
    assert same_extreme(got[1], expect_slot(oracle, hi, prior[1], 1), 0x7FC00000), (what, got, lo, hi)
    return got, up


def run_minmax_c(cabi, oracle, c, r, x32=None, prior=None):
    shape, axis, dt = c['shape'], c['axis'], c['dtype']
    n, (epc, C) = c['n'], channel_geometry(shape, axis)
    x32 = minmax_data(r, n) if x32 is None else x32
    keep, xp, up = dev_at(x32, dt, c['off'])
    pl, ph = prior if prior is not None else (np.full(C, np.inf, np.float32), np.full(C, -np.inf, np.float32))
    gl, gh = Guarded(np.float32(pl), 4), Guarded(np.float32(ph), 8)
    what = f'{case_id(c)}'
    assert cabi.ppq_b200_minmax_c_dt(xp, dt, n, epc, C, gl.ptr, gh.ptr, stream()) == 0, what
    lo, hi = gl.read(what), gh.read(what)
    wl, wh = oracle.minmax_c(up.reshape(shape), axis)
    for ch in range(C):
        assert same_extreme(lo[ch], expect_slot(oracle, wl[ch], pl[ch], 0), 0xFFC00000), (what, ch, lo[ch], wl[ch])
        assert same_extreme(hi[ch], expect_slot(oracle, wh[ch], ph[ch], 1), 0x7FC00000), (what, ch, hi[ch], wh[ch])
    return lo, hi, up


# ---- A: every case of the route table -----------------------------------------------------------------------------------------------
def cases_of(entry):
    return [c for c in ROUTE_CASES if c['entry'] == entry]


def test_hist_t_route_cases_vs_oracle(cabi, oracle):
    """Histogram_T under every `histogram` variant (0-8), every size of the table, clip both ways, an ordinary and an edge scale."""
    r = np.random.RandomState(100)
    for i, c in enumerate(cases_of('hist_t')):
        for clip in (True, False):
            run_hist_t(cabi, oracle, c, r, BASE_SCALE, clip)
        run_hist_t(cabi, oracle, c, r, scale_value(ALL_SCALES[i % len(ALL_SCALES)], BASE_SCALE), i % 2 == 0)


ASYM_RANGES = [(-1.5, 2.25), (0.0, 1.0), (1.0, 1.0), (2.0, -1.0), (-3e38, 3e38), (float('nan'), 1.0), (-1.0, float('nan')),
               (-np.inf, 1.0), (0.1, 0.1 + 2 ** -20)]


def test_hist_asym_route_cases_vs_oracle(cabi, oracle):
    """Histogram_Asymmetric_T on every route and dtype, with data below vmin and above vmax, vmin == vmax (a scale of 0), vmax < vmin
    (a negative scale), an infinite range (-3e38, 3e38), NaN bounds, clip both ways."""
    r = np.random.RandomState(101)
    for c in cases_of('hist_asym'):
        for vmin, vmax in ASYM_RANGES:
            for clip in (True, False):
                run_hist_asym(cabi, oracle, c, r, np.float32(vmin), np.float32(vmax), clip)


def test_dscale_route_cases_vs_oracle(cabi, oracle):
    r = np.random.RandomState(102)
    for c in cases_of('hist_dscale'):
        for name in ALL_SCALES:
            for clip in (True, False):
                run_dscale(cabi, oracle, c, r, scale_value(name, BASE_SCALE), clip)


def test_hist_c_route_cases_vs_oracle(cabi, oracle):
    """Histogram_C: epc at chunk - 1, chunk, + 1 and 2 chunk + 1, axis first / middle / last, C = 1, more items than CTAs (a CTA zeroes and
    flushes its bins more than once), clip both ways, every scale."""
    r = np.random.RandomState(103)
    for c in cases_of('hist_c'):
        for name in ALL_SCALES:
            for clip in (True, False):
                run_hist_c(cabi, oracle, c, r, scale_value(name, BASE_SCALE), clip)


def test_hist_c_refuses_more_than_12287_bins(cabi):
    """More than 12287 bins are refused before any launch, and nothing is written (DESIGN §2, deviation 7)."""
    x = torch.ones(64, device='cuda')
    for bins in (12288, 16384, 20000):
        g = Guarded(np.zeros((2, bins), np.int32))
        assert cabi.ppq_b200_histogram_c(x.data_ptr(), 64, 32, 2, 0.1, 1, g.ptr, bins, stream()) == 1
        assert not g.read(f'bins {bins}').any()
    g = Guarded(np.zeros((2, K_MAX_SMEM_BINS), np.int32))
    assert cabi.ppq_b200_histogram_c(x.data_ptr(), 64, 32, 2, 0.1, 1, g.ptr, K_MAX_SMEM_BINS, stream()) == 0
    assert g.read().sum() == 64


def test_minmax_t_route_cases_vs_oracle(cabi, oracle):
    r = np.random.RandomState(104)
    for i, c in enumerate(cases_of('minmax_t')):
        run_minmax_t(cabi, oracle, c, r)
        run_minmax_t(cabi, oracle, c, r, prior=(np.float32(0.75), np.float32(-0.75)))
        x = minmax_data(r, c['n'])
        x[(i * 7) % c['n']] = NANS[i % NANS.size]
        run_minmax_t(cabi, oracle, c, r, x32=x)


def test_minmax_c_route_cases_vs_oracle(cabi, oracle):
    """MinMax_C at epc 4095 / 4096 / 4097 / 8193, more items than resident warps, odd epc; then a NaN in one channel, which poisons only
    that channel, and earlier extremes in the slots."""
    r = np.random.RandomState(105)
    for c in cases_of('minmax_c'):
        run_minmax_c(cabi, oracle, c, r)
        epc, C = channel_geometry(c['shape'], c['axis'])
        x = minmax_data(r, c['n'])
        ch = C // 2
        rows = [row for row in range(c['n'] // epc) if row % C == ch]
        row = rows[len(rows) // 2]
        x[row * epc + (epc - 1) // 2] = NANS[(C + epc) % NANS.size]
        # the extremes of the other channels on the last element of a chunk: row ends and kRowChunk boundaries
        for j, row in enumerate(r.choice(c['n'] // epc, min(8, c['n'] // epc), replace=False)):
            if row % C != ch:
                end = min(epc, K_ROW_CHUNK * (1 + j % ((epc + K_ROW_CHUNK - 1) // K_ROW_CHUNK))) - 1
                x[row * epc + end] = np.float32(1e6 if j % 2 else -1e6) * (j + 1)
        lo, hi, up = run_minmax_c(cabi, oracle, c, r, x32=x,
                                  prior=((r.standard_normal(C) * 3).astype(np.float32), (r.standard_normal(C) * 3).astype(np.float32)))
        assert np.isnan(lo[ch]) and np.isnan(hi[ch]), case_id(c)
        assert not np.isnan(np.delete(lo, ch)).any() and not np.isnan(np.delete(hi, ch)).any(), case_id(c)


def test_minmax_signed_zeros_across_ctas(cabi, oracle):
    """Channels of +0 and -0 only, spread over many warps and CTAs: the min slot holds -0 when any -0 is present, the max slot +0 when any
    +0 is (min.NaN / max.NaN and the raw-bit atomics order -0 below +0), whatever order the CTAs publish in."""
    r = np.random.RandomState(106)
    for dt in (F32, F16, BF16):
        shape, axis = [16, 4, 4097], 1
        c = dict(entry='minmax_c', dtype=dt, shape=shape, axis=axis, n=int(np.prod(shape)), off=1, variant=0, route='once')
        x = np.where(r.rand(*shape) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
        x[:, 0] = 0.0                                                   # channel 0: +0 only
        x[:, 1] = -0.0                                                  # channel 1: -0 only
        x[3, 1, 17] = 0.0                                               # ... but one +0
        lo, hi, up = run_minmax_c(cabi, oracle, c, r, x32=x.reshape(-1))
        sign = lambda v: int(np.float32(v).view(np.uint32)) >> 31       # noqa: E731
        xs = up.reshape(shape)
        for ch in range(4):
            v = xs[:, ch].reshape(-1)
            has_neg, has_pos = bool((np.signbit(v)).any()), bool((~np.signbit(v)).any())
            assert lo[ch] == 0 and hi[ch] == 0
            assert sign(lo[ch]) == int(has_neg) and sign(hi[ch]) == int(not has_pos), (dt, ch, lo[ch], hi[ch])
        ct = dict(entry='minmax_t', dtype=dt, n=x.size, off=3, variant=0, route='')
        got, _ = run_minmax_t(cabi, oracle, ct, r, x32=x.reshape(-1))
        assert sign(got[0]) == 1 and sign(got[1]) == 0


# ---- B: the scale edges on every symmetric entry ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('variant', list(range(9)))
def test_hist_t_scale_edges_under_every_variant(cabi, oracle, variant):
    """Histogram_T with hist_scale 0, +inf, NaN, 1e-40, 2^-60 and the float below, 2^60 and the float above, negative and -0.0, for bins
    1 .. 20000, clip both ways, under set_variant('histogram', variant)."""
    r = np.random.RandomState(200 + variant)
    for bins in HIST_BINS + BIG_BINS:
        for n, off in ((4099, 1), (3 * 65536 + 5, 0)):
            c = dict(entry='hist_t', dtype=F32, n=n, bins=bins, variant=variant, off=off, route=hist_route(n, bins, variant)[0])
            for name in ALL_SCALES:
                for clip in (True, False):
                    run_hist_t(cabi, oracle, c, r, scale_value(name, BASE_SCALE), clip)


def test_hist_t_negative_scale_keeps_inside_the_bins(cabi, oracle):
    """A negative or -0.0 hist_scale: every count lands in bin 0 without clip (or stays in the sentinel-guarded buffer with clip, where
    nothing is counted but NaNs and zeros), on the shared-memory and the global-atomic routes."""
    r = np.random.RandomState(201)
    x = hist_data(r, 70001, BASE_SCALE, 4096)
    for bins in (1, 4096, 16384):
        for variant in (0, 3):
            for hs in (np.float32(-BASE_SCALE), np.float32(-0.0), np.float32(-1e30)):
                c = dict(entry='hist_t', dtype=F32, n=x.size, bins=bins, variant=variant, off=0, route='')
                for clip in (True, False):
                    run_hist_t(cabi, oracle, c, r, hs, clip, x32=x)
                want = oracle.histogram_t(x, hs, bins, False)
                assert want[0] == x.size and not want[1:].any()


def test_multi_histogram_scale_edges_in_one_table(cabi, oracle):
    """One Multi_Histogram_T table whose slots carry every edge scale next to ordinary slots, per dtype; each slot's histogram is the
    oracle's for its tensor and scale, and the arena outside the slots keeps its sentinel."""
    r = np.random.RandomState(202)
    for c in cases_of('multi_hist'):
        dt, bins = c['dtype'], c['bins']
        names = [s for name in ALL_SCALES for s in (name, 'ordinary')]
        ns = [(37 * k + 5) % 9000 + 1 + (70000 if k % 5 == 0 else 0) for k in range(len(names))]
        tensors, keep = [], []
        for k, (name, n) in enumerate(zip(names, ns)):
            hs = scale_value(name, np.float32(BASE_SCALE * (1 + k / 7)))
            buf, ptr, up = dev_at(hist_data(r, n, hs, bins), dt, k % 8)
            keep.append(buf)
            tensors.append((ptr, n, hs, up))
        slots = np.arange(len(names))[::-1].copy()                     # slots in reverse order of the rows
        descs = torch.tensor([[p, n, int(s)] for (p, n, hs, up), s in zip(tensors, slots)], dtype=torch.int64, device='cuda')
        scales = np.zeros(len(names), np.float32)
        for (p, n, hs, up), s in zip(tensors, slots):
            scales[s] = hs
        sd = torch.from_numpy(scales).cuda()
        for clip in (True, False):
            init = prefill(r, (len(names), bins))
            g = Guarded(init, 4)
            what = f'{case_id(c)} clip {clip}'
            rc = cabi.ppq_b200_multi_histogram_t_dt(descs.data_ptr(), len(names), max(ns), dt, sd.data_ptr(), int(clip), g.ptr, bins, stream())
            assert rc == 0, what
            got = g.read(what)
            for (p, n, hs, up), s in zip(tensors, slots):
                assert_hist(got[s], oracle.histogram_t(up, hs, clip_outliers=clip, hist=init[s].copy()), f'{what} slot {s} hs {hs!r} n {n}')


# ---- C: the half-precision oracle, directly ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dt', [F16, BF16])
def test_half_collectors_equal_the_oracle_on_the_upcast(cabi, oracle, dt):
    """fp16 / bf16 inputs against the oracle on their exact upcast (not only against the fp32 kernel): values at the half grid's own bin
    edges, half specials and NaNs, every head / tail length."""
    r = np.random.RandomState(300 + dt)
    hs = np.float32(0.0371)
    k = np.arange(-4100, 4100, dtype=np.float32)
    x = (k * hs).astype(np.float32)
    xh = torch.from_numpy(x).to(TORCH_DT[dt]).float().numpy()
    for off in range(8):
        for n in (8 * 1000 + off, 8 * 1000 + 7 - off):
            data = np.concatenate([xh, np.float32([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 6e-8, -6e-8])])[:n]
            r.shuffle(data)
            c = dict(entry='hist_dscale', dtype=dt, n=n, bins=4096, off=off, variant=0, route='smem')
            keep, xp, up = dev_at(data, dt, off)
            for clip in (True, False):
                for s in (hs, np.float32(-hs)):
                    sd = torch.tensor([s], device='cuda')
                    init = prefill(r, 4096)
                    g = Guarded(init, 4)
                    assert cabi.ppq_b200_histogram_t_dscale_dt(xp, dt, n, sd.data_ptr(), int(clip), g.ptr, 4096, stream()) == 0
                    assert_hist(g.read(), oracle.histogram_t(up, s, clip_outliers=clip, hist=init.copy()), f'{case_id(c)} {s} {clip}')
                init = prefill(r, 2048)
                g = Guarded(init, 8)
                assert cabi.ppq_b200_histogram_asym_t_dt(xp, dt, n, -100.0, 50.0, int(clip), g.ptr, 2048, stream()) == 0
                assert_hist(g.read(), oracle.histogram_asym_t(up, -100.0, 50.0, clip_outliers=clip, hist=init.copy()), f'asym d{dt} n{n} o{off}')
            ct = dict(entry='minmax_t', dtype=dt, n=n, off=off, variant=0, route='')
            assert half_split(n, off)[0] == (8 - off) % 8
            run_minmax_t(cabi, oracle, ct, r, x32=data)


# ---- D: the binding -----------------------------------------------------------------------------------------------------------------------
def test_binding_entries_equal_the_oracle(ext, oracle):
    """The torch entries over the same kernels: Histogram_T, Histogram_Asymmetric_T(_Half), Histogram_C, Histogram_T_DeviceScale, MinMax_T,
    MinMax_C and Multi_Histogram_T, each accumulating into a pre-filled output, on an edge scale and on a negative one."""
    r = np.random.RandomState(400)
    x = hist_data(r, 3 * 65536 + 7, BASE_SCALE, 2048)
    xd = torch.from_numpy(x).cuda()
    for hs in (BASE_SCALE, np.float32(0.0), np.float32(2.0 ** 60), np.float32(-BASE_SCALE)):
        for clip in (True, False):
            for bins in (2048, 16384):
                init = prefill(r, bins)
                h = torch.from_numpy(init.copy()).cuda()
                ext.Histogram_T(xd, float(hs), clip, h)
                assert_hist(h.cpu().numpy(), oracle.histogram_t(x, hs, clip_outliers=clip, hist=init.copy()), f'Histogram_T {hs} {clip} {bins}')
                h = torch.from_numpy(init.copy()).cuda()
                ext.Histogram_T_DeviceScale(xd, torch.tensor([hs], device='cuda'), clip, h)
                assert_hist(h.cpu().numpy(), oracle.histogram_t(x, hs, clip_outliers=clip, hist=init.copy()), f'DeviceScale {hs} {clip} {bins}')
            x4 = x[:4 * 1100 * 9].reshape(4, 1100, 3, 3)
            init = prefill(r, (1100, 256))
            h = torch.from_numpy(init.copy()).cuda()
            ext.Histogram_C(torch.from_numpy(x4).cuda(), 1, float(hs), clip, h)
            assert_hist(h.cpu().numpy(), oracle.histogram_c(x4, 1, hs, clip_outliers=clip, hist=init.copy()), f'Histogram_C {hs} {clip}')
            descs = torch.tensor([[xd.data_ptr(), x.size, 1], [xd.data_ptr() + 4, 1000, 0]], dtype=torch.int64, device='cuda')
            init = prefill(r, (2, 2048))
            h = torch.from_numpy(init.copy()).cuda()
            ext.Multi_Histogram_T(descs, x.size, torch.tensor([np.float32(0.5), hs], device='cuda'), clip, h, 2048)
            assert_hist(h.cpu().numpy()[1], oracle.histogram_t(x, hs, clip_outliers=clip, hist=init[1].copy()), f'Multi slot 1 {hs} {clip}')
            assert_hist(h.cpu().numpy()[0], oracle.histogram_t(x[1:1001], np.float32(0.5), clip_outliers=clip, hist=init[0].copy()), 'Multi slot 0')
    for clip in (True, False):
        for vmin, vmax in ((-1.0, 1.0), (1.0, -1.0), (0.5, 0.5)):
            init = prefill(r, 2048)
            h = torch.from_numpy(init.copy()).cuda()
            ext.Histogram_Asymmetric_T(vmin, vmax, xd, clip, h)
            assert_hist(h.cpu().numpy(), oracle.histogram_asym_t(x, vmin, vmax, clip_outliers=clip, hist=init.copy()), f'asym {vmin} {vmax}')
            xb = xd.to(torch.bfloat16)
            h = torch.from_numpy(init.copy()).cuda()
            ext.Histogram_Asymmetric_T_Half(vmin, vmax, xb, clip, h)
            assert_hist(h.cpu().numpy(), oracle.histogram_asym_t(xb.float().cpu().numpy(), vmin, vmax, clip_outliers=clip, hist=init.copy()),
                        f'asym bf16 {vmin} {vmax}')
    mm = torch.tensor([np.inf, -np.inf], device='cuda')
    ext.MinMax_T(xd, mm)
    lo, hi = oracle.minmax_t(x)
    assert same_extreme(mm[0].item(), lo, 0xFFC00000) and same_extreme(mm[1].item(), hi, 0x7FC00000)
    x3 = (r.standard_normal((16, 1024, 1, 1)) * 2).astype(np.float32)
    x3[5, 77, 0, 0] = np.nan
    lo_t, hi_t = torch.empty(1024, device='cuda'), torch.empty(1024, device='cuda')
    ext.MinMax_Init(lo_t, hi_t)
    ext.MinMax_C(torch.from_numpy(x3).cuda(), 1, lo_t, hi_t)
    wl, wh = oracle.minmax_c(x3, 1)
    lo, hi = lo_t.cpu().numpy(), hi_t.cpu().numpy()
    assert all(same_extreme(lo[c], wl[c], 0xFFC00000) and same_extreme(hi[c], wh[c], 0x7FC00000) for c in range(1024))


# ---- E: the profiler's view of one case per route ------------------------------------------------------------------------------------------
def mirrored_launch(c, sms):
    e, n, dt = c['entry'], c.get('n'), c['dtype']
    if e == 'hist_t':
        return hist_route(n, c['bins'], c['variant'], F32, sms)
    if e == 'hist_asym':
        return hist_route(n, c['bins'], c['variant'], dt, sms, binop='AsymBin')
    if e == 'hist_dscale':
        return dscale_route(n, c['bins'], dt, sms)
    if e == 'hist_c':
        return histogram_c_launch(n, c['epc'], c['bins'], sms)
    if e == 'minmax_t':
        return minmax_t_launch(n, dt, c['off'], sms)
    if e == 'minmax_c':
        return minmax_c_launch(n, c['epc'], dt, sms)
    return None


def kernel_regex(kernel):
    name, args = kernel
    return re.escape(name) + r'<' + r',\s*'.join(r'(ppqb::)?' + re.escape(a) for a in args) + r'>'


def test_profiled_kernel_is_the_mirrored_route(cabi, oracle, sms):
    """One case per (entry, route, dtype) cell: the kernel the profiler records carries the mirror's name and template arguments, and
    its grid, block and shared memory are the mirror's (the multi-tensor grid for either occupancy the device may report)."""
    from torch.profiler import ProfilerActivity, profile
    picked = {}
    for c in ROUTE_CASES:
        picked.setdefault((c['entry'], c['route'], c['dtype']), c)
    r = np.random.RandomState(500)
    checked = 0
    for key, c in sorted(picked.items(), key=lambda kv: str(kv[0])):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e = c['entry']
            if e == 'hist_t':
                run_hist_t(cabi, oracle, c, r, BASE_SCALE, True)
            elif e == 'hist_asym':
                run_hist_asym(cabi, oracle, c, r, np.float32(-1.5), np.float32(2.25), True)
            elif e == 'hist_dscale':
                run_dscale(cabi, oracle, c, r, BASE_SCALE, False)
            elif e == 'hist_c':
                run_hist_c(cabi, oracle, c, r, BASE_SCALE, True)
            elif e == 'minmax_t':
                run_minmax_t(cabi, oracle, c, r)
            elif e == 'minmax_c':
                run_minmax_c(cabi, oracle, c, r)
            else:
                n = 70001
                buf, ptr, up = dev_at(hist_data(r, n, BASE_SCALE, c['bins']), c['dtype'], 0)
                descs = torch.tensor([[ptr, n, 0]], dtype=torch.int64, device='cuda')
                g = Guarded(np.zeros(c['bins'], np.int32))
                sd = torch.tensor([BASE_SCALE], device='cuda')
                assert cabi.ppq_b200_multi_histogram_t_dt(descs.data_ptr(), 1, n, c['dtype'], sd.data_ptr(), 1, g.ptr, c['bins'], stream()) == 0
                assert_hist(g.read(), oracle.histogram_t(up, BASE_SCALE, c['bins'], True), case_id(c))
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory(prefix='collector_trace_') as d:
            path = os.path.join(d, 'trace.json')
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = [ev for ev in json.load(f).get('traceEvents', []) if ev.get('cat') == 'kernel' and 'ppqb::' in ev.get('name', '')]
        if not events:
            continue
        assert len(events) == 1, (case_id(c), [ev['name'] for ev in events])
        ev, args = events[0], events[0].get('args', {})
        assert {'grid', 'block', 'shared memory'} <= set(args), (case_id(c), args)
        if c['entry'] == 'multi_hist':
            T = {F32: 'float', F16: '__half', BF16: '__nv_bfloat16'}[c['dtype']]
            assert re.search(kernel_regex(('multi_stream_kernel', ('HistOp', T))), ev['name']), (case_id(c), ev['name'])
            assert args['grid'][0] in {multi_stream_grid(1, 70001, k, sms) for k in (1, 2)} and args['block'][0] == 544, (case_id(c), args)
        else:
            route, kernel, grid, block, smem = mirrored_launch(c, sms)
            assert route == c['route'] or sms != 132, (case_id(c), route)
            assert re.search(kernel_regex(kernel), ev['name']), (case_id(c), ev['name'], kernel)
            assert args['grid'] == [grid, 1, 1] and args['block'] == [block, 1, 1], (case_id(c), args, grid, block)
            assert smem <= args['shared memory'] < smem + 1024, (case_id(c), args, smem)
        checked += 1
    if not checked:
        pytest.skip('the profiler recorded no CUDA kernel activity')
    assert checked == len(picked)


# ---- F: the reference's own kernels -------------------------------------------------------------------------------------------------------
@pytest.fixture
def ref(request):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import refcuda
    return refcuda.reference(request.node.nodeid)


def test_bin_edges_and_scale_edges_pinned_to_reference(ref, oracle):
    """The oracle's Histogram_T, Histogram_Asymmetric_T and Histogram_C at bin edges, quotients next to 2^31 and the specials, with scales of
    0, +inf and NaN, asymmetric data outside the range and a reversed range, and Histogram_T above 12287 bins -- against the reference's own
    kernels (recorded on an H100).  Negative scales are undefined there and stay out of this set."""
    r = np.random.RandomState(600)
    for bins in (3, 50, 2048, 16384):
        x = hist_data(r, 20011, BASE_SCALE, bins)
        xd = torch.from_numpy(x).cuda()
        for hs in (BASE_SCALE, np.float32(0.0), np.float32(np.inf), np.float32(np.nan), np.float32(2.0 ** -60)):
            for clip in (True, False):
                h = torch.zeros(bins, dtype=torch.int32, device='cuda')
                ref.Histogram_T(xd, float(hs), clip, h)
                assert_hist(h.cpu().numpy(), oracle.histogram_t(x, hs, bins, clip), f'ref Histogram_T bins {bins} hs {hs} clip {clip}')
        if bins <= 2048:
            for vmin, vmax in ((-1.5, 2.25), (2.0, -1.0), (1.0, 1.0), (-3e38, 3e38), (-0.0371 * 10, 0.0371 * (bins - 10))):
                vmin, vmax = np.float32(vmin), np.float32(vmax)
                for clip in (True, False):
                    h = torch.zeros(bins, dtype=torch.int32, device='cuda')
                    ref.Histogram_Asymmetric_T(float(vmin), float(vmax), xd, clip, h)
                    assert_hist(h.cpu().numpy(), oracle.histogram_asym_t(x, vmin, vmax, bins, clip), f'ref asym [{vmin}, {vmax}] {clip}')
            for shape, axis in (([7, 2858], 0), ([3, 7, 952], 1), ([2858, 7], 1)):
                xs = x[:int(np.prod(shape))].reshape(shape)
                for hs in (BASE_SCALE, np.float32(0.0), np.float32(np.nan)):
                    for clip in (True, False):
                        C = shape[axis]
                        h = torch.zeros(C, bins, dtype=torch.int32, device='cuda')
                        ref.Histogram_C(torch.from_numpy(np.ascontiguousarray(xs)).cuda(), axis, float(hs), clip, h)
                        assert_hist(h.cpu().numpy(), oracle.histogram_c(xs, axis, hs, bins, clip), f'ref Histogram_C {shape} {axis} {hs} {clip}')
