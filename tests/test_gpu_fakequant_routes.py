"""Every fp32 fake-quant launch route against the oracle, bit for bit, at the edges of each route.

The routes, operator families and output types come from the host restatement in tests/test_cpu_fakequant_routes.py; each case names the
kernel it is meant to reach, and test_profiled_kernel_is_the_mirrored_route checks that name against the kernel the profiler saw, so a
case cannot drift off its route when a threshold changes.  The calls go through the C ABI so that x and y can sit at any offset, and y is
always carved out of a larger buffer filled with a sentinel: a store outside the output shows up as a changed guard byte.
"""
import ctypes
import os
import re
import zlib

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_cpu_fakequant_routes import (E4M3_FAST, E4M3_SLOW, FORMATS, OUT_BYTES, ROUTE_CASES, boundary_clips, case_id, channel_route,
                                       family, fp_tmax, y_aligned)

pytestmark = pytest.mark.gpu

F32, F16, BF16 = 0, 1, 2
GUARD = 256                                                    # sentinel bytes on each side of every output
V, I, L, Fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float


@pytest.fixture(scope='module')
def cabi():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    lib = ctypes.CDLL(os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so'))
    sig = {'ppq_b200_linear_quant_t_dt': [V, I, V, L, V, V, I, I, I, V],
           'ppq_b200_linear_quant_c_dt': [V, I, V, L, L, I, V, V, I, I, I, V],
           'ppq_b200_linear_quant_t_toint_dt': [V, I, V, I, L, V, V, I, I, I, V],
           'ppq_b200_linear_quant_c_toint_dt': [V, I, V, I, L, L, I, V, V, I, I, I, V],
           'ppq_b200_float_quant_t_dt': [V, I, V, L, V, V, I, I, Fl, Fl, I, V],
           'ppq_b200_float_quant_c_dt': [V, I, V, L, L, I, V, V, I, I, Fl, Fl, I, V],
           'ppq_b200_multi_linear_quant_c': [V, I, L, I, I, I, V],
           'ppq_b200_multi_linear_quant_t': [V, I, L, I, I, I, V],
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


def stream():
    return V(torch.cuda.current_stream().cuda_stream)


_PATTERN = ((np.arange(251) * 37 + 0x5B) & 0xFF).astype(np.uint8)


def sentinel(nbytes):
    return np.resize(_PATTERN, nbytes)


class Guarded:
    """`nbytes` of output at byte offset `off` inside a sentinel-filled device buffer."""

    def __init__(self, nbytes, off=0):
        self.off, self.nbytes = GUARD + off, nbytes
        self.init = sentinel(self.off + nbytes + GUARD)
        self.buf = torch.from_numpy(self.init.copy()).cuda()
        self.ptr = self.buf.data_ptr() + self.off

    def read(self, dtype, what=''):
        torch.cuda.synchronize()
        b = self.buf.cpu().numpy()
        lo, hi = self.off, self.off + self.nbytes
        assert np.array_equal(b[:lo], self.init[:lo]), f'{what}: a byte before the output changed'
        assert np.array_equal(b[hi:], self.init[hi:]), f'{what}: a byte after the output changed'
        return b[lo:hi].copy().view(dtype)


def dev_at(a, off_elems):
    """A device copy of `a` whose first element sits `off_elems` elements after an allocation's start; returns (keep-alive, pointer)."""
    a = np.ascontiguousarray(a).reshape(-1)
    t = torch.from_numpy(np.concatenate([np.zeros(off_elems, a.dtype), a, np.zeros(4, a.dtype)])).cuda()
    return t, t.data_ptr() + off_elems * a.itemsize


def assert_same(got, want, what):
    g, w = np.ascontiguousarray(got).reshape(-1), np.ascontiguousarray(want).reshape(-1)
    if g.dtype.itemsize == 4:
        g, w = g.view(np.uint32), w.view(np.uint32)
    if not np.array_equal(g, w):
        bad = np.flatnonzero(g != w)
        raise AssertionError(f'{what}: {bad.size} of {g.size} differ, first at {bad[0]}: {g[bad[0]]:#x} vs {w[bad[0]]:#x}')


# ---- inputs ------------------------------------------------------------------------------------------------------------------------
def channel_params(r, C):
    """Per-channel scales with two badly scaled channels (the IEEE slow path of the exact division) and integer offsets."""
    s = (r.rand(C) * 0.1 + 1e-3).astype(np.float32)
    if C >= 3:
        s[1], s[C - 2] = 1e-25, 1e25
    o = r.randint(-5, 6, size=C).astype(np.float32)
    return s, o


def linear_inputs(r, n, s_elem):
    """Random values plus exact ties of x / s, their float neighbours, signed zeros, infinities and NaN."""
    x = (r.standard_normal(n) * 40 * s_elem).astype(np.float32)
    k = (r.randint(-140, 140, size=n) + 0.5).astype(np.float32)
    tie = (k * s_elem).astype(np.float32)
    x[0::5] = tie[0::5]
    x[1::7] = np.nextafter(tie[1::7], np.float32(np.inf))
    x[2::7] = np.nextafter(tie[2::7], np.float32(-np.inf))
    sp = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 3e38, -3e38, 1e-45])
    x[3::11] = sp[np.arange(x[3::11].size) % sp.size]
    return x


def float_inputs(r, n, E, M, s_elem):
    t = float(fp_tmax(E, M))
    x = (r.standard_normal(n) * t / 3 * s_elem).astype(np.float32)
    x[1::5] = (r.standard_normal(x[1::5].size) * 2.0 ** (-(1 << (E - 1)) + 1) * s_elem[1::5]).astype(np.float32)      # sub-normal range
    k = x[2::5].size                                                    # half-way points between two normal grid points, both signs
    mid = 2.0 ** ((1 << (E - 1)) - 1) * (1 + (2 * r.randint(0, 1 << M, size=k) + 1) * 2.0 ** (-M - 1))
    x[2::5] = (np.where(r.rand(k) < 0.5, -1.0, 1.0) * mid * s_elem[2::5]).astype(np.float32)
    sp = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, 3e38, -3e38])
    x[3::13] = sp[np.arange(x[3::13].size) % sp.size]
    return x


# ---- one call of any fp32 entry, guarded ------------------------------------------------------------------------------------------
RANGE_OF_OUT = {'float': (-128, 127), 'int32': (-2 ** 31 + 1, 2 ** 31 - 1), 'int8': (-128, 127)}


def run_case(cabi, oracle, c, r, qrange=None, offsets=None, mode=None, fmt=None, scale_override=None):
    """Runs case `c` of ROUTE_CASES (optionally with another range / offsets / mode / format) through the C ABI and compares with the
    oracle; returns nothing, raises on any difference or changed guard byte."""
    op, ot = c['op'], c['out']
    mode = c['mode'] if mode is None else mode
    fmt = c['fmt'] if fmt is None else fmt
    lo, hi = qrange or RANGE_OF_OUT[ot]
    if c['kind'] == 'C':
        outer, C, epc = c['outer'], c['C'], c['epc']
        n = outer * C * epc
        s, o = channel_params(r, C)
    else:
        n, C, epc = c['n'], 1, c['n']
        s, o = np.float32([0.37]), np.float32([3.0])
    if scale_override is not None:
        s = np.asarray(scale_override, np.float32).reshape(-1)[:C] * np.ones(C, np.float32)
    if offsets is not None:
        o = np.asarray(offsets, np.float32).reshape(-1)[:C] * np.ones(C, np.float32)
    if op in ('FT', 'FC'):
        o = np.where(np.arange(C) % 2 == 0, 0.0, 2.5).astype(np.float32) if offsets is None else o
    s_elem = np.repeat(np.tile(s, n // (C * epc)), epc)
    x = float_inputs(r, n, fmt[0], fmt[1], s_elem) if op in ('FT', 'FC') else linear_inputs(r, n, s_elem)
    xk, xp = dev_at(x, c['x_off'])
    sk, ok = torch.from_numpy(s).cuda(), torch.from_numpy(o).cuda()
    sp, op_ = sk.data_ptr(), ok.data_ptr()
    ob = OUT_BYTES[ot]
    g = Guarded(n * ob, c['y_off'] * ob)
    if op in ('LT', 'LC', 'QT', 'QC'):
        x3 = x.reshape(-1, C, epc)
        want_y, want_q = oracle.linear_quant_c(x3, s, o, 1, lo, hi, mode, return_int=True)
    if op == 'LT':
        rc = cabi.ppq_b200_linear_quant_t_dt(xp, F32, g.ptr, n, sp, op_, lo, hi, mode, stream())
    elif op == 'LC':
        rc = cabi.ppq_b200_linear_quant_c_dt(xp, F32, g.ptr, n, epc, C, sp, op_, lo, hi, mode, stream())
    elif op == 'QT':
        rc = cabi.ppq_b200_linear_quant_t_toint_dt(xp, F32, g.ptr, 8 * ob, n, sp, op_, lo, hi, mode, stream())
    elif op == 'QC':
        rc = cabi.ppq_b200_linear_quant_c_toint_dt(xp, F32, g.ptr, 8 * ob, n, epc, C, sp, op_, lo, hi, mode, stream())
    else:
        E, M, cmin, cmax = fmt
        want_y = oracle.float_quant_c(x.reshape(-1, C, epc), s, o, 1, E, M, cmin, cmax, mode)
        if op == 'FT':
            rc = cabi.ppq_b200_float_quant_t_dt(xp, F32, g.ptr, n, sp, op_, E, M, cmin, cmax, mode, stream())
        else:
            rc = cabi.ppq_b200_float_quant_c_dt(xp, F32, g.ptr, n, epc, C, sp, op_, E, M, cmin, cmax, mode, stream())
    what = f'{case_id(c)} range {lo}..{hi} mode {mode} fmt {fmt}'
    assert rc == 0, what
    if ot == 'float':
        assert_same(g.read(np.float32, what), want_y, what)
    elif ot == 'int32':
        assert_same(g.read(np.int32, what), want_q.astype(np.int32), what)
    else:
        assert_same(g.read(np.uint8, what), (want_q.astype(np.int64) & 0xFF).astype(np.uint8), what)
    del xk


def with_variant(cabi, var, fn):
    cabi.ppq_b200_set_variant(b'linear_quant_c', var)
    try:
        return fn()
    finally:
        cabi.ppq_b200_set_variant(b'linear_quant_c', 0)


SMALL_CASES = [c for c in ROUTE_CASES if c['kind'] == 'C' or c['n'] < 1 << 25]
BIG_CASES = [c for c in ROUTE_CASES if c['kind'] == 'T' and c['n'] >= 1 << 25]


# ---- A: every case of the route table, and the profiler's view of one case per route -------------------------------------------------
def test_route_table_cases_vs_oracle(cabi, oracle):
    r = np.random.RandomState(1)
    for c in SMALL_CASES:
        with_variant(cabi, c.get('variant', 0), lambda: run_case(cabi, oracle, c, r))


KERNEL_OF_ROUTE = {('C', 'seg'): r'ew_channel_seg_kernel<', ('C', 'table4'): r'ew_channel_table_kernel<.*,\s*true>',
                   ('C', 'vec'): r'ew_channel_vec_kernel<', ('C', 'last'): r'ew_channel_last_kernel<',
                   ('C', 'ragged'): r'ew_channel_table_kernel<.*,\s*false>', ('C', 'generic'): r'ew_channel_generic_kernel<',
                   ('T', 'vec8'): r'ew_tensor_kernel<.*,\s*true,\s*8,', ('T', 'vec'): r'ew_tensor_kernel<.*,\s*true,\s*4,',
                   ('T', 'scalar'): r'ew_tensor_kernel<.*,\s*false,'}
OP_OF_FAMILY = {'lin': r'LinearOp<[0-7]>', 'lin_dyn': r'LinearOp<-1>', 'float_fast': r'FloatOp<[0-7],\s*true>',
                'float_slow': r'FloatOp<(0|-1),\s*false>'}


def test_profiled_kernel_is_the_mirrored_route(cabi, oracle):
    """One case per (route, family) cell: the kernel the profiler records must carry the route's name and the family's operator."""
    from torch.profiler import ProfilerActivity, profile
    picked = {}
    for c in ROUTE_CASES:
        key = (c['kind'], c['route'], c['family'])
        if key not in picked and (c['kind'] == 'C' or c['n'] < 1 << 25 or c['route'] == 'vec8'):
            picked[key] = c
    r = np.random.RandomState(2)
    seen_any = False
    for key, c in sorted(picked.items()):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with_variant(cabi, c.get('variant', 0), lambda: run_case(cabi, oracle, c, r))
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if 'ew_' in e.name]
        if not names:
            continue
        seen_any = True
        assert len(set(names)) == 1, (case_id(c), names)
        assert re.search(KERNEL_OF_ROUTE[(c['kind'], c['route'])], names[0]), (case_id(c), names[0])
        assert re.search(OP_OF_FAMILY[c['family']], names[0]), (case_id(c), names[0])
    if not seen_any:
        pytest.skip('the profiler recorded no CUDA kernel activity')


# ---- B: the per-channel matrix -------------------------------------------------------------------------------------------------------
CHANNEL_CASES = {}
for _c in ROUTE_CASES:
    if _c['kind'] == 'C' and _c['op'] == 'LC' and _c['mode'] == 3:
        CHANNEL_CASES[case_id(_c)] = _c

LC_RANGES = ((-128, 127, 'int'), (0, 255, 'half'), (-8, 7, 'int'), (-2 ** 31 + 1, 2 ** 31 - 1, 'large'), (0, 255, 'large'))


def offsets_of(kind, C, r):
    if kind == 'int':
        return r.randint(-5, 6, size=C).astype(np.float32)
    if kind == 'half':
        return (r.randint(0, 255, size=C) + np.where(np.arange(C) % 2, 0.5, -0.5)).astype(np.float32)       # roundf: away from zero
    return np.where(np.arange(C) % 2, 3e9, -1e6).astype(np.float32)


@pytest.mark.parametrize('variant', [0, 1])
@pytest.mark.parametrize('cid', sorted(CHANNEL_CASES))
def test_channel_matrix(cabi, oracle, cid, variant):
    """LC in modes 0-7 and 11 over INT8 / UINT8 / INT4 / full int32 ranges with integer, half-integer and large offsets; toInt in 8 and 32
    bits; FC with a fast and two slow clip ranges -- on the geometry's route under the default variant and under linear_quant_c = 1."""
    c0 = dict(CHANNEL_CASES[cid], variant=variant)
    r = np.random.RandomState(zlib.crc32(cid.encode()) + variant)
    C = c0['C']

    def body():
        for mode in (0, 1, 2, 3, 4, 5, 6, 7, 11):
            lo, hi, ok = LC_RANGES[mode % len(LC_RANGES)]
            run_case(cabi, oracle, dict(c0, op='LC', out='float'), r, (lo, hi), offsets_of(ok, C, r), mode)
        for lo, hi, ok in LC_RANGES:
            run_case(cabi, oracle, dict(c0, op='LC', out='float'), r, (lo, hi), offsets_of(ok, C, r), 11)
        for mode in (0, 1, 4, 11):
            run_case(cabi, oracle, dict(c0, op='QC', out='int8'), r, (-128, 127), offsets_of('int', C, r), mode)
            run_case(cabi, oracle, dict(c0, op='QC', out='int8'), r, (0, 255), offsets_of('half', C, r), mode)
            run_case(cabi, oracle, dict(c0, op='QC', out='int32'), r, (-2 ** 31 + 1, 2 ** 31 - 1), offsets_of('large', C, r), mode)
        for fmt, mode in ((E4M3_FAST, 0), (E4M3_FAST, 4), ((5, 2, -57344.0, 57344.0), 7), (E4M3_SLOW, 0), (E4M3_SLOW, 11),
                          ((4, 3, 0.0, 448.0), 1), ((3, 4, -30.0, 12.5), 6)):
            run_case(cabi, oracle, dict(c0, op='FC', out='float', fmt=fmt), r, mode=mode)

    with_variant(cabi, variant, body)


def test_channel_transposed_input(ext, oracle):
    """The torch entries make a transposed view contiguous before the kernel sees it."""
    r = np.random.RandomState(5)
    m = torch.from_numpy((r.standard_normal((48, 64)) * 3).astype(np.float32)).cuda().t()      # [64, 48], channel axis 0 -> epc 48
    s, o = channel_params(r, 64)
    want = oracle.linear_quant_c(m.contiguous().cpu().numpy(), s, o, 0, -128, 127, 11)
    y = ext.QuantizeTensor_LC(m, torch.from_numpy(s).cuda(), torch.from_numpy(o).cuda(), -128, 127, 0, 11)
    assert_same(y.cpu().numpy(), want, 'transposed LC')
    want = oracle.float_quant_c(m.contiguous().cpu().numpy(), np.abs(s), np.zeros(64, np.float32), 0, 4, 3, -300.0, 300.0, 2)
    y = ext.QuantizeTensor_FC(m, torch.from_numpy(np.abs(s)).cuda(), torch.zeros(64, device='cuda'), 4, 3, -300.0, 300.0, 0, 2)
    assert_same(y.cpu().numpy(), want, 'transposed FC')


# ---- C: per tensor ---------------------------------------------------------------------------------------------------------------------
def test_tensor_unknown_rounding_id(cabi, oracle):
    r = np.random.RandomState(6)
    for c in [c for c in ROUTE_CASES if c['kind'] == 'T' and c['n'] < 1 << 25]:
        if c['family'] in ('lin', 'lin_dyn'):
            run_case(cabi, oracle, c, r, mode=11)
            run_case(cabi, oracle, c, r, qrange=(0, 255), offsets=[127.5], mode=11)
        else:
            run_case(cabi, oracle, c, r, fmt=E4M3_SLOW, mode=11)


@pytest.mark.parametrize('cid', [case_id(c) for c in BIG_CASES])
def test_tensor_eight_deep_loop(cabi, oracle, cid):
    """n >= 2^25 on an aligned base takes the 8-deep vector loop for LinearOp<0>, int32 toInt and the fast FloatOp; 2^25 + 151 leaves a
    partial last warp segment, 2^25 + 3 only a scalar tail; the same tensor one float off takes the scalar loop."""
    c = {case_id(c): c for c in BIG_CASES}[cid]
    run_case(cabi, oracle, c, np.random.RandomState(7))
    torch.cuda.empty_cache()


@pytest.mark.parametrize('variant', [2, 3])
def test_linear_quant_t_launch_shape_variants(ext, oracle, variant):
    r = np.random.RandomState(8)
    x = linear_inputs(r, (1 << 20) + 4 * 37 + 3, np.float32(0.05))
    xd = torch.from_numpy(x).cuda()
    s, o = torch.tensor([0.05], device='cuda'), torch.tensor([0.0], device='cuda')
    ext.set_variant('linear_quant_t', variant)
    try:
        y = ext.QuantizeTensor_LT(xd, s, o, -128, 127, 0)
    finally:
        ext.set_variant('linear_quant_t', 0)
    assert_same(y.cpu().numpy(), oracle.linear_quant_t(x, np.float32(0.05), 0, -128, 127, 0), f'variant {variant}')


# ---- D: the float fast-path boundary ------------------------------------------------------------------------------------------------
MODES = (0, 1, 2, 3, 4, 5, 6, 7, 11)


def clips_of(E, M):
    out = [(float(a), float(b)) for a, b, _ in boundary_clips(E, M)]
    return out + ([(-300.0, 300.0), (-448.0, 240.0), (-500.0, 500.0)] if (E, M) == (4, 3) else [])


@pytest.mark.parametrize('E,M', FORMATS)
def test_float_boundary_vs_oracle(cabi, oracle, E, M):
    """FT with scales 1, 0.3, 2^-7 and offsets 0, 2.5, and FC with those scales and offsets on alternating channels, for every boundary
    clip in every rounding mode -- on both sides of float_fast_path_ok."""
    r = np.random.RandomState(E * 16 + M)
    ct = dict(kind='T', op='FT', out='float', n=4099, x_off=0, y_off=0, mode=0, route='vec', family='')
    cc = dict(kind='C', op='FC', out='float', outer=2, C=6, epc=516, x_off=0, y_off=0, mode=0, variant=0, route='seg', family='')
    for cmin, cmax in clips_of(E, M):
        for mode in MODES:
            for s, o in ((1.0, 0.0), (0.3, 2.5), (2.0 ** -7, 0.0), (0.3, 0.0)):
                run_case(cabi, oracle, ct, r, offsets=[o], mode=mode, fmt=(E, M, cmin, cmax), scale_override=[s])
            run_case(cabi, oracle, cc, r, mode=mode, fmt=(E, M, cmin, cmax),
                     scale_override=np.float32([1.0, 0.3, 2.0 ** -7, 1.0, 0.3, 2.0 ** -7]))


def boundary_inputs(E, M, n=2053):
    r = np.random.RandomState(E * 100 + M)
    t = float(fp_tmax(E, M))
    x = (r.standard_normal(n) * t / 2).astype(np.float32)
    x[1::4] = (r.standard_normal(x[1::4].size) * 2.0 ** (-(1 << (E - 1)) + 1)).astype(np.float32)
    sp = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, t, -t, t * 1.1])
    x[:sp.size] = sp
    return x


@pytest.fixture
def ref(request):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import refcuda
    return refcuda.reference(request.node.nodeid)


@pytest.mark.parametrize('E,M', FORMATS)
def test_float_boundary_oracle_pinned_to_reference(ref, oracle, E, M):
    """The oracle's forward float quantiser on the boundary clips, in every rounding mode, against the reference's own FT / FC kernels
    (recorded on an H100); and LT / LC with an unknown rounding id."""
    x = boundary_inputs(E, M)
    xd = torch.from_numpy(x).cuda()
    x3 = torch.from_numpy(x[:2052].reshape(2, 6, 171)).cuda()
    sc = np.float32([1.0, 0.3, 2.0 ** -7, 1.0, 0.3, 2.0 ** -7]); oc = np.float32([0, 2.5, 0, 2.5, 0, 0])
    for cmin, cmax in clips_of(E, M):
        for mode in MODES:
            y = ref.QuantizeTensor_FT(xd, torch.tensor([0.3], device='cuda'), torch.tensor([2.5], device='cuda'), E, M, cmin, cmax, mode)
            assert_same(y.cpu().numpy(), oracle.float_quant_t(x, 0.3, 2.5, E, M, cmin, cmax, mode), f'FT E{E}M{M} [{cmin}, {cmax}] mode {mode}')
            y = ref.QuantizeTensor_FC(x3, torch.from_numpy(sc).cuda(), torch.from_numpy(oc).cuda(), E, M, cmin, cmax, 1, mode)
            assert_same(y.cpu().numpy(), oracle.float_quant_c(x3.cpu().numpy(), sc, oc, 1, E, M, cmin, cmax, mode),
                        f'FC E{E}M{M} [{cmin}, {cmax}] mode {mode}')
    if (E, M) == (4, 3):
        r = np.random.RandomState(9)
        xl = linear_inputs(r, 2052, np.float32(0.05))
        for lo, hi, o in ((-128, 127, 0.0), (0, 255, 127.5), (-8, 7, 0.0)):
            y = ref.QuantizeTensor_LT(torch.from_numpy(xl).cuda(), torch.tensor([0.05], device='cuda'), torch.tensor([o], device='cuda'), lo, hi, 11)
            assert_same(y.cpu().numpy(), oracle.linear_quant_t(xl, np.float32(0.05), o, lo, hi, 11), f'LT id 11 {lo}..{hi}')
            s6 = np.float32([0.05, 0.1, 0.5, 0.05, 1e-25, 0.2]); o6 = np.full(6, o, np.float32)
            y = ref.QuantizeTensor_LC(torch.from_numpy(xl.reshape(2, 6, 171)).cuda(), torch.from_numpy(s6).cuda(), torch.from_numpy(o6).cuda(),
                                      lo, hi, 1, 11)
            assert_same(y.cpu().numpy(), oracle.linear_quant_c(xl.reshape(2, 6, 171), s6, o6, 1, lo, hi, 11), f'LC id 11 {lo}..{hi}')


# ---- E: weight tables built by hand --------------------------------------------------------------------------------------------------
class Pool:
    """One sentinel-filled device buffer that tensors are carved from at chosen float offsets, with gaps between them."""

    def __init__(self, floats):
        self.init = sentinel(4 * floats).view(np.float32)
        self.t = torch.from_numpy(self.init.copy()).cuda()
        self.base, self.used, self.spans = self.t.data_ptr(), 64, []

    def take(self, n, align_off, gap=64):
        start = (self.used + gap + 3) // 4 * 4 + align_off
        self.used = start + n
        self.spans.append((start, n))
        assert self.used + 64 <= self.init.size
        return start

    def ptr(self, start):
        return self.base + 4 * start


def build_table(r, entries, kind):
    """entries: (n, epc, C, x_off, y_off) -> descriptor table, pools, per-tensor (x, s, o, xs, ys)."""
    total = sum(e[0] for e in entries) + 80 * (len(entries) + 2)
    px, py = Pool(total), Pool(total)
    rows, data = [], []
    for n, epc, C, xo, yo in entries:
        xs, ys = px.take(n, xo), py.take(n, yo)
        x = (r.standard_normal(n) * 3).astype(np.float32)
        if n:
            x[::7] = (np.round(x[::7] * 4) + 0.5).astype(np.float32) * np.float32(0.25)          # ties at scale 0.25
        px.init[xs:xs + n] = x
        s = (r.rand(C) * 0.1 + 0.2).astype(np.float32); s[0] = 0.25
        o = r.randint(-3, 4, size=C).astype(np.float32)
        st, ot = torch.from_numpy(s).cuda(), torch.from_numpy(o).cuda()
        data.append((x, s, o, xs, ys, st, ot, n, epc, C))
        row = [px.ptr(xs), py.ptr(ys), st.data_ptr(), ot.data_ptr(), n]
        rows.append(row + [epc, C] if kind == 'C' else row)
    px.t.copy_(torch.from_numpy(px.init))
    descs = torch.tensor(rows, dtype=torch.int64).cuda()
    return descs, px, py, data


def check_table(cabi, oracle, descs, px, py, data, kind, qmin, qmax, mode, max_n, what):
    py.t.copy_(torch.from_numpy(py.init))
    fn = cabi.ppq_b200_multi_linear_quant_c if kind == 'C' else cabi.ppq_b200_multi_linear_quant_t
    assert fn(V(descs.data_ptr()), descs.shape[0], max_n, qmin, qmax, mode, stream()) == 0, what
    torch.cuda.synchronize()
    got = py.t.cpu().numpy()
    outside = np.ones(got.size, bool)
    for x, s, o, xs, ys, st, ot, n, epc, C in data:
        outside[ys:ys + n] = False
        if n == 0:
            continue
        if kind == 'C':
            want = oracle.linear_quant_c(x.reshape(-1, C, epc), s, o, 1, qmin, qmax, mode).reshape(-1)
        else:
            want = oracle.linear_quant_t(x, s[0], o[0], qmin, qmax, mode)
        assert_same(got[ys:ys + n], want, f'{what} n={n} epc={epc} C={C}')
    assert np.array_equal(got[outside].view(np.uint32), py.init[outside].view(np.uint32)), f'{what}: a write outside every output'
    return got


def single_launches(cabi, px, data, kind, qmin, qmax, mode):
    out = []
    for x, s, o, xs, ys, st, ot, n, epc, C in data:
        if n == 0:
            out.append(None)
            continue
        y = torch.empty(n + 4, device='cuda')
        if kind == 'C':
            rc = cabi.ppq_b200_linear_quant_c_dt(px.ptr(xs), F32, y.data_ptr(), n, epc, C, st.data_ptr(), ot.data_ptr(), qmin, qmax, mode, stream())
        else:
            rc = cabi.ppq_b200_linear_quant_t_dt(px.ptr(xs), F32, y.data_ptr(), n, st.data_ptr(), ot.data_ptr(), qmin, qmax, mode, stream())
        assert rc == 0
        out.append(y[:n].cpu().numpy())
    return out


TABLE_RANGES = ((-128, 127), (0, 255), (-8, 7), (0, 15))
# (n, epc, C): sizes 1, 3, 4, 511, 512, 513, 4099 and epc 1, 3, 4, 9, 512, 516, whole [outer, C, epc] tensors
TABLE_C = [(1, 1, 1), (3, 3, 1), (3, 1, 3), (4, 4, 1), (4, 1, 4), (511, 1, 7), (512, 512, 1), (512, 4, 8), (513, 9, 19), (513, 3, 19),
           (4099, 1, 4099), (4099, 4099, 1), (516 * 3, 516, 3), (516 * 4, 516, 2), (9 * 47 * 2, 9, 47), (4 * 130, 4, 130), (3 * 4 * 5, 3, 4),
           (512 * 5, 512, 5), (512 * 6, 512, 3)]
TABLE_T = [1, 3, 4, 7, 511, 512, 513, 2053, 4099, 4100, 516 * 3]


@pytest.mark.parametrize('kind', ['C', 'T'])
def test_weight_table_by_hand(cabi, oracle, kind):
    """Sizes around the 512-element warp segment, every epc class, x and y offsets chosen independently, empty entries interleaved; every
    rounding id with INT8 / UINT8 / INT4 / UINT4; several max_n (they change the grid and so the CTA spans) give the same bits."""
    r = np.random.RandomState(10 if kind == 'C' else 11)
    geoms = TABLE_C if kind == 'C' else [(n, n, 1) for n in TABLE_T]
    entries = []
    for i, (n, epc, C) in enumerate(geoms):
        entries.append((n, epc, C, i % 4, (i * 3 + 1) % 4 if i % 3 else 0))
        if i % 4 == 1:
            entries.append((0, 1, 1, 0, 0))
    descs, px, py, data = build_table(r, entries, kind)
    true_max = max(e[0] for e in entries)
    for mode in MODES:
        for qmin, qmax in TABLE_RANGES:
            got = check_table(cabi, oracle, descs, px, py, data, kind, qmin, qmax, mode, true_max, f'{kind} mode {mode} {qmin}..{qmax}')
            if mode in (0, 11) and qmin == -128:
                for d, y in zip(data, single_launches(cabi, px, data, kind, qmin, qmax, mode)):
                    if y is not None:
                        assert_same(got[d[4]:d[4] + d[7]], y, f'{kind} single launch n={d[7]}')
                for max_n in (true_max + 1, 3 * true_max, 1 << 20, 2 ** 31 - 1):
                    again = check_table(cabi, oracle, descs, px, py, data, kind, qmin, qmax, mode, max_n, f'{kind} max_n {max_n}')
                    assert np.array_equal(again.view(np.uint32), got.view(np.uint32))


@pytest.mark.parametrize('kind', ['C', 'T'])
def test_weight_table_limits(cabi, oracle, kind):
    """4096 tensors, one of 2^24 + 5 elements among 4095 tiny ones, are accepted; 4097 are refused before anything is written."""
    r = np.random.RandomState(12)
    entries = []
    for i in range(4096):
        if i == 1234:
            entries.append((2 ** 24 + 5, 1, 3, 1, 3) if kind == 'C' else (2 ** 24 + 5, 2 ** 24 + 5, 1, 1, 3))
        else:
            n = 1 + (i % 13)
            entries.append((n, 1, n, i % 4, (i // 4) % 4) if kind == 'C' else (n, n, 1, i % 4, (i // 4) % 4))
    descs, px, py, data = build_table(r, entries, kind)
    for mode in (0, 11):
        check_table(cabi, oracle, descs, px, py, data, kind, -128, 127, mode, 2 ** 24 + 5, f'{kind} 4096 tensors mode {mode}')
    py.t.copy_(torch.from_numpy(py.init))
    big = torch.cat([descs, descs[:1]])
    fn = cabi.ppq_b200_multi_linear_quant_c if kind == 'C' else cabi.ppq_b200_multi_linear_quant_t
    assert fn(V(big.data_ptr()), 4097, 2 ** 24 + 5, -128, 127, 0, stream()) == 1
    assert fn(V(descs.data_ptr()), 4096, 0, -128, 127, 0, stream()) == 1
    assert fn(V(descs.data_ptr()), 4096, 2 ** 31, -128, 127, 0, stream()) == 1
    torch.cuda.synchronize()
    assert np.array_equal(py.t.cpu().numpy().view(np.uint32), py.init.view(np.uint32)), 'a refused table wrote'


# ---- F: guard bands for the half-input entries -------------------------------------------------------------------------------------
HALF = {F16: (torch.float16, np.float16), BF16: (torch.bfloat16, None)}


def to_half_bits(y32, code):
    t = torch.from_numpy(np.ascontiguousarray(y32)).to(HALF[code][0])
    return t.view(torch.int16).numpy().view(np.uint16)


@pytest.mark.parametrize('code', [F16, BF16])
def test_half_entries_write_only_their_output(cabi, oracle, code):
    """The fp16 / bf16 entries, per tensor and per channel, with heads and tails of n mod 8 in {1, 7} and unaligned bases: the bytes around
    the output stay untouched and the output is the oracle's fp32 result rounded once."""
    r = np.random.RandomState(13 + code)
    tdt = HALF[code][0]
    for n, epc, C, xo, yo in ((8 * 100 + 1, 1, 1, 0, 0), (8 * 100 + 7, 1, 1, 3, 5), (7, 1, 1, 1, 0), (9 * 47 * 3, 9, 47, 0, 0),
                              (516 * 5, 516, 5, 7, 1), (4 * 4 * 7, 4, 4, 2, 6), (1 * 48 * 5, 1, 48, 0, 0)):
        x32 = (r.standard_normal(n) * 4).astype(np.float32)
        xh = torch.from_numpy(x32).to(tdt)
        x32 = xh.float().numpy()
        xk = torch.cat([torch.zeros(xo, dtype=tdt), xh, torch.zeros(8, dtype=tdt)]).cuda()
        xp = xk.data_ptr() + 2 * xo
        s, o = channel_params(r, C)
        s = np.abs(s).clip(1e-3, 1)
        st, ot = torch.from_numpy(s).cuda(), torch.from_numpy(o).cuda()
        per_c = C > 1 or epc > 1
        for op in ('L', 'F', 'Q'):
            g = Guarded(n * (1 if op == 'Q' else 2), yo * (1 if op == 'Q' else 2))
            if op == 'L':
                want = oracle.linear_quant_c(x32.reshape(-1, C, epc), s, o, 1, -128, 127, 11)
                rc = (cabi.ppq_b200_linear_quant_c_dt(xp, code, g.ptr, n, epc, C, st.data_ptr(), ot.data_ptr(), -128, 127, 11, stream()) if per_c
                      else cabi.ppq_b200_linear_quant_t_dt(xp, code, g.ptr, n, st.data_ptr(), ot.data_ptr(), -128, 127, 11, stream()))
            elif op == 'F':
                want = oracle.float_quant_c(x32.reshape(-1, C, epc), s, o, 1, 4, 3, -300.0, 300.0, 1)
                rc = (cabi.ppq_b200_float_quant_c_dt(xp, code, g.ptr, n, epc, C, st.data_ptr(), ot.data_ptr(), 4, 3, -300.0, 300.0, 1, stream()) if per_c
                      else cabi.ppq_b200_float_quant_t_dt(xp, code, g.ptr, n, st.data_ptr(), ot.data_ptr(), 4, 3, -300.0, 300.0, 1, stream()))
            else:
                want = oracle.linear_quant_c(x32.reshape(-1, C, epc), s, o, 1, -128, 127, 4, return_int=True)[1]
                rc = (cabi.ppq_b200_linear_quant_c_toint_dt(xp, code, g.ptr, 8, n, epc, C, st.data_ptr(), ot.data_ptr(), -128, 127, 4, stream()) if per_c
                      else cabi.ppq_b200_linear_quant_t_toint_dt(xp, code, g.ptr, 8, n, st.data_ptr(), ot.data_ptr(), -128, 127, 4, stream()))
            what = f'dtype {code} {op} n={n} epc={epc} C={C} x+{xo} y+{yo}'
            assert rc == 0, what
            if op == 'Q':
                assert_same(g.read(np.uint8, what), (want.astype(np.int64) & 0xFF).astype(np.uint8), what)
            else:
                assert np.array_equal(g.read(np.uint16, what), to_half_bits(want.reshape(-1), code)), what
