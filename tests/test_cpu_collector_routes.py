"""The collector launch routes, restated on the host: which kernel, grid, block and dynamic shared memory each entry of
ppq_b200/csrc/collectors.cu launches for a size, a bin count, a dtype, a base alignment and a `histogram` variant.

tests/test_gpu_collector_routes.py runs every case of ROUTE_CASES on the device, checks with the profiler that the kernel, grid, block and
shared memory it names are the ones that ran, and compares the result with the oracle.  The tests here need no GPU: they check that the
case table reaches every (entry x route x dtype) cell and sits on both sides of each threshold, and that the grid formulas of the mirror
agree with the C++ ones.  For that they cut the grid arithmetic out of collectors.cu and common.cuh, compile it with g++ behind a stub
sm_count(), and compare both on a sweep of sizes; a change of a formula in the kernels' source fails here until the mirror follows it.
"""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT

H100_SMS = 132
CSRC = os.path.join(ROOT, 'ppq_b200', 'csrc')
F32, F16, BF16 = 0, 1, 2
ELEM_BYTES = {F32: 4, F16: 2, BF16: 2}
K_THREADS, K_HIST_THREADS, K_MAX_SMEM_BINS, K_ROW_CHUNK = 256, 1024, 12287, 4096


# ---- the dispatch, restated ---------------------------------------------------------------------------------------------------
def grid_for(work, threads, per_thread, ctas_per_sm, sms=H100_SMS):
    """common.cuh:201-208."""
    per_cta = threads * per_thread
    return max(1, min((work + per_cta - 1) // per_cta, sms * ctas_per_sm))


def hist_grid(n, bins, sms=H100_SMS):
    """collectors.cu:585-592: each CTA should own max(16 bins, 65536) elements; at most one CTA per SM."""
    per_cta = max(bins * 16, 65536)
    return max(1, min((n + per_cta - 1) // per_cta, sms))


def _kernel(name, *args):
    return (name, tuple(str(a) for a in args))


def hist_route(n, bins, variant, dtype=F32, sms=H100_SMS, binop='SymBin'):
    """launch_hist (collectors.cu:595-617) for fp32, launch_hist_half (:621-630) for fp16 / bf16.
    Returns (route, kernel, grid, block, dynamic shared memory bytes)."""
    T = {F32: 'float', F16: '__half', BF16: '__nv_bfloat16'}[dtype]
    if dtype != F32:                                                   # one layout; the variant is not read
        if bins > K_MAX_SMEM_BINS:
            return 'global', _kernel('histogram_kernel', 3, binop, 4, 256, 1, T), grid_for(n, K_THREADS, 16, 8, sms), K_THREADS, 0
        g = hist_grid(n, bins, sms)
        return 'default', _kernel('histogram_kernel', 0, binop, 2, 1024, 2, T), min(g * 2, sms * 2), K_HIST_THREADS, (bins + 1) * 4
    var = 3 if bins > K_MAX_SMEM_BINS else variant                     # :597
    grid = grid_for(n, K_THREADS, 16, 8, sms) if var == 3 else hist_grid(n, bins, sms)
    smem = 0 if var == 3 else (bins + 1) * 4
    hk = lambda *a: _kernel('histogram_kernel', *a)                   # noqa: E731
    if var == 1:
        return 'v1', hk(1, binop, 4, 1024, 1, T), grid, K_HIST_THREADS, smem
    if var == 2:
        return 'v2', hk(2, binop, 4, 1024, 1, T), grid, K_HIST_THREADS, smem
    if var == 3:
        return 'global', hk(3, binop, 4, 256, 1, T), grid, K_THREADS, smem
    if var == 4:
        return 'v4', hk(0, binop, 8, 256, 1, T), min(grid * 8, sms * 8), K_THREADS, smem
    if var == 5:
        return 'v5', hk(0, binop, 4, 1024, 1, T), grid, K_HIST_THREADS, smem
    if var == 6:
        return 'v6', hk(0, binop, 4, 1024, 2, T), min(grid * 2, sms * 2), K_HIST_THREADS, smem
    if var == 7:
        if grid >= 2:
            return 'cluster2', _kernel('histogram_cluster_kernel', binop, 2), grid & ~1, K_HIST_THREADS, smem
        return 'v7_single', hk(0, binop, 4, 1024, 1, T), grid, K_HIST_THREADS, smem
    if var == 8:
        if grid >= 4:
            return 'cluster4', _kernel('histogram_cluster_kernel', binop, 4), grid & ~3, K_HIST_THREADS, smem
        return 'v8_single', hk(0, binop, 4, 1024, 1, T), grid, K_HIST_THREADS, smem
    return 'default', hk(0, binop, 2, 1024, 2, T), min(grid * 2, sms * 2), K_HIST_THREADS, smem


def dscale_route(n, bins, dtype, sms=H100_SMS):
    """ppq_b200_histogram_t_dscale_dt, collectors.cu:724-739."""
    T = {F32: 'float', F16: '__half', BF16: '__nv_bfloat16'}[dtype]
    if bins > K_MAX_SMEM_BINS:
        return 'global', _kernel('histogram_dscale_kernel', 3, 256, 1, T), grid_for(n, K_THREADS, 16, 8, sms), K_THREADS, 0
    return 'smem', _kernel('histogram_dscale_kernel', 0, 1024, 2, T), min(hist_grid(n, bins, sms) * 2, sms * 2), K_HIST_THREADS, (bins + 1) * 4


def histogram_c_plan(n, epc, bins, sms=H100_SMS):
    """ppq_b200_histogram_c, collectors.cu:746-758: (chunk, chunks per row, items, grid); None where the entry refuses the bin count.
    One CTA per (row, chunk) item, grid-strided over the items: 'loop' when a CTA zeroes and flushes its bins more than once."""
    if bins > K_MAX_SMEM_BINS:
        return None
    rows = n // epc
    chunk = max(bins * 8, 32768)
    chunks = (epc + chunk - 1) // chunk
    items = rows * chunks
    grid = min(items, sms * 8)
    return dict(chunk=chunk, chunks=chunks, items=items, grid=grid, route='loop' if items > grid else 'once')


def histogram_c_launch(n, epc, bins, sms=H100_SMS):
    p = histogram_c_plan(n, epc, bins, sms)
    return p['route'], _kernel('histogram_c_kernel', 0), p['grid'], K_THREADS, (bins + 1) * 4


def head_elems(byte_off):
    """half.cuh:90-92: half elements before the first 16-byte boundary of a base `byte_off` bytes past one."""
    return ((16 - (byte_off & 15)) & 15) >> 1


def minmax_t_launch(n, dtype, off, sms=H100_SMS):
    """ppq_b200_minmax_t_dt, collectors.cu:669-677, and the path stream_elements (:74-124) takes inside.  `off` is in elements past a
    16-byte-aligned base.  fp32: 'vec' (float4 loop + <= 3 tail elements) or 'scalar'; halves: 'head_only' when the <= 7 elements before
    the first 16-byte boundary are the whole tensor, else 'body' (head, whole 8-element vectors, <= 7 tail elements)."""
    eb = ELEM_BYTES[dtype]
    T = {F32: 'float', F16: '__half', BF16: '__nv_bfloat16'}[dtype]
    per = 16 // eb
    grid = grid_for((n + per - 1) // per, K_THREADS, 4 * 4, 8, sms)
    if dtype == F32:
        route = 'vec' if (off * 4) % 16 == 0 else 'scalar'
    else:
        route = 'head_only' if n <= head_elems(off * 2) else 'body'
    return route, _kernel('minmax_t_kernel', T), grid, K_THREADS, 0


def half_split(n, off):
    """(head, whole vectors, tail) of a half tensor at element offset `off` (stream_elements, collectors.cu:102-103)."""
    head = min(n, head_elems(off * 2))
    nv = (n - head) >> 3
    return head, nv, n - head - 8 * nv


def minmax_c_plan(n, epc, sms=H100_SMS):
    """ppq_b200_minmax_c_dt, collectors.cu:683-697: one warp per (row, kRowChunk-element chunk) item, 8 warps per CTA, at most
    8 CTAs per SM; 'loop' when a warp takes more than one item."""
    rows = n // epc
    chunks = (epc + K_ROW_CHUNK - 1) // K_ROW_CHUNK
    items = rows * chunks
    grid = min((items + 7) // 8, sms * 8)
    return dict(chunks=chunks, items=items, grid=grid, warps=grid * 8, route='loop' if items > grid * 8 else 'once')


def minmax_c_launch(n, epc, dtype, sms=H100_SMS):
    T = {F32: 'float', F16: '__half', BF16: '__nv_bfloat16'}[dtype]
    p = minmax_c_plan(n, epc, sms)
    return p['route'], _kernel('minmax_c_kernel', T), p['grid'], K_THREADS, 0


def multi_stream_grid(count, max_n, resident, sms=H100_SMS):
    """launch_multi_stream, collectors.cu:650-652 (`resident` = the occupancy query, clamped to 1..2)."""
    return max(1, min((count * max_n + 65535) // 65536, sms * resident))


# ---- the case table -------------------------------------------------------------------------------------------------------------
SMALL_N = list(range(1, 10)) + [31, 32, 33, 4095, 4096, 4097]
# hist_grid's per-CTA share +- 1 (4096 bins: 65536; 12287 bins: 196592), and the saturation of the grid at the SM count
SHARE_N = [65535, 65536, 65537, 2 * 65536 + 1, 3 * 65536 + 1, 196591, 196592, 196593]
SAT_N = [(H100_SMS - 1) * 65536 + 1, H100_SMS * 65536, H100_SMS * 65536 + 1]
SCALE_EDGES = ('zero', 'inf', 'nan', '1e-40', '2^-60', 'below 2^-60', '2^60', 'above 2^60')
NEG_SCALES = ('negative', '-0')
HIST_BINS = (1, 2, 3, 50, 2047, 2048, 4096, 12287)
BIG_BINS = (12288, 16384, 20000)


def scale_value(name, base):
    return np.float32({'ordinary': base, 'zero': 0.0, 'inf': np.inf, 'nan': np.nan, '1e-40': 1e-40, '2^-60': 2.0 ** -60,
                       'below 2^-60': np.nextafter(np.float32(2.0 ** -60), np.float32(0)), '2^60': 2.0 ** 60,
                       'above 2^60': np.nextafter(np.float32(2.0 ** 60), np.float32(np.inf)), 'negative': -base, '-0': -0.0}[name])


def _hist_t_cases():
    out = []
    for v in range(9):
        sizes = SMALL_N[::3] + [4095, 4097] if v not in (0, 7, 8) else SMALL_N
        for i, n in enumerate(sizes):
            out.append(dict(n=n, bins=(50, 2048, 4096, 3)[i % 4], variant=v, off=i % 4))
        for i, n in enumerate(SHARE_N[:3] + [2 * 65536 + 1, 3 * 65536 + 1, 4 * 65536 + 1, 5 * 65536 + 1]):
            out.append(dict(n=n, bins=4096, variant=v, off=(i + 1) % 4))
        for i, n in enumerate(SHARE_N[5:]):                            # 12287 bins: a share of 196592 elements
            out.append(dict(n=n, bins=12287, variant=v, off=i))
    for n in SAT_N:
        out.append(dict(n=n, bins=4096, variant=0, off=0))
        out.append(dict(n=n, bins=4096, variant=8, off=0))
    for b in HIST_BINS + BIG_BINS:
        out.append(dict(n=70001, bins=b, variant=0, off=b % 4))
    for b in BIG_BINS:
        for v in (0, 5, 7):
            out.append(dict(n=4097, bins=b, variant=v, off=1))
    res = []
    for c in out:
        route, k, g, blk, sm = hist_route(c['n'], c['bins'], c['variant'])
        res.append(dict(c, entry='hist_t', dtype=F32, route=route))
    return res


def _hist_asym_cases():
    res = []
    for v in range(9):
        for i, n in enumerate([1, 5, 33, 4097, 65537, 5 * 65536 + 1]):
            res.append(dict(n=n, bins=(2048, 50, 4096)[i % 3], variant=v, off=i % 4))
    for dt in (F16, BF16):
        for i, n in enumerate([1, 7, 8, 9, 31, 33, 4097, 65537, 196593]):
            res.append(dict(n=n, bins=(2048, 4096, 50)[i % 3], variant=0, off=i % 8, dtype=dt))
        res.append(dict(n=4099, bins=16384, variant=0, off=3, dtype=dt))
    res.append(dict(n=4099, bins=20000, variant=0, off=2))
    for c in res:
        c.setdefault('dtype', F32)
        c['entry'] = 'hist_asym'
        c['route'] = hist_route(c['n'], c['bins'], c['variant'], c['dtype'], binop='AsymBin')[0]
    return res


def _dscale_cases():
    res = []
    for dt in (F32, F16, BF16):
        for i, n in enumerate([1, 3, 9, 33, 4097, 65537, 196593]):
            res.append(dict(n=n, bins=(4096, 2048, 12287)[i % 3], off=i % (4 if dt == F32 else 8), dtype=dt))
        for b in BIG_BINS:
            res.append(dict(n=20011, bins=b, off=1, dtype=dt))
    for c in res:
        c['entry'], c['variant'] = 'hist_dscale', 0
        c['route'] = dscale_route(c['n'], c['bins'], c['dtype'])[0]
    return res


# Histogram_C: (shape, axis, bins).  chunk = max(8 bins, 32768): epc at chunk +- 1 and 2 chunk + 1 for three chunks -- the floor 32768
# (256 and 4096 bins), 40000 (5000 bins) and 98296 (12287 bins) --, axis first / middle / last, C = 1, odd epc (rows start misaligned),
# and [4, 1100, 3, 3] on axis 1: 4400 items > 132 x 8 CTAs.
HIST_C_GEOMS = [([3, 32767], 0, 256), ([3, 32768], 0, 256), ([2, 32769], 0, 256), ([2, 65537], 0, 256), ([1, 32769], 0, 256),
                ([2, 3, 32767], 1, 4096), ([2, 32768], 0, 4096), ([2, 32769], 0, 4096), ([1, 65537], 0, 4096),
                ([5, 7, 9], 2, 50), ([4, 1100, 3, 3], 1, 256), ([3, 5, 9], 0, 2048), ([16, 3, 3, 3], 0, 1), ([6, 2, 5], 1, 3),
                ([9, 1], 0, 12287), ([2, 7, 3], 2, 2), ([1, 131073], 0, 4096), ([1200, 3], 0, 50),
                ([2, 39999], 0, 5000), ([2, 40000], 0, 5000), ([2, 3, 40001], 1, 5000), ([1, 80001], 0, 5000),
                ([2, 98295], 0, 12287), ([2, 98296], 0, 12287), ([2, 98297], 0, 12287), ([1, 196593], 0, 12287)]


def channel_geometry(shape, axis):
    epc = int(np.prod(shape[axis + 1:])) if axis + 1 < len(shape) else 1
    return epc, shape[axis]


def _hist_c_cases():
    res = []
    for shape, axis, bins in HIST_C_GEOMS:
        n = int(np.prod(shape))
        epc, C = channel_geometry(shape, axis)
        res.append(dict(entry='hist_c', dtype=F32, shape=shape, axis=axis, bins=bins, n=n, epc=epc, C=C, variant=0, off=0,
                        route=histogram_c_plan(n, epc, bins)['route']))
    return res


def _minmax_t_cases():
    res = []
    for dt in (F32, F16, BF16):
        maxoff = 4 if dt == F32 else 8
        for i, n in enumerate(SMALL_N + [65537, 1 << 20]):
            for off in ((i % maxoff, (i + 1) % maxoff) if n > 9 else (i % maxoff,)):
                res.append(dict(entry='minmax_t', dtype=dt, n=n, off=off, variant=0))
        for off in range(maxoff):
            res.append(dict(entry='minmax_t', dtype=dt, n=8 * 37 + off, off=off, variant=0))
    for c in res:
        c['route'] = minmax_t_launch(c['n'], c['dtype'], c['off'])[0]
    return res


# MinMax_C: (shape, axis).  epc at kRowChunk - 1, kRowChunk, + 1 and 2 kRowChunk + 1; [16, 1024, 1, 1] on axis 1 puts 16384 items on
# 8448 warps; odd epc; C = 1.
MINMAX_C_GEOMS = [([3, 4095], 0), ([3, 4096], 0), ([3, 4097], 0), ([2, 8193], 0), ([16, 1024, 1, 1], 1), ([5, 7, 9], 2), ([4, 3, 33], 1),
                  ([1, 12289], 0), ([20000, 1], 0), ([9, 1, 5], 1), ([2, 6, 700], 1), ([3, 40000], 1)]


def _minmax_c_cases():
    res = []
    for dt in (F32, F16, BF16):
        for i, (shape, axis) in enumerate(MINMAX_C_GEOMS):
            n = int(np.prod(shape))
            epc, C = channel_geometry(shape, axis)
            res.append(dict(entry='minmax_c', dtype=dt, shape=shape, axis=axis, n=n, epc=epc, C=C, variant=0,
                            off=i % (4 if dt == F32 else 8), route=minmax_c_plan(n, epc)['route']))
    return res


def _multi_cases():
    return [dict(entry='multi_hist', dtype=dt, bins=b, variant=0, route='table') for dt in (F32, F16, BF16) for b in (2048, 4096)]


ROUTE_CASES = (_hist_t_cases() + _hist_asym_cases() + _dscale_cases() + _hist_c_cases() + _minmax_t_cases() + _minmax_c_cases()
               + _multi_cases())


def case_id(c):
    geo = f'{c["shape"]}a{c["axis"]}' if 'shape' in c else f'n{c.get("n", "")}'
    return f'{c["entry"]}-{c["route"]}-d{c["dtype"]}-{geo}-b{c.get("bins", 0)}-v{c["variant"]}-o{c.get("off", 0)}'


HIST_T_ROUTES = ('default', 'v1', 'v2', 'global', 'v4', 'v5', 'v6', 'cluster2', 'cluster4', 'v7_single', 'v8_single')
WANT_CELLS = ({('hist_t', r, F32) for r in HIST_T_ROUTES} | {('hist_asym', r, F32) for r in HIST_T_ROUTES}
              | {('hist_asym', r, d) for r in ('default', 'global') for d in (F16, BF16)}
              | {('hist_dscale', r, d) for r in ('smem', 'global') for d in (F32, F16, BF16)}
              | {('hist_c', r, F32) for r in ('once', 'loop')}
              | {('minmax_t', r, F32) for r in ('vec', 'scalar')} | {('minmax_t', r, d) for r in ('head_only', 'body') for d in (F16, BF16)}
              | {('minmax_c', r, d) for r in ('once', 'loop') for d in (F32, F16, BF16)}
              | {('multi_hist', 'table', d) for d in (F32, F16, BF16)})


# ---- tests ----------------------------------------------------------------------------------------------------------------------
def test_case_table_covers_every_entry_route_and_dtype_cell():
    have = {(c['entry'], c['route'], c['dtype']) for c in ROUTE_CASES}
    assert WANT_CELLS - have == set(), sorted(WANT_CELLS - have)
    assert have - WANT_CELLS == set(), sorted(have - WANT_CELLS)


def test_case_table_sits_on_both_sides_of_each_threshold():
    ht = [c for c in ROUTE_CASES if c['entry'] == 'hist_t']
    ns = {c['n'] for c in ht}
    assert set(SMALL_N) <= ns and {65535, 65536, 65537} <= ns and set(SAT_N) <= ns
    assert {196591, 196592, 196593} <= {c['n'] for c in ht if c['bins'] == 12287}
    # the grid reaches the SM count at (sms - 1) x 65536 + 1 elements and stays there one share later, where the quotient is sms + 1
    assert hist_grid(SAT_N[0] - 1, 4096) == H100_SMS - 1
    assert [hist_grid(n, 4096) for n in SAT_N] == [H100_SMS] * 3 and -(-SAT_N[2] // 65536) == H100_SMS + 1
    assert hist_grid(65536, 4096) == 1 and hist_grid(65537, 4096) == 2 and hist_grid(196592, 12287) == 1 and hist_grid(196593, 12287) == 2
    # the cluster variants fall back to one-CTA kernels under 2 / 4 CTAs, and round 5 CTAs down to one cluster of 4
    assert hist_route(3 * 65536 + 1, 4096, 8)[0] == 'cluster4' and hist_route(3 * 65536 + 1, 4096, 8)[2] == 4
    assert hist_route(5 * 65536 + 1, 4096, 8)[2] == 4 and hist_route(3 * 65536, 4096, 8)[0] == 'v8_single'
    assert hist_route(65536, 4096, 7)[0] == 'v7_single' and hist_route(65537, 4096, 7)[0] == 'cluster2'
    assert {c['bins'] for c in ht} >= set(HIST_BINS) | set(BIG_BINS)
    assert all(c['route'] == 'global' for c in ht if c['bins'] > K_MAX_SMEM_BINS)
    assert {c['off'] for c in ROUTE_CASES if c['dtype'] == F32 and 'off' in c and c['entry'] != 'hist_c'} == {0, 1, 2, 3}
    assert {c['off'] for c in ROUTE_CASES if c['dtype'] != F32 and 'off' in c} == set(range(8))
    # Histogram_C: epc at chunk - 1, chunk, chunk + 1 and 2 chunk + 1 for three distinct chunk sizes; more items than CTAs; refusal
    # above 12287
    hc = [c for c in ROUTE_CASES if c['entry'] == 'hist_c']
    assert sorted(histogram_c_plan(1, 1, b)['chunk'] for b in (256, 5000, 12287)) == [32768, 40000, 98296]
    for bins in (256, 5000, 12287):
        ch = histogram_c_plan(1, 1, bins)['chunk']
        assert {ch - 1, ch, ch + 1, 2 * ch + 1} <= {c['epc'] for c in hc if c['bins'] == bins}, bins
    assert histogram_c_plan(4 * 1100 * 9, 9, 256)['items'] == 4400 > H100_SMS * 8
    assert {c['axis'] for c in hc if c['axis'] == len(c['shape']) - 1} and {c['axis'] for c in hc if 0 < c['axis'] < len(c['shape']) - 1}
    assert any(c['C'] == 1 for c in hc) and any(c['epc'] % 2 for c in hc)
    assert histogram_c_plan(10, 1, 12288) is None
    # MinMax_C: epc at kRowChunk - 1, kRowChunk, + 1, 2 kRowChunk + 1; more items than resident warps
    mc = [c for c in ROUTE_CASES if c['entry'] == 'minmax_c']
    assert {4095, 4096, 4097, 8193} <= {c['epc'] for c in mc}
    assert minmax_c_plan(16 * 1024, 1)['items'] == 16384 > H100_SMS * 8 * 8
    # half min/max: every head and tail length 0..7 occurs
    hm = [c for c in ROUTE_CASES if c['entry'] == 'minmax_t' and c['dtype'] == F16]
    assert {half_split(c['n'], c['off'])[0] for c in hm} == set(range(8))
    assert {half_split(c['n'], c['off'])[2] for c in hm} == set(range(8))


def test_scale_edges_straddle_the_exact_division_range():
    """ExactDiv (common.cuh:102-109) takes the fast reciprocal for 2^-60 <= |s| <= 2^60 only; the edge scales sit on both sides."""
    lo, hi = np.float32(8.6736174e-19), np.float32(1.1529215e18)
    assert lo == np.float32(2.0 ** -60) and hi == np.float32(2.0 ** 60)
    ok = lambda s: bool(lo <= abs(s) <= hi)                            # noqa: E731
    v = {k: scale_value(k, 0.0371) for k in SCALE_EDGES}
    assert ok(v['2^-60']) and not ok(v['below 2^-60']) and ok(v['2^60']) and not ok(v['above 2^60'])
    assert not any(ok(v[k]) for k in ('zero', 'inf', 'nan', '1e-40'))


# ---- the grid formulas of the C++ source, compiled and compared -------------------------------------------------------------------
def _cut(pattern, text, what):
    m = re.search(pattern, text, re.S)
    assert m, f'{what}: not found in the source; the mirror in this file needs to follow the change'
    return m.group(0) if m.lastindex is None else m.group(1)


def _harness_source():
    common = open(os.path.join(CSRC, 'common.cuh')).read()
    coll = open(os.path.join(CSRC, 'collectors.cu')).read()
    src = ['#include <cstdint>', '#include <cstdio>', '#include <algorithm>', 'using std::min; using std::max;',
           'static int g_sms = 132; inline int sm_count() { return g_sms; }', 'enum { cudaErrorInvalidValue = 1 };']
    for k in ('kThreads', 'kUnroll', 'kRowChunk', 'kHistThreads', 'kMaxSmemBins'):
        src.append(_cut(rf'constexpr int {k} = \d+;', coll, k))
    src.append(_cut(r'inline int grid_for\(.*?\n}\n', common, 'grid_for'))
    src.append(_cut(r'static inline int hist_grid\(.*?\n}\n', coll, 'hist_grid'))
    launch = _cut(r'static int launch_hist\(.*?\n}\n', coll, 'launch_hist')
    # the launch shape of every case of the variant switch; a cluster case has its one-CTA fallback on the next line
    body, lines = [], launch.splitlines()
    for i, line in enumerate(lines):
        m = re.match(r'\s*(case (\d)|default):.*?<<<([^,]+),\s*([^,]+),', line)
        if not m:
            continue
        cond = re.search(r'if \((grid >= \d)\)', line)
        test = f'var == {m.group(2)}' if m.group(2) else 'true'
        if cond:
            fb = re.search(r'<<<([^,]+),\s*([^,]+),', lines[i + 1])
            body.append(f'  if ({test}) {{ if ({cond.group(1)}) {{ g = {m.group(3)}; b = {m.group(4)}; }} else {{ g = {fb.group(1)}; '
                        f'b = {fb.group(2)}; }} return; }}')
        else:
            body.append(f'  if ({test}) {{ g = {m.group(3)}; b = {m.group(4)}; return; }}')
    assert len(body) == 9, body                                        # cases 1-8 and default
    src.append('void hist_launch(int64_t n, int64_t bins, int var, int &base, int &g, int &b) {\n  ' +
               _cut(r'if \(bins > kMaxSmemBins\) var = 3;', launch, 'bin override') + '\n  ' +
               _cut(r'const int grid = var == 3 \?[^;]*;', launch, 'grid') + '\n  base = grid;\n' + '\n'.join(body) + '\n}')
    dsc = _cut(r'int ppq_b200_histogram_t_dscale_dt\(.*?\n}\n', coll, 'dscale')
    src.append('int dscale_grid(int64_t n, int64_t bins) {\n  if (bins > kMaxSmemBins) return ' +
               _cut(r'<<<(grid_for\([^>]*?\)), kThreads', dsc, 'dscale global grid') + ';\n  ' +
               _cut(r'const int grid = hist_grid[^;]*;', dsc, 'dscale grid') + '\n  return grid;\n}')
    hc = _cut(r'int ppq_b200_histogram_c\(.*?\n}\n', coll, 'histogram_c')
    src.append('void hc_plan(int64_t n, int64_t epc, int64_t bins, int64_t *o) {\n' +
               _cut(r'(const int64_t rows = n / epc;.*?)histogram_c_kernel', hc, 'histogram_c plan') +
               '\n  o[0] = chunk; o[1] = chunks; o[2] = items; o[3] = grid;\n}')
    mc = _cut(r'int ppq_b200_minmax_c_dt\(.*?\n}\n', coll, 'minmax_c')
    src.append('int mc_plan(int64_t n, int64_t epc, int64_t *o) {\n' +
               _cut(r'(const int64_t rows = n / epc;.*?)return with_elem_type', mc, 'minmax_c plan') +
               '\n  o[0] = chunks; o[1] = items; o[2] = grid; return 0;\n}')
    mt = _cut(r'int ppq_b200_minmax_t_dt\(.*?\n}\n', coll, 'minmax_t')
    src.append('template <int S> int mt_grid(int64_t n) { struct T { char b[S]; };\n  ' +
               _cut(r'const int grid = grid_for\(\(n \+ 16 / sizeof\(T\)[^;]*;', mt, 'minmax_t grid') + '\n  return grid;\n}')
    ms = _cut(r'static int launch_multi_stream\(.*?\n}\n', coll, 'launch_multi_stream')
    src.append('int64_t ms_grid(int count, int64_t max_n, int resident) {\n' +
               _cut(r'(int64_t g = \(\(int64_t\)count \* max_n.*?if \(g < 1\) g = 1;)', ms, 'multi grid') + '\n  return g;\n}')
    src.append(r'''
int main() {
  int sms; long long n, bins, epc, count, max_n; int var, resident;
  char kind;
  while (scanf(" %c %d", &kind, &sms) == 2) {
    g_sms = sms;
    if (kind == 'h') { scanf("%lld %lld %d", &n, &bins, &var); int base, g, b; hist_launch(n, bins, var, base, g, b);
                       printf("%d %d %d\n", base, g, b); }
    else if (kind == 'd') { scanf("%lld %lld", &n, &bins); printf("%d\n", dscale_grid(n, bins)); }
    else if (kind == 'c') { scanf("%lld %lld %lld", &n, &epc, &bins); int64_t o[4]; hc_plan(n, epc, bins, o);
                            printf("%lld %lld %lld %lld\n", (long long)o[0], (long long)o[1], (long long)o[2], (long long)o[3]); }
    else if (kind == 'm') { scanf("%lld %lld", &n, &epc); int64_t o[3]; mc_plan(n, epc, o);
                            printf("%lld %lld %lld\n", (long long)o[0], (long long)o[1], (long long)o[2]); }
    else if (kind == 't') { scanf("%lld", &n); printf("%d %d\n", mt_grid<4>(n), mt_grid<2>(n)); }
    else if (kind == 's') { scanf("%lld %lld %d", &count, &max_n, &resident); printf("%lld\n", (long long)ms_grid((int)count, max_n, resident)); }
  }
  return 0;
}''')
    return '\n'.join(src)


@pytest.fixture(scope='module')
def cxx_twin(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('collector_twin'))
    src, exe = os.path.join(d, 'twin.cc'), os.path.join(d, 'twin')
    with open(src, 'w') as f:
        f.write(_harness_source())
    r = subprocess.run(['g++', '-std=c++17', '-O1', src, '-o', exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]

    def run(lines):
        p = subprocess.run([exe], input='\n'.join(lines) + '\n', capture_output=True, text=True, check=True)
        return [list(map(int, ln.split())) for ln in p.stdout.splitlines()]
    return run


SWEEP_N = sorted(set(SMALL_N + SHARE_N + SAT_N + [1 << 20, 1 << 24, 10 ** 9, 3 * 10 ** 9] + [k * 65536 + d for k in (1, 2, 3, 4, 5, 131, 132, 133, 263, 264)
                                                                                         for d in (-1, 0, 1)]))
SWEEP_SMS = (132, 114, 1, 7)


def test_hist_grids_agree_with_the_source(cxx_twin):
    q, want = [], []
    for sms in SWEEP_SMS:
        for n in SWEEP_N:
            for bins in (1, 50, 2048, 4096, 4097, 12287, 12288, 20000):
                for var in range(10):
                    q.append(f'h {sms} {n} {bins} {var}')
                    r = hist_route(n, bins, var, F32, sms)
                    base = grid_for(n, K_THREADS, 16, 8, sms) if (bins > K_MAX_SMEM_BINS or var == 3) else hist_grid(n, bins, sms)
                    want.append((base, r, bins > K_MAX_SMEM_BINS))
    got = cxx_twin(q)
    assert len(got) == len(q)
    for qq, g, (base, r, big) in zip(q, got, want):
        assert g == [base, r[2], r[3]], (qq, g, r)


def test_other_grids_agree_with_the_source(cxx_twin):
    q, want = [], []
    for sms in SWEEP_SMS:
        for n in SWEEP_N:
            for bins in (1, 50, 4096, 12287, 12288, 20000):
                q.append(f'd {sms} {n} {bins}')
                want.append([dscale_route(n, bins, F32, sms)[2]])
            q.append(f't {sms} {n}')
            want.append([minmax_t_launch(n, F32, 0, sms)[2], minmax_t_launch(n, F16, 0, sms)[2]])
            for epc in sorted({1, 3, 4095, 4096, 4097, 8193, 32767, 32768, 32769, 65537, n}):
                if n % epc or epc > n:
                    continue
                for bins in (1, 256, 4096, 12287):
                    p = histogram_c_plan(n, epc, bins, sms)
                    q.append(f'c {sms} {n} {epc} {bins}')
                    want.append([p['chunk'], p['chunks'], p['items'], p['grid']])
                p = minmax_c_plan(n, epc, sms)
                q.append(f'm {sms} {n} {epc}')
                want.append([p['chunks'], p['items'], p['grid']])
        for count in (1, 3, 106, 4096):
            for max_n in (1, 4097, 65536, 65537, 1 << 24):
                for resident in (1, 2):
                    q.append(f's {sms} {count} {max_n} {resident}')
                    want.append([multi_stream_grid(count, max_n, resident, sms)])
    got = cxx_twin(q)
    assert len(got) == len(q)
    for qq, g, w in zip(q, got, want):
        assert g == w, (qq, g, w)
