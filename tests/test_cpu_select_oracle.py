"""The exact oracle of the radix select (Quantile_T, Multi_Quantile_T, Isotone_T), and the host-side mirrors the GPU tests use to prove
which route a call took -- no device needed.

* `oracle.select_t` sorts by the order-preserving 32-bit key of select.cu:72-75 in two semantics: 'device' (one key per bit pattern:
  -NaN < -inf < ... < -0 < +0 < ... < +inf < +NaN, NaNs ordered by payload) and 'reference' (thrust::sort's stable radix sort, where -0 and
  +0 share a key).  Both are checked against numpy's stable argsort of the keys and against np.sort on NaN-free data; they differ only in
  the sign of a selected zero; the reference semantics is pinned by what the reference's own kernels returned (ref_cuda_select.npz).
* `SelectState` mirrors the per-tensor state of select.cu:41-60 and `simulate()` restates the state machine that fills it
  (select_init_kernel, select_pass, select_scan, level_needed); tests/test_gpu_select_paths.py compares the device's state after a call with it.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, cases_of, load_golden

# ---- keys ------------------------------------------------------------------------------------------------------------------------------


def order_keys(x, semantics='device'):
    """select.cu:72-75 as uint32: flip every bit of a negative float, only the sign bit of any other; 'reference' gives -0 the key of +0."""
    b = np.ascontiguousarray(x, dtype=np.float32).reshape(-1).view(np.uint32).copy()
    if semantics == 'reference':
        b[b == 0x80000000] = 0
    return np.where(b >> 31 == 1, ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def torch_order_stats(x, ranks):
    """The elements at `ranks` of the device semantics, from a stable torch.sort of the int64 keys (works on a CUDA tensor of any size:
    the GPU tests use it for large n).  Returns fp32 with the selected elements' exact bits."""
    b = x.reshape(-1).contiguous().view(torch.int32).long() & 0xFFFFFFFF
    keys = torch.where(b >= 0x80000000, b ^ 0xFFFFFFFF, b | 0x80000000)
    order = torch.sort(keys, stable=True)[1]
    r = torch.as_tensor(ranks, dtype=torch.int64, device=x.device)
    return x.reshape(-1)[order[r]]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# ---- the state mirror --------------------------------------------------------------------------------------------------------------
DIGITS, CAP = 2048, 1 << 18                                  # select.cu:36 kDigits, :39 kDefaultCap
SAMPLE_KEYS = 16384                                          # select.cu:121 kSampleKeys
HIST, COMPACT, DONE = 0, 1, 2                                # select.cu:38
MARGIN_INIT, MARGIN_MIN, MARGIN_MAX = 1 << 19, 1 << 12, 1 << 24   # select.cu:62
U32x2, I64x2 = ctypes.c_uint32 * 2, ctypes.c_int64 * 2


class SelectState(ctypes.Structure):
    """select.cu:41-60, field for field."""
    _fields_ = [('hist', (ctypes.c_uint64 * DIGITS) * 2), ('prefix', U32x2), ('mode', U32x2), ('shared', ctypes.c_uint32),
                ('done', ctypes.c_uint32), ('ccount', U32x2), ('cbuf', U32x2), ('clevel', U32x2), ('compacted', U32x2),
                ('kmin', U32x2), ('kmax', U32x2), ('rank', I64x2), ('count', I64x2), ('spec', ctypes.c_uint32),
                ('g', U32x2), ('k', U32x2), ('d', U32x2), ('eqc', U32x2), ('veq', U32x2), ('vkey', U32x2), ('pad2_', ctypes.c_uint32)]


WITNESS = ('prefix', 'mode', 'shared', 'done', 'ccount', 'cbuf', 'clevel', 'compacted', 'rank', 'count', 'spec', 'eqc', 'veq', 'vkey', 'g', 'k', 'd')


def witness_of(raw: bytes):
    """The route fields of one SelectState read back from the device."""
    st = SelectState.from_buffer_copy(raw[:ctypes.sizeof(SelectState)])
    out = {}
    for f in WITNESS:
        v = getattr(st, f)
        out[f] = [int(a) for a in v] if hasattr(v, '__len__') else int(v)
    return out


def shift(level): return (21, 10, 0)[level]            # select.cu:64-66
def dmask(level): return 0x3FF if level == 2 else 0x7FF
def pmask(level): return (0, 0xFFE00000, 0xFFFFFC00)[level]


def sample_thresholds(keys, r0, r1, cap):
    """select_sample_kernel + select_init_kernel (select.cu:124-130, 166-199): the 16384 keys at the sampler's hashed positions, and the
    thresholds {g_hi, g_lo} they give (None where the tail is too heavy for the buffer)."""
    n = keys.size
    stride = n // SAMPLE_KEYS
    i = np.arange(SAMPLE_KEYS, dtype=np.uint64)
    off = ((i * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) % np.uint64(stride)
    s = np.sort(keys[(i * np.uint64(stride) + off).astype(np.int64)])

    def j_of(need):
        return max(12, (3 * need * SAMPLE_KEYS + n - 1) // n)

    def ok(j):
        return j <= SAMPLE_KEYS // 4 and 3 * j * (n // SAMPLE_KEYS) <= 2 * cap
    jh, jl = j_of(n - r0), j_of(r1 + 1)
    return (int(s[SAMPLE_KEYS - jh]) if ok(jh) else None), (int(s[jl - 1]) if ok(jl) else None)


def margin_after(d, app, eq, need, cap, first_call):
    """select_scan<0>'s verdict on one side (select.cu:224-238): (candidates hold the order statistic, new margin)."""
    cnt = app + eq
    if app <= cap and cnt >= need:
        if cnt > 4 * need + 64 and d > MARGIN_MIN: d >>= 1
        return True, d
    if app > cap:
        if d > MARGIN_MIN: d >>= 1
    elif not first_call and d < MARGIN_MAX:
        d <<= 1
    return False, d


def next_guess(key, d, side):
    """select_finish_kernel's guess words for the next call (select.cu:666-671): {threshold, key, margin, 0}."""
    g = (key - d if key > d else 0) if side == 0 else (key + d if key < 0xFFFFFFFF - d else 0xFFFFFFFF)
    return [g, key, d, 0]


def simulate(keys, r0, r1, cap, guess=None):
    """The SelectState one call leaves behind, restated from select.cu for keys `keys` (uint32, device semantics), ranks r0 (upper) and
    r1 (lower), buffer `cap`; `guess` = (g_hi, k_hi, d_hi, g_lo, k_lo, d_lo) when the call speculates on thresholds (a guess buffer or a
    cold sample).  Also returns the selected keys."""
    n = keys.size
    k64 = keys.astype(np.int64)
    st = dict(prefix=[0, 0], mode=[HIST, HIST], shared=1, done=0, ccount=[0, 0], cbuf=[0, 1], clevel=[0, 0], compacted=[0, 0],
              rank=[r0, r1], count=[n, n], spec=0, eqc=[0, 0], veq=[0, 0], vkey=[0, 0], g=[0xFFFFFFFF, 0], k=[0xFFFFFFFF, 0],
              d=[MARGIN_INIT, MARGIN_INIT])
    bufs = [None, None]
    if guess is not None:
        g_hi, k_hi, d_hi, g_lo, k_lo, d_lo = guess
        st.update(spec=1, g=[g_hi, g_lo], k=[k_hi, k_lo], d=[d_hi, d_lo])
        hi, lo = k64[k64 >= g_hi], k64[k64 <= g_lo]
        st['eqc'] = [int((hi == k_hi).sum()), int((lo == k_lo).sum())]
        bufs = [hi[hi != k_hi], lo[lo != k_lo]]
        st['ccount'] = [bufs[0].size, bufs[1].size]
    hist, kmin, kmax = [None, None], [0, 0], [0, 0]
    for L in range(3):
        m, comp = st['mode'], st['compacted']
        need = [L == 0 or m[0] == HIST or (m[0] == COMPACT and not comp[0]),
                L > 0 and not st['shared'] and (m[1] == HIST or (m[1] == COMPACT and not comp[1]))]
        if not any(need):
            break                                                       # no CTA takes a ticket: no scan
        for r in (0, 1):
            if not need[r]: continue
            sel = k64 if L == 0 else k64[(k64 & pmask(L)) == st['prefix'][r]]
            if L == 0 or m[r] == HIST:
                hist[r] = np.bincount((sel >> shift(L)) & dmask(L), minlength=DIGITS)
                if sel.size: kmin[r], kmax[r] = int(sel.min()), int(sel.max())
                else: kmin[r], kmax[r] = 0xFFFFFFFF, 0
            else:
                bufs[r] = sel
                st['ccount'][r] += sel.size
        # select_scan<L>
        if L == 0 and st['spec']:
            for r in (0, 1):
                app, eq = st['ccount'][r], st['eqc'][r]
                nd = n - st['rank'][0] if r == 0 else st['rank'][1] + 1
                first = st['g'][0] == 0xFFFFFFFF if r == 0 else st['g'][1] == 0
                ok, st['d'][r] = margin_after(st['d'][r], app, eq, nd, cap, first)
                if ok:
                    st['mode'][r], st['compacted'][r], st['clevel'][r], st['prefix'][r], st['cbuf'][r] = COMPACT, 1, 0, 0, r
                    st['rank'][r] = app + eq - nd if r == 0 else st['rank'][1]
                    st['veq'][r], st['vkey'][r] = eq, st['k'][r]
                else:
                    st['ccount'][r] = 0
                    bufs[r] = None
        shared_in = st['shared']
        for r in (0, 1):
            src = 0 if (r == 1 and shared_in) else r
            if st['mode'][r] == DONE: continue
            if st['mode'][r] == COMPACT:
                st['compacted'][r] = 1
                continue
            if L > 0 and kmin[src] == kmax[src]:
                st['prefix'][r], st['mode'][r] = kmin[src], DONE
                continue
            h = hist[src]
            cum = np.cumsum(h)
            dg = int(np.searchsorted(cum, st['rank'][r], side='right'))
            before = int(cum[dg] - h[dg])
            st['prefix'][r] |= dg << shift(L)
            st['rank'][r] -= before
            st['count'][r] = int(h[dg])
            if L == 2: st['mode'][r] = DONE
            elif h[dg] <= cap: st['mode'][r], st['clevel'][r] = COMPACT, L + 1
        m, comp = st['mode'], st['compacted']
        same = st['prefix'][0] == st['prefix'][1] and m[0] == m[1] and m[0] != DONE and not comp[0] and not comp[1]
        st['shared'] = int(same)
        if m[0] == COMPACT and not comp[0]: st['cbuf'][0] = 0
        if m[1] == COMPACT and not comp[1]: st['cbuf'][1] = 0 if same else 1
        st['done'] = 0
    # select_finish_kernel: the selected key of each rank
    sel = []
    for r in (0, 1):
        if st['mode'][r] != COMPACT:
            sel.append(st['prefix'][r])
            continue
        b = st['cbuf'][r]
        cand = np.concatenate([bufs[b], np.full(st['veq'][r], st['vkey'][r], np.int64)])
        sel.append(int(np.sort(cand)[st['rank'][r]]))
    return st, sel


def route_of(st, r):
    """A short name of the route rank r took, for messages and the coverage table."""
    if st['spec'] and st['mode'][r] == COMPACT and st['clevel'][r] == 0:
        return 'speculated'
    if st['mode'][r] == COMPACT:
        return f'compact@{st["clevel"][r]}' + ('-shared' if r == 1 and st['cbuf'][1] == 0 else '')
    return 'histogram'


# ---- the oracle ------------------------------------------------------------------------------------------------------------------------
NAN_BITS = (0x7FC00000, 0x7F800001, 0x7FFFFFFF, 0xFFC00000, 0xFF800001, 0xFFFFFFFF)


def adversarial(r):
    """Inputs a value sort gets wrong: NaNs of both signs and several payloads, +-inf, runs of +-0, subnormals, repeats."""
    specials = np.concatenate([np.asarray(NAN_BITS, np.uint32).view(np.float32),
                               np.float32([np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 3.4e38, -3.4e38, 1.0, 1.0])])
    out = []
    for n in (1, 2, 3, 5, 17, 64, 333):
        for _ in range(4):
            x = r.standard_normal(n).astype(np.float32)
            m = r.rand(n) < 0.6
            x[m] = r.choice(specials, int(m.sum()))
            out.append(x)
    return out


@pytest.mark.parametrize('semantics', ['device', 'reference'])
def test_select_matches_stable_argsort_of_the_keys(oracle, semantics):
    r = np.random.RandomState(7)
    inputs = adversarial(r) + [r.standard_normal(n).astype(np.float32) for n in (1, 4, 1000)]
    for x in inputs:
        want = x[np.argsort(order_keys(x, semantics), kind='stable')]
        got = oracle.select_t(x, np.arange(x.size), semantics)
        assert np.array_equal(bits(got), bits(want)), (semantics, x)
        # shuffled, repeated ranks
        ranks = r.randint(x.size, size=7)
        assert np.array_equal(bits(oracle.select_t(x, ranks, semantics)), bits(want[ranks]))


def test_select_matches_value_sort_without_nans(oracle):
    r = np.random.RandomState(8)
    for x in adversarial(r):
        x = x[~np.isnan(x)]
        if x.size == 0: continue
        for sem in ('device', 'reference'):
            got = oracle.select_t(x, np.arange(x.size), sem)
            assert np.array_equal(got, np.sort(x)), sem                 # as values: -0 == +0


def test_the_two_semantics_differ_only_in_the_sign_of_a_zero(oracle):
    r = np.random.RandomState(9)
    differ = 0
    for x in adversarial(r) + [np.float32([0.0, -0.0, -0.0, 0.0, -0.0]), np.float32([-0.0, 0.0])]:
        d, f = oracle.select_t(x, np.arange(x.size), 'device'), oracle.select_t(x, np.arange(x.size), 'reference')
        same = bits(d) == bits(f)
        assert ((d == 0) & (f == 0) | same).all()
        differ += int((~same).sum())
        # device: every -0 before every +0;  reference: the zeros in input order
        z = x[(x == 0)]
        zd = d[d == 0]
        assert np.array_equal(bits(zd), np.sort(bits(z))[::-1]), x       # 0x80000000 (-0) first
        assert np.array_equal(bits(f[f == 0]), bits(z))
    assert differ > 0


def test_quantile_ranks_follow_the_fp32_products(oracle):
    for n, q in [(10, 0.25), (4, 0.375), (4, 0.125), (8, 0.0625), (2, 0.75), (2, 0.25), ((1 << 24) + 1, 0.5), ((1 << 24) + 3, 0.9999),
                 (1000, 1e-7), (1000, 1 - 2 ** -24), (1, 0.5), (7, 0.0), (7, 1.0), (401408, 0.9999)]:
        fa = np.float32(n) * np.float32(q); fb = np.float32(n) * (np.float32(1) - np.float32(q))
        want = tuple(int(min(max(np.rint(v), 0), n - 1)) for v in (fa, fb))      # np.rint: half-even, as __float2int_rn
        assert oracle.quantile_ranks(n, q) == want, (n, q)
    assert oracle.quantile_ranks(4, 0.375) == (2, 2)                    # 1.5 and 2.5 both round to 2
    assert oracle.quantile_ranks((1 << 24) + 1, 0.5)[0] == 1 << 23      # (float)(2^24 + 1) == 2^24


def test_quantile_and_isotone_read_the_selected_ranks(oracle):
    r = np.random.RandomState(10)
    for x in adversarial(r):
        for sem in ('device', 'reference'):
            for q in (0.0, 0.3, 0.5, 0.9999, 1.0):
                assert np.array_equal(bits(oracle.quantile_t(x, q, sem)), bits(oracle.select_t(x, oracle.quantile_ranks(x.size, q), sem)))
            iso = oracle.isotone_t(x, sem)
            want = [x[0]] * 4 if x.size == 1 else oracle.select_t(x, [x.size - 1, x.size - 2, 0, 1], sem)
            assert np.array_equal(bits(iso), bits(want)), (sem, x)
    assert np.array_equal(bits(oracle.isotone_t(np.float32([-0.0]))), bits(np.float32([-0.0] * 4)))


def test_torch_sort_of_the_keys_equals_the_oracle(oracle):
    """The formulation the GPU tests use for large n (a stable torch.sort of int64 keys) selects what the C oracle selects."""
    r = np.random.RandomState(11)
    for x in adversarial(r):
        ranks = np.arange(x.size)
        got = torch_order_stats(torch.from_numpy(x), ranks).numpy()
        assert np.array_equal(bits(got), bits(oracle.select_t(x, ranks, 'device')))


def test_simulated_selection_equals_the_oracle(oracle):
    """The state-machine restatement ends on the oracle's keys, on every route it models (small cap to force them all)."""
    r = np.random.RandomState(12)
    for x in adversarial(r) + [np.maximum(r.standard_normal(5000).astype(np.float32), 0), np.float32(r.randint(-3, 3, 3000))]:
        keys = order_keys(x)
        for q in (0.0, 0.5, 0.9, 1.0):
            r0, r1 = oracle.quantile_ranks(x.size, q)
            for cap in (1, 16, 1 << 18):
                _, sel = simulate(keys, r0, r1, cap)
                assert sel == [int(k) for k in order_keys(oracle.select_t(x, [r0, r1]))], (x.size, q, cap)
            srt = np.sort(keys.astype(np.int64))
            for g_off in (0, 3, 40):                                  # hand-written thresholds around the selected keys
                g_hi, g_lo = int(srt[max(r0 - g_off, 0)]), int(srt[min(r1 + g_off, x.size - 1)])
                _, sel = simulate(keys, r0, r1, 64, (g_hi, g_hi, 1 << 12, g_lo, g_lo, 1 << 12))
                assert sel == [int(k) for k in order_keys(oracle.select_t(x, [r0, r1]))], (x.size, q, g_off)


def test_margin_update_restatement():
    need = 100
    assert margin_after(1 << 19, 99, 0, need, 1000, False) == (False, 1 << 20)          # one short: widen
    assert margin_after(1 << 19, 60, 40, need, 1000, False) == (True, 1 << 19)          # exactly need, copies count
    assert margin_after(1 << 19, 4 * need + 64, 0, need, 1000, False) == (True, 1 << 19)
    assert margin_after(1 << 19, 4 * need + 65, 0, need, 1000, False) == (True, 1 << 18)   # far more than needed: tighten
    assert margin_after(1 << 12, 4 * need + 65, 0, need, 1000, False) == (True, 1 << 12)   # not below 2^12
    assert margin_after(1 << 19, 1001, 0, need, 1000, False) == (False, 1 << 18)        # overflow: halve
    assert margin_after(1 << 24, 5, 0, need, 1000, False) == (False, 1 << 24)           # not above 2^24
    assert margin_after(1 << 19, 5, 0, need, 1000, True) == (False, 1 << 19)            # first call: no verdict


# ---- C ABI sizes (host functions: no device needed) ---------------------------------------------------------------------------------
def test_state_mirror_matches_the_workspace_sizes():
    lib = ctypes.CDLL(os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so'))
    lib.ppq_b200_quantile_workspace_bytes.restype = ctypes.c_int64
    lib.ppq_b200_multi_quantile_workspace_bytes.restype = ctypes.c_int64
    lib.ppq_b200_multi_quantile_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int64]
    assert ctypes.sizeof(SelectState) == lib.ppq_b200_quantile_workspace_bytes() - (2 * CAP + SAMPLE_KEYS) * 4
    for cap in (1, 64, 1 << 16):
        assert ctypes.sizeof(SelectState) == lib.ppq_b200_multi_quantile_workspace_bytes(1, cap) - 2 * cap * 4
        assert lib.ppq_b200_multi_quantile_workspace_bytes(3, cap) == 3 * (ctypes.sizeof(SelectState) + 2 * cap * 4)


# ---- the reference's own kernels -----------------------------------------------------------------------------------------------------
def _maker():
    spec = importlib.util.spec_from_file_location('make_ref_select', os.path.join(GOLDEN, 'make_ref_select.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_reference_semantics_pinned_by_the_reference_kernels(oracle):
    """ref_cuda_select.npz holds what the reference's Quantile_T / Isotone_T (thrust::sort) returned on the H100.  The oracle's reference
    semantics must reproduce every bit, zero signs and NaN payloads included; the device semantics must agree except in zero signs."""
    mk = _maker()
    rec = cases_of(load_golden('ref_cuda_select.npz'))
    small = mk.cases()
    assert [c['name'] for c in rec['small']] == [name for name, _, _ in small]
    zero_sign_differs = 0
    for c, (name, x, qs) in zip(rec['small'], small):
        assert np.array_equal(np.uint32(c['x']), bits(x)), name
        for q, want in zip(qs, c['quantile']):
            assert list(bits(oracle.quantile_t(x, q, 'reference'))) == want, (name, q)
            dev, w = oracle.quantile_t(x, q, 'device'), np.uint32(want)
            differs = bits(dev) != w
            assert (~differs | ((dev == 0) & (w.view(np.float32) == 0))).all(), (name, q)
            zero_sign_differs += int(differs.sum())
        assert list(bits(oracle.isotone_t(x, 'reference'))) == c['isotone'], name
    assert zero_sign_differs > 0                                        # the fixture does tell the two semantics apart
    for c in rec['large']:                                              # one sort per input: all ranks in one call
        x, n = mk.big(c['n'], c['seed']), c['n']
        ranks = [r for q in c['q'] for r in oracle.quantile_ranks(n, q)] + [n - 1, n - 2, 0, 1]
        got = [int(v) for v in bits(oracle.select_t(x, ranks, 'reference'))]
        assert got == [v for pair in c['quantile'] for v in pair] + c['isotone'], n
