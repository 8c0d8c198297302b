"""Sizes past 2^31 elements, on the host: the quantile ranks, the size class of every binding, and the data generator of the GPU cases.

* The ranks of _Quantile_T are `round-half-even((float)n * q)` clipped to [0, n - 1] in 64 bits.  The reference clips with an int, which goes
  negative above 2^31 - 1 elements (DESIGN §2, deviation 12); below, the two forms must agree exactly, and this file shows that they do.
* tests/test_gpu_large_counts.py declares for every launching binding whether it refuses more than 2^31 - 1 elements or takes int64 n; the
  declaration is checked here against the CheckSize calls of the binding sources, so a new binding has to declare its class.
* The GPU cases generate their data on the device from a hash of the element index and regenerate windows of it on the host; the host twin
  must reproduce the torch expression the device runs.
"""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT

CSRC = os.path.join(ROOT, 'ppq_b200', 'csrc')
INT_MAX = 2 ** 31 - 1


def rank_formula(n, frac):
    """round-half-even(float32(n) * float32(frac)), clipped to [0, n - 1] in 64 bits; NaN gives 0."""
    f = np.float32(n) * np.float32(frac)
    if not f > 0:
        return 0
    return min(int(np.rint(f)), n - 1)


def rank_int_clip(n, frac):
    """The reference's form: __float2int_rn (half-even, saturating at the int range, NaN -> 0), then CLIP<int>(pos, 0, (int)(n - 1))."""
    f = np.float32(n) * np.float32(frac)
    pos = 0 if f != f else int(min(max(np.rint(np.float64(f)), -2 ** 31), INT_MAX))
    last = ((n - 1 + 2 ** 31) % 2 ** 32) - 2 ** 31                  # (int)(n - 1)
    return last if pos > last else (0 if pos < 0 else pos)


NS = [1, 2, 2 ** 24 + 1, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 31 + 8, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 100, 3 * 10 ** 9, 2 ** 40]
QS = [0.0, 1e-4, 0.5, 0.999, 0.9999, 1.0, 1.5, -0.5, float('nan')]


@pytest.mark.parametrize('n', NS)
def test_quantile_ranks_follow_the_64_bit_formula(oracle, n):
    for q in QS:
        one_minus = float(np.float32(1) - np.float32(q))
        want = (rank_formula(n, q), rank_formula(n, one_minus))
        assert oracle.quantile_ranks(n, q) == want, (n, q)
        assert all(0 <= r < n for r in want)


def test_quantile_ranks_at_or_below_2_31_are_the_reference_ranks(oracle):
    """Where n - 1 fits an int, the 64-bit clip and the reference's int clip agree, including q outside [0, 1], NaN q and the values of n
    where (float)n rounds (2^24 + 1, 2^31 - 1, odd n above 2^24)."""
    r = np.random.RandomState(12)
    ns = [1, 2, 3, 2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 25 + 5, 10 ** 9 + 7, 2 ** 31 - 65, 2 ** 31 - 1, 2 ** 31]
    ns += [int(v) for v in r.randint(1, 2 ** 31, 200, dtype=np.int64)]
    qs = QS + [2.0, -1e-30, 1e-30, float('inf'), float('-inf'), 0.99999994, 5.96e-8] + [float(v) for v in r.rand(50)]
    for n in ns:
        for q in qs:
            one_minus = float(np.float32(1) - np.float32(q))
            got = oracle.quantile_ranks(n, q)
            assert got == (rank_int_clip(n, q), rank_int_clip(n, one_minus)), (n, q)


def test_quantile_ranks_above_2_31_stay_in_range(oracle):
    """The cases where the int clip breaks: it gives a negative rank for n = 2^31 + 8 and rank 99 for n = 2^32 + 100."""
    assert rank_int_clip(2 ** 31 + 8, 0.9999) == -2147483641 and rank_int_clip(2 ** 32 + 100, 0.9999) == 99
    for n in (2 ** 31 + 8, 2 ** 32 + 100):
        hi, lo = oracle.quantile_ranks(n, 0.9999)
        assert hi == int(np.rint(np.float32(n) * np.float32(0.9999))) and lo == int(np.rint(np.float32(n) * (np.float32(1) - np.float32(0.9999))))
        assert n - 1 - hi < n // 5000 and lo < n // 5000


# ---------------------------------------------------------------------------------------------------------------- size classes
def function_bodies():
    """{function name: body} of the top-level functions of the binding sources."""
    src = ''.join(open(os.path.join(CSRC, f)).read() for f in ('torch_binding.cc', 'torch_binding_more.inc'))
    bodies = {}
    for m in re.finditer(r'^[A-Za-z][\w:<>, ]*?\b(\w+)\(([^;{]*?)\)\s*\{', src, re.M):
        depth, i = 1, m.end()
        while depth:
            depth += {'{': 1, '}': -1}.get(src[i], 0); i += 1
        bodies[m.group(1)] = src[m.end():i]
    return bodies


def refusing_functions(bodies):
    """Functions that call CheckSize, directly or through one of the other functions."""
    refusing = {name for name, body in bodies.items() if re.search(r'\bCheckSize\(', body)}
    changed = True
    while changed:
        changed = False
        for name, body in bodies.items():
            if name not in refusing and any(re.search(rf'\b{f}\(', body) for f in refusing):
                refusing.add(name); changed = True
    return refusing


def test_every_launching_binding_declares_its_size_class():
    from test_cpu_stream_contract import exported_names
    import test_gpu_large_counts as lc
    import test_gpu_stream_contract as sc
    launching = exported_names() - sc.HOST_ONLY
    assert set(lc.SIZE_CLASS) == launching, (f'undeclared: {sorted(launching - set(lc.SIZE_CLASS))}, '
                                            f'not launching bindings: {sorted(set(lc.SIZE_CLASS) - launching)}')
    assert not lc.REFUSES & lc.INT64
    refusing = refusing_functions(function_bodies()) & launching
    assert refusing == lc.REFUSES, (f'refuse without being declared: {sorted(refusing - lc.REFUSES)}, '
                                    f'declared but take int64 n: {sorted(lc.REFUSES - refusing)}')
    import inspect
    called = set(re.findall(r"^\s*'(\w+)': lambda: ext\.(\w+)\(", inspect.getsource(lc.refusal_calls), re.M))
    assert all(key == fn for key, fn in called), 'a refusal case calls another binding than the one it is listed under'
    assert {key for key, _ in called} == lc.REFUSES, 'every refusing binding needs a call in refusal_calls, and only those'


def test_check_size_limit_is_2_31_minus_1():
    src = open(os.path.join(CSRC, 'torch_binding.cc')).read()
    body = function_bodies()['CheckSize']
    assert 'numel() > 0x7fffffffLL' in body and 'too many element' in body, body
    assert 'void CheckSize(' in src


# ---------------------------------------------------------------------------------------------------------------- data generator
@pytest.mark.parametrize('kind', ['f32', 'b16', 'relu', 'near1'])
def test_host_twin_reproduces_the_generator(kind):
    """fill() (the torch expression the device runs, evaluated here on CPU tensors) equals host_values() on windows across the boundaries."""
    import test_gpu_large_counts as lc
    dtype = torch.float32 if kind == 'f32' else torch.bfloat16
    for a in (0, 2 ** 31 - 2000, 2 ** 32 - 777, 2 ** 33 + 12345, 3 * 10 ** 9):
        b = a + 3000
        idx = torch.arange(a, b, dtype=torch.int64)
        dev = lc.values_torch(kind, lc.hash_of(idx)).to(dtype).float().numpy()
        host = lc.host_values(kind, a, b)
        assert np.array_equal(dev.view(np.uint32), host.view(np.uint32)), (kind, a)
        h = lc.hash_of(np.arange(a, b, dtype=np.int64))
        assert h.min() >= 0 and h.max() <= 0xFFFFFFFF
        assert np.array_equal(h, lc.hash_of(idx).numpy())
    if kind == 'near1':
        assert 1.0 not in set(host.tolist()) and np.all(np.abs(host - 1.0) <= 7 * 2 ** -7)


def test_generator_is_spread_and_windows_cover_the_boundaries():
    import test_gpu_large_counts as lc
    h = lc.hash_of(np.arange(2 ** 31 - 2 ** 20, 2 ** 31 + 2 ** 20, dtype=np.int64))
    c = np.bincount(h & 0x1FF, minlength=512)
    assert c.min() > 0.9 * c.mean() and c.max() < 1.1 * c.mean()
    n = 2 ** 32 + 100
    assert lc.boundary_indices(n) == [0, 2 ** 31 - 2, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, n - 1]
    wins = lc.windows(n, 0)
    for i in lc.boundary_indices(n):
        assert any(a <= i < b for a, b in wins), i
    per = 144
    for a, b in lc.windows(2 ** 31 + 144, 1, per):
        assert a % per == 0 and (b % per == 0 or b == 2 ** 31 + 144)
