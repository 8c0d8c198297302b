"""Every route of the radix select (select.cu), each case built for one route and proved to have taken it.

A call's SelectState (the caller's workspace) records the route each rank took: mode, the level compaction started at (clevel), the keys
compacted (ccount), the bucket population (count), speculation (spec, eqc, veq), shared buffers, the pass tickets (done).  Every case
compares the whole state with `simulate()` (tests/test_cpu_select_oracle.py, a restatement of select.cu's state machine) and asserts the
route it was built for; the result bits must equal the device-semantics oracle, and value plus NaN bits the reference semantics.

    route (rank r)                                         cases
    compact@1: top-digit bucket of exactly cap keys        test_cap_boundary[cap]
    histogram -> compact@2: cap + 1 keys                    test_cap_boundary[cap+1]
    histogram to level 2 (pass 2)                          test_pass_two_histogram
    one value resolved at level 1 (+0 / -0 buckets)        test_one_value_buckets[zeros]
    one value resolved at level 2 (clipped maxima)         test_one_value_buckets[clipped]
    both ranks in one compacted buffer (shared)            test_shared_bucket
    shared histogram, then compact / histogram split       test_ranks_diverge_at_level_one
    ranks at bucket edges, digits 0 and 2047 (NaNs)        test_bucket_edges_and_nan_ends
    q in {0, 1, 1e-7, 1 - 2^-24}, n q = k + 0.5            test_extreme_and_tied_q
    finish: 8192 k +- 1, 32768 +- 1 candidates             test_finish_populations
    pass-0 x pass-1 variants, +- bit 64, n <= 2^23 + 5     test_select_variants
    cold sample on n >= 2^23                               test_cold_sample_thresholds
    speculation verdicts at need - 1 / need / need + 1,
      cap / cap + 1 stored, veq copies, margin updates     test_speculation_single, test_speculation_table
    table: spans, misaligned bases, ticket-only CTAs,
      tiny cap, scrambled slots, out_stride 3, n = 0       test_table_spans_and_tickets, test_table_ticket_only_small_tensors,
                                                           test_table_count_limit, test_table_empty_entry
    Isotone_T (two calls of the select, n = 1 path)        test_isotone
    bf16 / fp16 inputs                                     test_half_inputs

Mutants each of these must kill (each built and run once): quantile_rank rounding half-up (test_extreme_and_tied_q), order_key merging
-0 into +0 (test_one_value_buckets[zeros]), the compact test `s_cnt < cap` (test_cap_boundary[cap], through the state only), the
speculation verdict `cnt >= need - 1` (test_speculation_single), the finish dropping the veq copies (test_speculation_single,
test_speculation_table), the finish loading one register group too few (test_finish_populations), and a sub-vector overlap taking no
ticket (test_table_ticket_only_small_tensors, whose tensors are at most cap / 2 so that the broken state machine cannot overrun a buffer).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_cpu_select_oracle import (CAP, COMPACT, DONE, MARGIN_MIN, WITNESS, SelectState, bits, next_guess, order_keys,
                                    route_of, sample_thresholds, simulate, torch_order_stats, witness_of)

pytestmark = pytest.mark.gpu

F32, F16, BF16 = 0, 1, 2
V, I, L, Fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
SENT = np.float32(-7.5)
INIT_GUESS = [0xFFFFFFFF, 0xFFFFFFFF, 1 << 19, 0, 0, 0, 1 << 19, 0]           # ppq_b200_quantile_guess_init (select.cu:750)
SAMPLE_MIN = 1 << 23                                                            # select.cu:122


@pytest.fixture(scope='module')
def cabi():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    lib = ctypes.CDLL(os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so'))
    sig = {'ppq_b200_quantile_t_dt': [V, I, L, Fl, V, V, V, V],
           'ppq_b200_isotone_t': [V, L, V, V, V],
           'ppq_b200_multi_quantile_t': [V, I, L, Fl, V, L, V, L, V, V],
           'ppq_b200_set_variant': [ctypes.c_char_p, I]}
    for name, args in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, ctypes.c_int
    lib.ppq_b200_quantile_workspace_bytes.restype = L
    lib.ppq_b200_multi_quantile_workspace_bytes.restype = L
    lib.ppq_b200_multi_quantile_workspace_bytes.argtypes = [I, L]
    return lib


def stream():
    return V(torch.cuda.current_stream().cuda_stream)


SMALL = 1 << 20                                                                 # up to here the C oracle sorts on the host


def expected(x, ranks, semantics='device'):
    xf = x.float().reshape(-1)
    if semantics == 'device' and xf.numel() > SMALL:
        return torch_order_stats(xf, ranks).cpu().numpy()
    import oracle
    return oracle.select_t(xf.cpu().numpy(), ranks, semantics)


def check_values(got, x, ranks, what):
    """Bits against the device semantics; value and NaN bits against the reference's (they differ in zero signs only)."""
    want = expected(x, ranks)
    assert np.array_equal(bits(got), bits(want)), f'{what}: {got} vs {want} ({bits(got)} vs {bits(want)})'
    if x.numel() <= SMALL:
        ref = expected(x, ranks, 'reference')
        nan = np.isnan(ref)
        assert np.array_equal(got[~nan], ref[~nan]) and np.array_equal(bits(got)[nan], bits(ref)[nan]), f'{what}: {got} vs reference {ref}'


def check_state(got, want, what):
    bad = {f: (got[f], want[f]) for f in WITNESS if got[f] != want[f]}
    assert not bad, f'{what}: state differs from the restated route: {bad}'


def single(cabi, x, q, guess=None, dtype=F32):
    """One ppq_b200_quantile_t_dt call; out is carved from a sentinel buffer.  Returns (out2, state, guess words after)."""
    ws = torch.empty(cabi.ppq_b200_quantile_workspace_bytes(), dtype=torch.uint8, device='cuda')
    buf = torch.full((4,), float(SENT), device='cuda')
    g = None if guess is None else torch.tensor(np.asarray(guess, np.uint32).view(np.int32), device='cuda')
    rc = cabi.ppq_b200_quantile_t_dt(V(x.data_ptr()), dtype, x.numel(), float(np.float32(q)), V(buf.data_ptr() + 4), V(ws.data_ptr()),
                                     None if g is None else V(g.data_ptr()), stream())
    torch.cuda.synchronize()
    assert rc == 0, rc
    b = buf.cpu().numpy()
    assert b[0] == SENT and b[3] == SENT, 'a store outside out2'
    st = witness_of(ws[:ctypes.sizeof(SelectState)].cpu().numpy().tobytes())
    return b[1:3].copy(), st, (None if g is None else [int(v) for v in g.cpu().numpy().view(np.uint32)])


def spec_words_for(keys, r0, r1, guess, sampled):
    """The thresholds the init kernel starts from (select.cu:183-199)."""
    if guess is None and not sampled:
        return None
    w = INIT_GUESS if guess is None else guess
    g_hi, k_hi, d_hi, g_lo, k_lo, d_lo = w[0], w[1], w[2], w[4], w[5], w[6]
    if sampled and g_hi == 0xFFFFFFFF and g_lo == 0:
        s_hi, s_lo = sample_thresholds(keys, r0, r1, CAP)
        if s_hi is not None: g_hi = k_hi = s_hi
        if s_lo is not None: g_lo = k_lo = s_lo
    return g_hi, k_hi, d_hi, g_lo, k_lo, d_lo


def run_case(cabi, x, q, what, guess=None, dtype=F32, variant=0, memo=None):
    """Single-tensor call checked against the oracle and the restated state; returns (state, selected keys, guess after).
    `memo` (a dict) keeps the expectations of an input across calls that must agree (the variants)."""
    import oracle
    n = x.numel()
    r0, r1 = oracle.quantile_ranks(n, q)
    tag = (x.data_ptr(), n, float(q), bool(variant & 64), None if guess is None else tuple(guess))
    if memo is None or tag not in memo:
        keys = order_keys(x.float().reshape(-1).cpu().numpy())
        # the host samples (select.cu:697-701) when either tail is light enough for the buffer
        sampled = n >= SAMPLE_MIN and not (variant & 64) and any(v is not None for v in sample_thresholds(keys, r0, r1, CAP))
        want_st, sel = simulate(keys, r0, r1, CAP, spec_words_for(keys, r0, r1, guess, sampled))
        if memo is not None: memo[tag] = want_st, sel, expected(x, [r0, r1])
    want_st, sel = memo[tag][:2] if memo is not None else (want_st, sel)
    got, st, g_after = single(cabi, x, q, guess, dtype)
    if memo is not None:
        assert np.array_equal(bits(got), bits(memo[tag][2])), f'{what}: {got} vs {memo[tag][2]}'
    else:
        check_values(got, x, [r0, r1], what)
    assert [int(k) for k in order_keys(got)] == sel, what
    check_state(st, want_st, what)
    if guess is not None:
        assert g_after == next_guess(sel[0], want_st['d'][0], 0) + next_guess(sel[1], want_st['d'][1], 1), (what, g_after)
    return st, sel, g_after


def q_for_rank(n, rank):
    """A q with clip(rn(n q)) == rank (fp32 arithmetic)."""
    import oracle
    q = np.float32(rank / n)
    for _ in range(64):
        r = oracle.quantile_ranks(n, float(q))[0]
        if r == rank: return float(q)
        q = np.nextafter(q, np.float32(2 if r < rank else -1))
    raise AssertionError((n, rank))


def f32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def spread(lo, count):
    """`count` distinct floats from `lo` upwards, 8 ulps apart (2^18 of them fill [1.0, 1.25), one top digit)."""
    return (np.float32(lo).view(np.uint32) + np.arange(count, dtype=np.uint32) * 8).view(np.float32)


# ---------------------------------------------------------------------------------------------------------------- single tensor
@pytest.mark.parametrize('extra', [0, 1], ids=['cap', 'cap+1'])
def test_cap_boundary(cabi, extra):
    """The top-digit buckets of both ranks, [1, 1.25) and (-1.25, -1], hold exactly cap keys (compacted after pass 0) or cap + 1
    (histogrammed in pass 1, whose level-1 bucket then compacts at clevel 2)."""
    r = np.random.RandomState(1)
    m = CAP + extra
    a = spread(1.0, CAP)
    if extra: a = np.append(a, np.float32(1.2))
    b = -a
    f = 1000
    x = np.concatenate([r.uniform(-8, -2, f), b, r.uniform(-0.5, 0.5, f), a, r.uniform(2, 8, f)]).astype(np.float32)
    x = x[r.permutation(x.size)]
    n = x.size
    q = q_for_rank(n, f + m + f + m // 2)
    st, _, _ = run_case(cabi, f32(x), q, f'cap boundary +{extra}')
    assert st['mode'] == [COMPACT, COMPACT] and st['clevel'] == [2 - (not extra)] * 2, st
    if not extra: assert st['count'] == [CAP, CAP] and st['ccount'] == [CAP, CAP]


def test_pass_two_histogram(cabi):
    """A level-1 bucket of > cap keys with several distinct values: histogrammed on all three levels."""
    r = np.random.RandomState(2)
    close = (np.float32(1.0).view(np.uint32) + r.randint(0, 1024, CAP + 5000).astype(np.uint32)).view(np.float32)
    x = np.concatenate([close, -close, r.standard_normal(3000).astype(np.float32) * 10])
    x = x[r.permutation(x.size)]
    st, _, _ = run_case(cabi, f32(x), 0.75, 'pass 2')
    assert st['mode'] == [DONE, DONE] and st['compacted'] == [0, 0] and all(c < CAP for c in st['count'])


@pytest.mark.parametrize('kind', ['zeros', 'clipped'])
def test_one_value_buckets(cabi, kind):
    """zeros: > cap post-ReLU +0 (top digit 1024) and > cap negated-ReLU -0 (top digit 1023), one rank in each, resolved from
    kmin == kmax in pass 1.  clipped: > cap copies of a clipped maximum share their top digit with other values, so the level-1 bucket
    is the one value, resolved in pass 2."""
    r = np.random.RandomState(3)
    if kind == 'zeros':
        x = np.concatenate([np.zeros(CAP + 7, np.float32), np.full(CAP + 9, -0.0, np.float32), r.standard_normal(5000).astype(np.float32)])
        n = x.size
        x = x[r.permutation(n)]
        q = 0.75                                                         # upper rank among the +0, lower among the -0
    else:
        x = np.concatenate([np.full(CAP + 11, 6.0, np.float32), r.uniform(6.5, 7.0, 3000).astype(np.float32),
                            -np.full(CAP + 11, 6.0, np.float32), -r.uniform(6.5, 7.0, 3000).astype(np.float32),
                            r.standard_normal(2000).astype(np.float32)])
        x = x[r.permutation(x.size)]
        q = 0.8
    st, sel, _ = run_case(cabi, f32(x), q, f'one value {kind}')
    assert st['mode'] == [DONE, DONE] and st['compacted'] == [0, 0]
    if kind == 'zeros':
        assert sel == [0x80000000, 0x7FFFFFFF]                           # +0 and -0: the device keeps the signs apart
        assert st['count'] == [CAP + 7, CAP + 9]                         # the top-digit populations: resolved before any level-1 pick
    else:
        assert all(c > CAP for c in st['count'])                         # the level-1 bucket population, > cap


def test_shared_bucket(cabi):
    """Both ranks in one bucket of <= cap keys: one compaction into buffer 0, read by both."""
    x = f32(np.random.RandomState(4).standard_normal(100003))
    st, _, _ = run_case(cabi, x, 0.5, 'shared')
    assert st['cbuf'] == [0, 0] and st['ccount'][1] == 0 and st['mode'] == [COMPACT, COMPACT]


def test_ranks_diverge_at_level_one(cabi):
    """q = 0.5 + 1/n: both ranks share the top-digit histogram, then split at level 1 -- rank 1 into a > cap level-1 bucket
    (histogram, pass 2), rank 0 into a small one (compacted at clevel 2)."""
    r = np.random.RandomState(5)
    n = 1 << 20
    a1 = (np.float32(1.0).view(np.uint32) + r.randint(0, 1024, CAP + 100).astype(np.uint32)).view(np.float32)
    a2 = spread(np.float32(1.0 + 2.0 ** -12), 1000)
    below, above = n // 2 - a1.size, n // 2 - a2.size
    x = np.concatenate([r.uniform(-8, -2, below), a1, a2, r.uniform(2, 8, above)]).astype(np.float32)
    x = x[r.permutation(n)]
    st, _, _ = run_case(cabi, f32(x), 0.5 + 1.0 / n, 'diverge')
    assert st['mode'] == [COMPACT, DONE] and st['clevel'][0] == 2 and st['compacted'] == [1, 0] and st['cbuf'] == [0, 1]


def test_bucket_edges_and_nan_ends(cabi):
    """Ranks on the first and last key of a bucket, and at digits 0 and 2047: -NaN 0xFFFFFFFF (key 0) and +NaN 0x7FFFFFFF (key ~0) among
    other NaN payloads."""
    r = np.random.RandomState(6)
    x = r.standard_normal(50000).astype(np.float32)
    nans = np.uint32([0xFFFFFFFF, 0xFFC00000, 0xFF800001, 0x7FFFFFFF, 0x7FC00000, 0x7F800001]).view(np.float32)
    x[r.randint(x.size, size=nans.size)] = nans
    n = x.size
    keys = np.sort(order_keys(x).astype(np.int64))
    top = keys >> 21
    edges = [0, 1, 2, n - 3, n - 2, n - 1]
    for dg in np.unique(top)[3:-3:7]:
        idx = np.flatnonzero(top == dg)
        edges += [int(idx[0]), int(idx[-1])]
    for rank in edges:
        run_case(cabi, f32(x), q_for_rank(n, rank), f'edge rank {rank}')
    for q in (0.0, 1.0):
        _, sel, _ = run_case(cabi, f32(x), q, f'q={q}')
        assert sorted(sel) == [0, 0xFFFFFFFF]


def test_extreme_and_tied_q(cabi):
    r = np.random.RandomState(7)
    for n in (1, 2, 3, 5, 1000, 4096, 4097, 123457):
        x = r.standard_normal(n).astype(np.float32)
        x[:: 3] = -0.0
        x[1:: 7] = 0.0
        for q in (0.0, 1.0, 1e-7, 1 - 2.0 ** -24, 0.5, 0.9999):
            run_case(cabi, f32(x), q, f'n={n} q={q}')
        if n % 2 == 0:
            for k in (1, n // 2 - 1):                                # n q = k + 0.5 exactly: half-even
                q = (k + 0.5) / n
                assert np.float32(n) * np.float32(q) == k + 0.5
                run_case(cabi, f32(x), q, f'n={n} tie {k}')
    for n in ((1 << 24) + 1, (1 << 24) + 3):                          # (float)n rounds
        x = np.maximum(r.standard_normal(n).astype(np.float32), 0)
        run_case(cabi, f32(x), 0.5, f'n={n}')


@pytest.mark.parametrize('m', [8191, 8192, 8193, 16383, 16385, 24575, 24577, 32767, 32768, 32769, 40961])
def test_finish_populations(cabi, m):
    """The finish holds 4 groups of 8 x 1024 candidates in registers and streams the rest (select.cu:611-654): a compacted bucket of
    exactly m keys, the rank on its first, middle and last key."""
    r = np.random.RandomState(m)
    f = 700
    x = np.concatenate([r.uniform(-8, -2, f), spread(1.0, m), r.uniform(2, 8, f)]).astype(np.float32)
    x = x[r.permutation(x.size)]
    for rank in (f, f + m // 2, f + m - 1):
        st, _, _ = run_case(cabi, f32(x), q_for_rank(x.size, rank), f'finish m={m} rank={rank}')
        assert st['mode'][0] == COMPACT and st['ccount'][0] == m and st['clevel'][0] == 1


@pytest.fixture
def variant(cabi):
    yield lambda v: cabi.ppq_b200_set_variant(b'select', v)
    cabi.ppq_b200_set_variant(b'select', 0)


def test_select_variants(cabi, variant):
    """Every pass-0 x pass-1 variant of the single-tensor select, with and without bit 64 (no cold sample), on n <= 4096, 4097, 8192
    and 2^23 + 5: the same route and the same bits."""
    r = np.random.RandomState(8)
    inputs = []
    for n in (1000, 4096, 4097, 8192):
        x = r.standard_normal(n).astype(np.float32)
        x[::5] = 0.0
        inputs.append((f32(x), (0.9999, 0.5)))
    big = np.maximum(r.standard_normal((1 << 23) + 5).astype(np.float32), 0)
    inputs.append((f32(big), (0.9999,)))
    memo = {}
    for x, qs in inputs:
        for v0 in range(5):
            for v1 in range(5):
                for b64 in (0, 64):
                    v = v0 | (v1 << 3) | b64
                    assert variant(v) == 0
                    for q in qs:
                        run_case(cabi, x, q, f'variant {v} n={x.numel()} q={q}', variant=v, memo=memo)


def test_cold_sample_thresholds(cabi):
    """n >= 2^23 without a guess buffer: thresholds from the 16384 sampled keys (restated in sample_thresholds); the state shows the
    speculation and its verdict."""
    r = np.random.RandomState(9)
    n = (1 << 23) + 4099
    base = r.standard_normal(n).astype(np.float32)
    for tag, x in (('randn', base), ('relu', np.maximum(base, 0)), ('clipped', np.clip(base, -1.5, 1.5))):
        for q in (0.9999, 0.999):
            st, _, _ = run_case(cabi, f32(x), q, f'cold {tag} q={q}')
            assert st['spec'] == 1


# ---------------------------------------------------------------------------------------------------------------- speculation
def spec_input(r, n):
    x = np.unique(r.standard_normal(n).astype(np.float32))               # distinct values: candidate counts are exact
    return x[r.permutation(x.size)]


def test_speculation_single(cabi):
    """Hand-written guess words put select_scan<0>'s verdict exactly on its boundaries: candidates need - 1 / need / need + 1, stored
    candidates cap / cap + 1, copies of the threshold key (veq), and a first call; the words after each call follow the margin rules."""
    r = np.random.RandomState(10)
    x = spec_input(r, 300000)
    n = x.size
    import oracle
    q = 0.999
    r0, r1 = oracle.quantile_ranks(n, q)
    srt = np.sort(order_keys(x).astype(np.int64))
    need_hi, need_lo = n - r0, r1 + 1
    absent_hi, absent_lo = 0, 0xFFFFFFFF                                 # keys no element has (-NaN 0xFFFFFFFF, +NaN 0x7FFFFFFF)
    d = 1 << 16
    for dc in (-1, 0, 1):
        words = [int(srt[n - (need_hi + dc)]), absent_hi, d, 0, int(srt[need_lo + dc - 1]), absent_lo, d, 0]
        st, _, _ = run_case(cabi, f32(x), q, f'spec candidates need{dc:+d}', guess=words)
        assert st['spec'] == 1
        assert [m == COMPACT and c == 0 for m, c in zip(st['mode'], st['clevel'])] == [dc >= 0] * 2, st
        assert st['d'] == ([d, d] if dc >= 0 else [2 * d, 2 * d])
    # far more candidates than needed: tighten, not below 2^12
    for dd in (d, MARGIN_MIN):
        words = [int(srt[n - 4 * need_hi - 65]), absent_hi, dd, 0, int(srt[4 * need_lo + 64]), absent_lo, dd, 0]
        st, _, _ = run_case(cabi, f32(x), q, f'spec tighten {dd}', guess=words)
        assert st['d'] == [max(dd // 2, MARGIN_MIN)] * 2
    # stored candidates cap / cap + 1 (single tensor: cap = 2^18)
    y = spec_input(r, 3 * CAP)
    ny = y.size
    r0, r1 = oracle.quantile_ranks(ny, q)
    sy = np.sort(order_keys(y).astype(np.int64))
    for extra in (0, 1):
        words = [int(sy[ny - CAP - extra]), absent_hi, d, 0, int(sy[CAP + extra - 1]), absent_lo, d, 0]
        st, _, _ = run_case(cabi, f32(y), q, f'spec stored cap+{extra}', guess=words)
        assert [route_of(st, k) == 'speculated' for k in (0, 1)] == [not extra] * 2, st   # a full buffer speculates, cap + 1 does not
        assert st['d'] == [d // 2, d // 2]                              # tightened (cap >> need) or halved (overflow)
    # first call (the init words): no verdict on the margin
    st, _, g = run_case(cabi, f32(x), q, 'spec first call', guess=INIT_GUESS)
    assert st['d'] == [1 << 19, 1 << 19]
    # and the call after it uses the words it left behind
    run_case(cabi, f32(x), q, 'spec second call', guess=g)
    # the threshold key repeated: copies are counted (veq), not stored
    z = np.clip(r.standard_normal(200000).astype(np.float32), -1.5, 1.5)
    k15, km15 = int(order_keys(np.float32([1.5]))[0]), int(order_keys(np.float32([-1.5]))[0])
    st, _, _ = run_case(cabi, f32(z), 0.9999, 'spec veq', guess=[k15, k15, d, 0, km15, km15, d, 0])
    assert st['ccount'] == [0, 0] and min(st['veq']) > 1000 and st['mode'] == [COMPACT, COMPACT]


def table(cabi, xs, slots, q, cap, guess=None, out_stride=3, max_n=None, count_rows=None):
    """One ppq_b200_multi_quantile_t call over the tensors `xs` (None = an n = 0 entry); out carved from a sentinel buffer."""
    count = len(xs)
    descs = torch.tensor([[0 if x is None else x.data_ptr(), 0 if x is None else x.numel(), s] for x, s in zip(xs, slots)],
                         dtype=torch.int64, device='cuda')
    ws = torch.empty(cabi.ppq_b200_multi_quantile_workspace_bytes(count, cap), dtype=torch.uint8, device='cuda')
    rows = count_rows or (max(slots) + 1)
    out = torch.full((rows * out_stride + 8,), float(SENT), device='cuda')
    g = None if guess is None else torch.tensor(np.asarray(guess, np.uint32).reshape(-1).view(np.int32), device='cuda')
    mn = max_n or max(1, max(0 if x is None else x.numel() for x in xs))
    rc = cabi.ppq_b200_multi_quantile_t(V(descs.data_ptr()), count, mn, float(np.float32(q)), V(out.data_ptr() + 16), out_stride,
                                        V(ws.data_ptr()), cap, None if g is None else V(g.data_ptr()), stream())
    torch.cuda.synchronize()
    if rc: return rc, None, None, None
    o = out.cpu().numpy()
    assert (o[:4] == SENT).all() and (o[4 + rows * out_stride:] == SENT).all(), 'a store outside the output rows'
    body = o[4:4 + rows * out_stride].reshape(rows, out_stride)
    if out_stride > 2: assert (body[:, 2:] == SENT).all(), 'a store between slots'
    raw = ws.cpu().numpy().tobytes()
    sz = ctypes.sizeof(SelectState)
    states = [witness_of(raw[i * sz:(i + 1) * sz]) for i in range(count)]
    return 0, body[:, :2].copy(), states, (None if g is None else g.cpu().numpy().view(np.uint32).reshape(-1, 8))


def check_table(xs, slots, q, cap, body, states, guess=None):
    import oracle
    for i, (x, s) in enumerate(zip(xs, slots)):
        if x is None: continue
        keys = order_keys(x.cpu().numpy())
        r0, r1 = oracle.quantile_ranks(x.numel(), q)
        words = None
        if guess is not None:
            w = [int(v) for v in guess[s]]
            words = (w[0], w[1], w[2], w[4], w[5], w[6])
        want, sel = simulate(keys, r0, r1, cap, words)
        check_values(body[s], x, [r0, r1], f'tensor {i} slot {s}')
        check_state(states[i], want, f'tensor {i} (n={x.numel()}, cap={cap})')
        assert [int(k) for k in order_keys(body[s])] == sel


def ticket_only(sizes, grid):
    """(cta, tensor) pairs whose span overlaps a tensor by fewer elements than a vector after rounding (select.cu:569-586)."""
    prefix = np.concatenate([[0], np.cumsum(sizes)])
    total = int(prefix[-1])
    span = (total + grid - 1) // grid
    span = (span + 3) & ~3
    out = []
    for c in range(grid):
        s0, s1 = c * span, min(c * span + span, total)
        if s0 >= total: break
        for t, n in enumerate(sizes):
            if n <= 0 or prefix[t + 1] <= s0 or prefix[t] >= s1: continue
            a = max(s0 - prefix[t], 0); b = min(s1 - prefix[t], n)
            a = min((a + 3) & ~3, n)
            if b < n: b = min((b + 3) & ~3, n)
            if b <= a: out.append((c, t))
    return out


def sizes_with_ticket_only(count, max_n, total, r):
    """`count` tensor sizes summing to `total`, none above max_n, where a CTA of pass 0 and one of pass 1 each start 1-3 elements before
    the end of a tensor whose size is a multiple of 4: that CTA's share rounds to nothing (select.cu:579-586)."""
    g0, g1, _ = grids(count, max_n)
    cuts = [round(k * total / count) + int(r.randint(-total // (8 * count), total // (8 * count))) for k in range(1, count)]
    for g, c, k in ((g0, g0 // 2, 2), (g1, g1 // 3, 1)):
        span = (((total + g - 1) // g) + 3) & ~3
        b = c * span + k
        near = sorted(range(len(cuts)), key=lambda i: abs(cuts[i] - b))[:2]
        cuts[near[0]], cuts[near[1]] = b - 400, b
    sizes = list(np.diff([0] + sorted(cuts) + [total]))
    assert len(sizes) == count and min(sizes) >= 1 and max(sizes) <= max_n, sizes
    assert ticket_only(sizes, g0) and ticket_only(sizes, g1)
    return [int(v) for v in sizes]


def grids(count, max_n):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    work = count * max_n
    g0 = min(max((work + 16383) // 16384, 1), 2 * sms)                # select.cu:675-684
    g1 = min(max((work + 4095) // 4096, 1), 6 * sms)
    return g0, g1, min(g1, 2 * sms)


def test_table_spans_and_tickets(cabi):
    """Tensors at misaligned bases, sized so that some CTA of pass 0 and of pass 1 overlaps a tensor by 1-3 elements (the ticket-only
    path); post-ReLU and cap-sized buckets so that passes 1 and 2 run; scrambled slots; out_stride 3; caps 1 << 16, 64, 4 and 1."""
    r = np.random.RandomState(11)
    base = torch.from_numpy(r.standard_normal(1 << 22).astype(np.float32)).cuda()
    base[::3] = 0.0
    max_n = 401408
    sizes = sizes_with_ticket_only(9, max_n, 1000003, r)
    offs = [1, 2, 3, 5, 0, 6, 7, 9, 11]
    xs, at = [], 0
    for k, (n, o) in enumerate(zip(sizes, offs)):
        x = base[at + o: at + o + n]
        if k == 2: x = torch.relu(x)
        xs.append(x)
        at += o + n + 16
    slots = list(r.permutation(len(xs)))
    for cap in (1 << 16, 64, 4, 1):
        for q in (0.9999, 0.5, 0.0):
            rc, body, states, _ = table(cabi, xs, slots, q, cap, max_n=max_n)
            assert rc == 0
            check_table(xs, slots, q, cap, body, states)


def test_table_ticket_only_small_tensors(cabi):
    """Many tensors of at most cap / 2 elements, sized so that CTAs of pass 0 and pass 1 overlap a tensor by 1-3 elements: a missing
    ticket leaves that tensor's pass unresolved, and the state shows it (done != 0) even where the value happens to survive."""
    r = np.random.RandomState(17)
    cap = 1 << 15
    sizes = sizes_with_ticket_only(40, cap // 2, 240001, r)
    base = torch.from_numpy(r.standard_normal(sum(sizes) + 8 * len(sizes)).astype(np.float32)).cuda()
    xs, at = [], 0
    for k, n in enumerate(sizes):
        xs.append(base[at + k % 4: at + k % 4 + n])
        at += n + 4
    slots = list(r.permutation(len(xs)))
    for q in (0.9999, 0.5):
        rc, body, states, _ = table(cabi, xs, slots, q, cap, max_n=cap // 2)
        assert rc == 0
        check_table(xs, slots, q, cap, body, states)


def test_table_count_limit(cabi):
    """The span prefix lives in 24 KB of shared memory: 3071 tensors are accepted, 3072 refused before a launch."""
    r = np.random.RandomState(12)
    base = torch.from_numpy(r.standard_normal(3072 * 5).astype(np.float32)).cuda()
    xs = [base[5 * i: 5 * i + 1 + i % 5] for i in range(3072)]
    rc, _, _, _ = table(cabi, xs, list(range(3072)), 0.5, 4)
    assert rc == 1                                                       # cudaErrorInvalidValue
    xs = xs[:3071]
    slots = list(r.permutation(3071))
    rc, body, states, _ = table(cabi, xs, slots, 0.5, 4)
    assert rc == 0
    check_table(xs, slots, 0.5, 4, body, states)


def test_table_empty_entry(cabi):
    """An n = 0 entry has no order statistics: its slot keeps what it held and its guess words stay as they were; its neighbours are
    served as usual."""
    r = np.random.RandomState(13)
    xs = [f32(r.standard_normal(1000)), None, f32(r.standard_normal(77))]
    slots = [2, 0, 1]
    rc, body, states, _ = table(cabi, xs, slots, 0.99, 64)
    assert rc == 0 and (body[0] == SENT).all()
    check_table(xs, slots, 0.99, 64, body, states)
    guess = np.tile(np.uint32(INIT_GUESS), (3, 1))
    guess[0] = [123, 456, 789, 0, 1, 2, 3, 0]
    rc, body, states, g = table(cabi, xs, slots, 0.99, 64, guess=guess)
    assert rc == 0 and (body[0] == SENT).all() and list(g[0]) == [123, 456, 789, 0, 1, 2, 3, 0]


def test_speculation_table(cabi):
    """The table form's verdicts with a tiny cap: stored candidates cap / cap + 1 and need - 1 / need / need + 1 on different tensors of
    one call, threshold copies counted on a post-ReLU tensor, and the guess words after the call."""
    import oracle
    r = np.random.RandomState(14)
    cap, q = 64, 0.999
    xs, words = [], []
    d = 1 << 14
    for k, (dc, kind) in enumerate([(-1, 'n'), (0, 'n'), (1, 'n'), ('cap', 'n'), ('cap+1', 'n'), ('veq', 'relu')]):
        x = spec_input(r, 40000)
        if kind == 'relu': x = np.maximum(x, 0)
        n = x.size
        r0, r1 = oracle.quantile_ranks(n, q)
        srt = np.sort(order_keys(x).astype(np.int64))
        need_hi, need_lo = n - r0, r1 + 1
        if dc == 'cap': c_hi = c_lo = cap
        elif dc == 'cap+1': c_hi = c_lo = cap + 1
        elif dc == 'veq': c_hi = c_lo = None
        else: c_hi, c_lo = need_hi + dc, need_lo + dc
        if c_hi is None:
            kz = int(order_keys(np.float32([0.0]))[0])
            words.append([int(srt[n - need_hi - 3]), 0, d, 0, kz, kz, d, 0])
        else:
            words.append([int(srt[n - c_hi]), 0, d, 0, int(srt[c_lo - 1]), 0xFFFFFFFF, d, 0])
        xs.append(f32(x))
    slots = [3, 0, 5, 1, 4, 2]
    guess = np.zeros((6, 8), np.uint32)
    for w, s in zip(words, slots): guess[s] = w
    rc, body, states, g = table(cabi, xs, slots, q, cap, guess=guess)
    assert rc == 0
    check_table(xs, slots, q, cap, body, states, guess=guess)
    verdict = [[st['mode'][k] == COMPACT and st['clevel'][k] == 0 for k in (0, 1)] for st in states]
    assert verdict[0] == [False, False] and verdict[1] == [True, True] and verdict[2] == [True, True]
    assert verdict[4] == [False, False] and states[4]['d'] == [d // 2, d // 2]
    assert states[5]['veq'][1] > 10000 and verdict[5][1]
    for st, x, s in zip(states, xs, slots):
        keys = [int(k) for k in order_keys(body[s])]
        assert list(g[s]) == next_guess(keys[0], st['d'][0], 0) + next_guess(keys[1], st['d'][1], 1)


# ---------------------------------------------------------------------------------------------------------------- isotone and half
def test_isotone(cabi):
    import oracle
    r = np.random.RandomState(15)
    ws = torch.empty(cabi.ppq_b200_quantile_workspace_bytes(), dtype=torch.uint8, device='cuda')
    for n in (1, 2, 3, 5, 4097, 100003):
        for kind in ('randn', 'zeros', 'nan'):
            x = r.standard_normal(n).astype(np.float32)
            if kind == 'zeros': x[r.rand(n) < 0.7] = -0.0
            if kind == 'nan': x[r.randint(n, size=max(1, n // 50))] = np.uint32(0xFFC00001).view(np.float32)
            xd = f32(x)
            out = torch.full((6,), float(SENT), device='cuda')
            assert cabi.ppq_b200_isotone_t(V(xd.data_ptr()), n, V(out.data_ptr() + 4), V(ws.data_ptr()), stream()) == 0
            o = out.cpu().numpy()
            assert o[0] == SENT and o[5] == SENT
            assert np.array_equal(bits(o[1:5]), bits(oracle.isotone_t(x, 'device'))), (n, kind)
            ref = oracle.isotone_t(x, 'reference')
            assert np.array_equal(o[1:5][~np.isnan(ref)], ref[~np.isnan(ref)]), (n, kind)


@pytest.mark.parametrize('dtype', [BF16, F16], ids=['bf16', 'fp16'])
def test_half_inputs(cabi, dtype):
    """bf16 / fp16 through the single-tensor forms: the oracle and the route on the exact fp32 upcast.  bf16 repeats values, so its
    buckets resolve from one value."""
    r = np.random.RandomState(16 + dtype)
    tdt = torch.bfloat16 if dtype == BF16 else torch.float16
    for n in (1, 5, 4097, 300001, 2 * CAP + 17):
        x = torch.from_numpy(r.standard_normal(n).astype(np.float32)).cuda().to(tdt)
        x[::4] = 0.0
        x[1::9] = -0.0
        for q in (0.9999, 0.5, 0.0):
            run_case(cabi, x, q, f'{tdt} n={n} q={q}', dtype=dtype)
        if n > 1:
            run_case(cabi, x[1:], 0.99, f'{tdt} n={n} offset', dtype=dtype)     # an odd storage offset
    st, _, _ = run_case(cabi, torch.relu(torch.from_numpy(r.standard_normal(CAP * 3).astype(np.float32)).cuda()).to(tdt), 0.3,
                        f'{tdt} relu', dtype=dtype)
    assert st['mode'][0] == DONE and st['count'][0] > CAP                # rank 0 among the zeros: one value, resolved in pass 1
