"""The stream contract of every binding that launches device work (include/ppq_b200.h: kernels are enqueued on `stream`, nothing
synchronises, nothing allocates), held to the oracle in three launch contexts:

  A. side-stream gate   poison the buffers, sleep ~250 ms on a fresh (non-blocking) stream s, load data set k and call the entry on s.
                        The call must return before the sleep ends (the host did not wait), and the results, read on s, must equal the
                        oracle's: a launch on any other stream would read the poison.  A second pass sleeps on the default (legacy) stream
                        instead and reads the results on s while the default stream is still asleep: work queued behind the legacy stream
                        has not run yet, so the results would be stale.
  B. graph replay       one eager warm-up on a side stream, then capture under torch.cuda.graph (capture_error_mode "global": any use of
                        the legacy stream during capture raises).  Each replay runs on new contents of the same buffers -- new inputs and
                        new values in the static scale / offset / histogram-scale tensors -- chosen so that the device takes a different
                        route from the captured one.  Data set 0 replayed again must be bit-identical to its first replay (except for the
                        fp32 atomic sums of the training kernels).
  C. carried state      the guess words of Quantile_T_Guess and Multi_Quantile_T after a captured sequence hit, miss, hit, heavy tail,
                        hit equal the words the same sequence leaves when run eagerly.

CASES maps every launching binding name to its builders; tests/test_cpu_stream_contract.py fails when a name exported by
torch_binding.cc / torch_binding_more.inc has no case.  Importing this module does not touch CUDA: the builders run inside the tests.

Comparison rules are those of the route tests: bits (any NaN matches any NaN) for fake-quant, integers, counts, min/max, selected elements,
scales and offsets; the chain-length bounds of test_gpu_training_kernels.py for grad_s and the rounding loss; layerwise_oracle.moments_bound
for the paired moments; the KL argmin tie rule of DESIGN.md §2 deviation 2.
"""
import builtins
import contextlib
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F32 = np.float32
NAN, INF = float('nan'), float('inf')
SENT = -7.5                                            # poison of output slots an entry must leave alone
INIT_GUESS = [0xFFFFFFFF, 0xFFFFFFFF, 1 << 19, 0, 0, 0, 1 << 19, 0]
GATE_MS = 250.0                                        # long enough that a collector pause or a clock change cannot end it early

# Exported names that launch nothing on the device.
HOST_ONLY = {'compute_mse_loss', 'Multi_Quantile_Workspace_Bytes', 'Multi_Paired_Moments_Workspace_Bytes', 'abi_version', 'build_info',
             'set_variant', 'get_variant'}

CASES = {}                                             # binding name -> {label: (builder, knob, params)}


def case(name, *variants):
    """Register a builder for `name`.  variants: (label, knob, params); knob = (kernel, value) for set_variant, or None."""
    def reg(fn):
        for label, knob, params in (variants or [('default', None, {})]):
            CASES.setdefault(name, {})[label] = (fn, knob, params)
        return fn
    return reg


def case_ids():
    return [(n, lab) for n in CASES for lab in CASES[n]]


# ------------------------------------------------------------------------------------------------------------------ helpers
def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def host(t):
    return t.detach().float().cpu().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.detach().cpu().numpy()


def same(got, want, what, zero_sign=True):
    """Bit-identical; any NaN matches any NaN (floats), exact for integers.  zero_sign=False: +0 also matches -0, the rule of the scale and
    offset tests (an offset of -0.0 is rint(-0.0 / scale))."""
    g = got.reshape(-1) if isinstance(got, np.ndarray) else np.asarray(got).reshape(-1)
    w = np.asarray(want).reshape(-1)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    if g.dtype.kind == 'f':
        w = w.astype(g.dtype)
        ib = {2: np.int16, 4: np.int32, 8: np.int64}[g.dtype.itemsize]
        bad = (g.view(ib) != w.view(ib)) & ~(np.isnan(g) & np.isnan(w))
        if not zero_sign: bad &= ~((g == 0) & (w == 0))
    else:
        bad = g != w.astype(g.dtype)
    assert not bad.any(), (what, int(bad.sum()), np.flatnonzero(bad)[:5], g[bad][:5], w[bad][:5])


def same_half(got_t, want32, what):
    """A half result against the fp32 oracle on the exact upcast, rounded once: compare as the half bit patterns."""
    want = torch.from_numpy(np.ascontiguousarray(want32, F32)).to(got_t.dtype)
    g, w = got_t.reshape(-1).view(torch.int16).numpy(), want.reshape(-1).view(torch.int16).numpy()
    gn, wn = torch.isnan(got_t.reshape(-1).float()).numpy(), torch.isnan(want.reshape(-1).float()).numpy()
    bad = (g != w) & ~(gn & wn)
    assert not bad.any(), (what, int(bad.sum()), np.flatnonzero(bad)[:5])


def zero_signs(x, lo, hi):
    """The collectors' order of signed zeros (test_gpu_collector_routes.py::test_minmax_signed_zeros_across_ctas): a zero minimum is -0 when
    any -0 is present, a zero maximum +0 when any +0 is."""
    z = x[x == 0]
    neg, pos = bool(np.signbit(z).any()), bool((~np.signbit(z)).any())
    return (F32(-0.0 if neg else 0.0) if lo == 0 else F32(lo)), (F32(0.0 if pos else -0.0) if hi == 0 else F32(hi))


def minmax_want(oracle, x):
    lo, hi = oracle.minmax_t(x)
    return np.array(zero_signs(x.reshape(-1), lo, hi), F32)


def minmax_c_want(oracle, x, axis):
    lo, hi = oracle.minmax_c(x, axis)
    epc, C = oracle.channel_geometry(x.shape, axis)
    ch = (np.arange(x.size) // epc) % C
    pairs = [zero_signs(x.reshape(-1)[ch == c], lo[c], hi[c]) for c in range(C)]
    return np.array([p[0] for p in pairs], F32), np.array([p[1] for p in pairs], F32)


def specials(r, x, k=7):
    """x with NaN payloads of both signs, +-inf and +-0 at random places."""
    x = np.array(x, F32, copy=True).reshape(-1)
    sp = np.uint32([0x7FC00000, 0xFFC00001, 0x7F800001, 0x7F800000, 0xFF800000, 0x00000000, 0x80000000]).view(F32)[:min(k, x.size)]
    x[r.choice(x.size, sp.size, replace=False)] = sp
    return x


class Inst:
    """Static buffers of one case.  bank[key][k]: data set k on the device; load(k) copies it into buf[key] with ordinary device ops.
    run(buf) calls the entry (after resetting any accumulator it adds into) and returns the output tensors; check(k, outs) compares
    host copies of them with the oracle on data set k.  `poison` lists outputs an entry writes in place: they get NaN / SENT / -1."""

    def __init__(self, bank, run, check, exact=True, poison=()):
        self.bank = {k: [v if isinstance(v, torch.Tensor) else dev(v) for v in vs] for k, vs in bank.items()}
        self.K = len(next(iter(self.bank.values())))
        assert all(len(v) == self.K for v in self.bank.values())
        self.buf = {k: v[0].clone() for k, v in self.bank.items()}
        self.np = {k: [host(t) for t in v] for k, v in self.bank.items()}
        self._run, self._check, self.exact, self.poison_list = run, check, exact, list(poison)
        self._want = {}

    def load(self, k):
        for key, b in self.buf.items(): b.copy_(self.bank[key][k])

    def poison(self):
        for t, v in self.poison_list: t.fill_(v)

    def run(self):
        out = self._run(self.buf)
        return list(out) if isinstance(out, (list, tuple)) else [out]

    def want(self, k, fn):
        if k not in self._want: self._want[k] = fn(k)
        return self._want[k]

    def check(self, k, outs):
        self._check(self, k, outs)


@contextlib.contextmanager
def knob(ext, kn):
    if kn is None:
        yield
        return
    assert ext.set_variant(kn[0], kn[1]) == 0
    try:
        yield
    finally:
        ext.set_variant(kn[0], 0)


def readback(outs, stream, pins):
    """Copy `outs` to pinned host buffers on `stream` and wait for that stream only."""
    with torch.cuda.stream(stream):
        for p, o in zip(pins, outs): p.copy_(o, non_blocking=True)
    stream.synchronize()
    return [p.clone() for p in pins]


def pinned_like(outs):
    return [torch.empty(o.shape, dtype=o.dtype).pin_memory() for o in outs]


# ------------------------------------------------------------------------------------------------------------------ fake-quant
QMIN, QMAX = -128, 127
# per data set: (scale, offset); 2^-70 and 2^70 leave the exactly divided range, NaN propagates
LT_PARAMS = [(0.05, 0.0), (3e-3, 3.0), (2.0 ** -70, -5.0), (2.0 ** 70, 0.5), (NAN, 0.0)]


def xs_for(n, seed, sets=5, shape=None):
    r = np.random.RandomState(seed)
    out = []
    for k in range(sets):
        s = [1.0, 0.5, 2.0 ** -70, 2.0 ** 70, 1.0][k % 5]
        x = specials(r, (r.standard_normal(n) * 3 * s).astype(F32))
        out.append(x.reshape(shape) if shape else x)
    return out


def chan_params(C, sets=5, seed=1):
    r = np.random.RandomState(seed)
    sc, of = [], []
    for k in range(sets):
        base = LT_PARAMS[k][0]
        s = (base * r.uniform(0.5, 2.0, C)).astype(F32)
        s[0] = base
        if C > 2: s[1] = 2.0 ** -75; s[2] = NAN if k else 0.02
        sc.append(s)
        of.append(np.round(r.uniform(-4, 4, C) * 2).astype(F32) / 2)
    return sc, of


def lq_check_t(inst, k, outs, half=None):
    s, o = float(inst.np['s'][k][0]), float(inst.np['o'][k][0])
    want = inst.want(k, lambda k: inst.oracle.linear_quant_t(inst.np['x'][k], s, o, QMIN, QMAX, 0))
    (same_half(outs[0], want, f'LT set {k}') if half else same(outs[0].numpy(), want, f'LT set {k}'))


@case('QuantizeTensor_LT', ('default', None, {}), ('tma', ('linear_quant_t', 1), {}))
def build_lt(ext, oracle, half=None):
    n = (1 << 18) + 3
    xs = xs_for(n, 11)
    bank = {'x': [dev(x, half) for x in xs], 's': [F32([p[0]]) for p in LT_PARAMS], 'o': [F32([p[1]]) for p in LT_PARAMS]}
    fn = ext.QuantizeTensor_LT_Half if half else ext.QuantizeTensor_LT
    inst = Inst(bank, lambda b: fn(b['x'], b['s'], b['o'], QMIN, QMAX, 0), lambda i, k, o: lq_check_t(i, k, o, half))
    if half:                                                     # the oracle works on the exact upcast
        inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    return inst


@case('QuantizeTensor_LT_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_lt_half(ext, oracle, half):
    return build_lt(ext, oracle, half)


def lc_check(inst, k, outs, axis, half=None, floating=None):
    if floating:
        E, M, cmin, cmax = floating
        f = lambda k: inst.oracle.float_quant_c(inst.np['x'][k], inst.np['s'][k], inst.np['o'][k], axis, E, M, cmin, cmax, 0)
    else:
        f = lambda k: inst.oracle.linear_quant_c(inst.np['x'][k], inst.np['s'][k], inst.np['o'][k], axis, QMIN, QMAX, 0)
    want = inst.want(k, f)
    (same_half(outs[0], want, f'C set {k}') if half else same(outs[0].numpy(), want, f'C set {k}'))


@case('QuantizeTensor_LC', ('default', None, {}), ('table1', ('linear_quant_c', 1), {}))
def build_lc(ext, oracle, half=None, floating=None):
    shape, axis = (4, 24, 37), 1
    xs = xs_for(int(np.prod(shape)), 12, shape=shape)
    sc, of = chan_params(shape[axis])
    if floating: of = [np.zeros_like(o) for o in of]
    bank = {'x': [dev(x, half) for x in xs], 's': sc, 'o': of}
    if floating:
        E, M, cmin, cmax = floating
        fn = ext.QuantizeTensor_FC_Half if half else ext.QuantizeTensor_FC
        run = lambda b: fn(b['x'], b['s'], b['o'], E, M, cmin, cmax, axis, 0)
    else:
        fn = ext.QuantizeTensor_LC_Half if half else ext.QuantizeTensor_LC
        run = lambda b: fn(b['x'], b['s'], b['o'], QMIN, QMAX, axis, 0)
    inst = Inst(bank, run, lambda i, k, o: lc_check(i, k, o, axis, half, floating))
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    return inst


@case('QuantizeTensor_LC_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_lc_half(ext, oracle, half):
    return build_lc(ext, oracle, half)


FP8 = (4, 3, -448.0, 448.0)
FT_PARAMS = [(1.0, 0.0), (0.01, 0.0), (2.0 ** -70, 0.0), (2.0 ** 70, 0.0), (NAN, 0.0)]


def ft_check(inst, k, outs, half):
    s, o = float(inst.np['s'][k][0]), float(inst.np['o'][k][0])
    want = inst.want(k, lambda k: inst.oracle.float_quant_t(inst.np['x'][k], s, o, *FP8, 0))
    (same_half(outs[0], want, f'FT set {k}') if half else same(outs[0].numpy(), want, f'FT set {k}'))


@case('QuantizeTensor_FT')
def build_ft(ext, oracle, half=None):
    xs = xs_for(70001, 13)
    bank = {'x': [dev(x, half) for x in xs], 's': [F32([p[0]]) for p in FT_PARAMS], 'o': [F32([p[1]]) for p in FT_PARAMS]}
    fn = ext.QuantizeTensor_FT_Half if half else ext.QuantizeTensor_FT
    inst = Inst(bank, lambda b: fn(b['x'], b['s'], b['o'], *FP8, 0), lambda i, k, o: ft_check(i, k, o, half))
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    return inst


@case('QuantizeTensor_FT_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_ft_half(ext, oracle, half):
    return build_ft(ext, oracle, half)


@case('QuantizeTensor_FC')
def build_fc(ext, oracle, half=None):
    return build_lc(ext, oracle, half, FP8)


@case('QuantizeTensor_FC_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_fc_half(ext, oracle, half):
    return build_lc(ext, oracle, half, FP8)


def toint_check(inst, k, outs, axis):
    def f(k):
        x, s, o = inst.np['x'][k], inst.np['s'][k], inst.np['o'][k]
        if axis is None: return inst.oracle.linear_quant_t(x, float(s[0]), float(o[0]), QMIN, QMAX, 0, return_int=True)[1]
        return inst.oracle.linear_quant_c(x, s, o, axis, QMIN, QMAX, 0, return_int=True)[1]
    same(outs[0].numpy(), inst.want(k, f), f'toInt set {k}')


@case('QuantizeTensor_toInt', ('T8', None, {'axis': None, 'bits': 8}), ('T32', None, {'axis': None, 'bits': 32}),
      ('C8', None, {'axis': 1, 'bits': 8}), ('C8_bf16', None, {'axis': 1, 'bits': 8, 'half': torch.bfloat16}))
def build_toint(ext, oracle, axis, bits, half=None):
    shape = (4, 24, 37)
    xs = xs_for(int(np.prod(shape)), 14, shape=shape)
    if axis is None:
        sc, of = [F32([p[0]]) for p in LT_PARAMS], [F32([p[1]]) for p in LT_PARAMS]
    else:
        sc, of = chan_params(shape[axis], seed=2)
    bank = {'x': [dev(x, half) for x in xs], 's': sc, 'o': of}
    ax = -1000 if axis is None else axis
    inst = Inst(bank, lambda b: ext.QuantizeTensor_toInt(b['x'], b['s'], b['o'], QMIN, QMAX, ax, 0, bits), lambda i, k, o: toint_check(i, k, o, axis))
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    return inst


def table_tensors(sizes, sets, seed, half=None):
    r = np.random.RandomState(seed)
    return [[dev(specials(r, r.standard_normal(n).astype(F32) * (1 + k) * [1, 1, 1e-3, 30, 1][k % 5], min(7, n)), half) for k in range(sets)]
            for n in sizes]


@case('Multi_QuantizeTensor_LT')
def build_multi_lt(ext, oracle):
    sizes, K = [70001, 1, 4096, 333], 5
    xs = table_tensors(sizes, K, 21)
    bank = {f'x{i}': xs[i] for i in range(len(sizes))}
    for i in range(len(sizes)):                                   # each row its own scale / offset, moving between data sets
        bank[f's{i}'] = [F32([LT_PARAMS[(k + i) % 5][0]]) for k in range(K)]
        bank[f'o{i}'] = [F32([LT_PARAMS[(k + i) % 5][1]]) for k in range(K)]
    inst = Inst(bank, None, None)
    ys = [torch.empty(n, device='cuda') for n in sizes]
    b = inst.buf
    descs = torch.tensor([[b[f'x{i}'].data_ptr(), ys[i].data_ptr(), b[f's{i}'].data_ptr(), b[f'o{i}'].data_ptr(), n] for i, n in enumerate(sizes)],
                         dtype=torch.int64, device='cuda')

    def run(b):
        ext.Multi_QuantizeTensor_LT(descs, max(sizes), QMIN, QMAX, 0)
        return ys

    def check(inst, k, outs):
        for i in range(len(sizes)):
            want = oracle.linear_quant_t(inst.np[f'x{i}'][k], float(inst.np[f's{i}'][k][0]), float(inst.np[f'o{i}'][k][0]), QMIN, QMAX, 0)
            same(outs[i].numpy(), want, f'multi LT row {i} set {k}')
    inst._run, inst._check, inst.poison_list, inst.keep = run, check, [(y, NAN) for y in ys], descs
    return inst


@case('Multi_QuantizeTensor_LC', ('default', None, {}))
def build_multi_lc(ext, oracle, half=None):
    shapes, K = [(16, 3, 3, 3), (1, 5), (64, 129), (3, 1)], 5
    xs = table_tensors([int(np.prod(s)) for s in shapes], K, 22, half)
    bank = {f'x{i}': xs[i] for i in range(len(shapes))}
    for i, sh in enumerate(shapes):
        sc, of = chan_params(sh[0], K, seed=30 + i)
        bank[f's{i}'], bank[f'o{i}'] = sc, of
    inst = Inst(bank, None, None)
    if half:
        for i in range(len(shapes)): inst.np[f'x{i}'] = [host(t.float()) for t in inst.bank[f'x{i}']]
    ys = [torch.empty(int(np.prod(s)), device='cuda', dtype=half or torch.float32) for s in shapes]
    b = inst.buf
    rows = []
    for i, sh in enumerate(shapes):
        n = int(np.prod(sh))
        rows.append([b[f'x{i}'].data_ptr(), ys[i].data_ptr(), b[f's{i}'].data_ptr(), b[f'o{i}'].data_ptr(), n, n // sh[0], sh[0]])
    descs = torch.tensor(rows, dtype=torch.int64, device='cuda')
    max_n = max(int(np.prod(s)) for s in shapes)

    def run(b):
        if half: ext.Multi_QuantizeTensor_LC_Half(descs, max_n, half, QMIN, QMAX, 0)
        else: ext.Multi_QuantizeTensor_LC(descs, max_n, QMIN, QMAX, 0)
        return ys

    def check(inst, k, outs):
        for i, sh in enumerate(shapes):
            want = oracle.linear_quant_c(inst.np[f'x{i}'][k].reshape(sh[0], -1), inst.np[f's{i}'][k], inst.np[f'o{i}'][k], 0, QMIN, QMAX, 0)
            (same_half(outs[i], want, f'multi LC row {i} set {k}') if half else same(outs[i].numpy(), want, f'multi LC row {i} set {k}'))
    inst._run, inst._check, inst.poison_list, inst.keep = run, check, [(y, NAN) for y in ys], descs
    return inst


@case('Multi_QuantizeTensor_LC_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_multi_lc_half(ext, oracle, half):
    return build_multi_lc(ext, oracle, half)


# ------------------------------------------------------------------------------------------------------------------ collectors
BINS = 2048


def coll_xs(n, seed, sets=5, half=None):
    """Sets with different extremes: plain, with NaN / inf, all signed zeros, clipped outliers, tiny."""
    r = np.random.RandomState(seed)
    out = []
    for k in range(sets):
        x = (r.standard_normal(n) * [2.0, 2.0, 0.0, 40.0, 1e-3][k % 5]).astype(F32)
        if k % 5 == 1: x = specials(r, x, 5)                     # NaN payloads and +-inf (no zeros: those are set 2)
        if k % 5 == 2: x[r.rand(n) < 0.5] = -0.0
        out.append(dev(x, half))
    return out


def hist_check(inst, k, outs, f):
    same(outs[0].numpy(), inst.want(k, f), f'histogram set {k}')


@case('Histogram_T', *[(f'v{v}_clip{int(c)}', ('histogram', v), {'clip': c}) for v in range(9) for c in (True, False)
                       if c or v in (0, 3)])
def build_hist_t(ext, oracle, clip):
    hs = F32(4.0 / BINS)
    inst = Inst({'x': coll_xs(300007, 31)}, None, None)
    hist = torch.empty(BINS, dtype=torch.int32, device='cuda')

    def run(b):
        hist.zero_(); ext.Histogram_T(b['x'], float(hs), clip, hist)
        return hist
    inst._run = run
    inst._check = lambda i, k, o: hist_check(i, k, o, lambda k: oracle.histogram_t(i.np['x'][k], hs, BINS, clip))
    return inst


@case('Histogram_Asymmetric_T', ('clip', None, {'clip': True}), ('noclip', None, {'clip': False}))
def build_hist_asym(ext, oracle, clip, half=None):
    lo, hi = -3.0, 5.0
    inst = Inst({'x': coll_xs(200003, 32, half=half)}, None, None)
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    hist = torch.empty(BINS, dtype=torch.int32, device='cuda')
    fn = ext.Histogram_Asymmetric_T_Half if half else ext.Histogram_Asymmetric_T

    def run(b):
        hist.zero_(); fn(lo, hi, b['x'], clip, hist)
        return hist
    inst._run = run
    inst._check = lambda i, k, o: hist_check(i, k, o, lambda k: oracle.histogram_asym_t(i.np['x'][k], lo, hi, BINS, clip))
    return inst


@case('Histogram_Asymmetric_T_Half', ('fp16', None, {'half': torch.float16, 'clip': True}), ('bf16', None, {'half': torch.bfloat16, 'clip': False}))
def build_hist_asym_half(ext, oracle, half, clip):
    return build_hist_asym(ext, oracle, clip, half)


@case('Histogram_C', ('clip', None, {'clip': True}), ('noclip', None, {'clip': False}))
def build_hist_c(ext, oracle, clip):
    shape, bins = (3, 8, 4099), 512
    hs = F32(4.0 / bins)
    xs = [t.view(shape) for t in coll_xs(int(np.prod(shape)), 33)]
    inst = Inst({'x': xs}, None, None)
    hist = torch.empty(shape[1] * bins, dtype=torch.int32, device='cuda')

    def run(b):
        hist.zero_(); ext.Histogram_C(b['x'], 1, float(hs), clip, hist)
        return hist
    inst._run = run
    inst._check = lambda i, k, o: hist_check(i, k, o, lambda k: oracle.histogram_c(i.np['x'][k], 1, hs, bins, clip))
    return inst


HSCALES = [4.0 / BINS, 0.0, NAN, -1.0 / BINS, 1e-30]             # device histogram scales, one per data set


@case('Histogram_T_DeviceScale', *[(f'{b}_clip{int(c)}', None, {'bins': b, 'clip': c}) for b in (BINS, 16384) for c in (True, False)],
      ('bf16', None, {'bins': BINS, 'clip': True, 'half': torch.bfloat16}))
def build_hist_dscale(ext, oracle, bins, clip, half=None):
    inst = Inst({'x': coll_xs(250001, 34, half=half), 'hs': [F32([h]) for h in HSCALES]}, None, None)
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    hist = torch.empty(bins, dtype=torch.int32, device='cuda')

    def run(b):
        hist.zero_(); ext.Histogram_T_DeviceScale(b['x'], b['hs'], clip, hist)
        return hist
    inst._run = run
    inst._check = lambda i, k, o: hist_check(i, k, o, lambda k: oracle.histogram_t(i.np['x'][k], F32(i.np['hs'][k][0]), bins, clip))
    return inst


@case('MinMax_Init')
def build_minmax_init(ext, oracle):
    inst = Inst({'dummy': [F32([k]) for k in range(3)]}, None, None)
    mins, maxs = torch.empty(300, device='cuda'), torch.empty(300, device='cuda')

    def run(b):
        ext.MinMax_Init(mins, maxs)
        return [mins, maxs]

    def check(inst, k, outs):
        same(outs[0].numpy(), np.full(300, INF, F32), 'mins'); same(outs[1].numpy(), np.full(300, -INF, F32), 'maxs')
    inst._run, inst._check, inst.poison_list = run, check, [(mins, NAN), (maxs, NAN)]
    return inst


@case('MinMax_T', ('fp32', None, {}), ('fp16', None, {'half': torch.float16}))
def build_minmax_t(ext, oracle, half=None):
    inst = Inst({'x': coll_xs(300007, 35, half=half)}, None, None)
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    mm = torch.empty(2, device='cuda')

    def run(b):
        ext.MinMax_Init(mm[0:1], mm[1:2]); ext.MinMax_T(b['x'], mm)
        return mm
    inst._run = run
    inst._check = lambda i, k, o: same(o[0].numpy(), np.array(i.want(k, lambda k: minmax_want(oracle, i.np['x'][k])), F32), f'minmax set {k}')
    return inst


@case('MinMax_C', ('fp32', None, {}), ('bf16', None, {'half': torch.bfloat16}))
def build_minmax_c(ext, oracle, half=None):
    shape = (5, 6, 3001)
    inst = Inst({'x': [t.view(shape) for t in coll_xs(int(np.prod(shape)), 36, half=half)]}, None, None)
    if half: inst.np['x'] = [host(t.float()) for t in inst.bank['x']]
    mins, maxs = torch.empty(6, device='cuda'), torch.empty(6, device='cuda')

    def run(b):
        ext.MinMax_Init(mins, maxs); ext.MinMax_C(b['x'], 1, mins, maxs)
        return [mins, maxs]

    def check(inst, k, outs):
        lo, hi = inst.want(k, lambda k: minmax_c_want(oracle, inst.np['x'][k], 1))
        same(outs[0].numpy(), lo, f'mins set {k}'); same(outs[1].numpy(), hi, f'maxs set {k}')
    inst._run, inst._check = run, check
    return inst


TABLE_SIZES = [300007, 1, 4099, 70001]
TABLE_SLOTS = [2, 0, 3, 1]


def table_descs(inst, sizes, slots, prefix='x'):
    return torch.tensor([[inst.buf[f'{prefix}{i}'].data_ptr(), n, s] for i, (n, s) in enumerate(zip(sizes, slots))], dtype=torch.int64, device='cuda')


def table_bank(sizes, seed, half=None, K=5):
    return {f'x{i}': coll_xs(n, seed + i, K, half) for i, n in enumerate(sizes)}


@case('Multi_MinMax_T', ('fp32', None, {}))
def build_multi_minmax(ext, oracle, half=None):
    inst = Inst(table_bank(TABLE_SIZES, 40, half), None, None)
    if half:
        for i in range(len(TABLE_SIZES)): inst.np[f'x{i}'] = [host(t.float()) for t in inst.bank[f'x{i}']]
    descs = table_descs(inst, TABLE_SIZES, TABLE_SLOTS)
    arena = torch.empty(len(TABLE_SIZES), 2, device='cuda')

    def run(b):
        arena[:, 0] = INF; arena[:, 1] = -INF
        if half: ext.Multi_MinMax_T_Half(descs, max(TABLE_SIZES), half, arena)
        else: ext.Multi_MinMax_T(descs, max(TABLE_SIZES), arena)
        return arena

    def check(inst, k, outs):
        for i, s in enumerate(TABLE_SLOTS):
            same(outs[0][s].numpy(), minmax_want(oracle, inst.np[f'x{i}'][k]), f'multi minmax row {i} set {k}')
    inst._run, inst._check, inst.keep = run, check, descs
    return inst


@case('Multi_MinMax_T_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_multi_minmax_half(ext, oracle, half):
    return build_multi_minmax(ext, oracle, half)


@case('Multi_Histogram_T', ('clip', None, {'clip': True}), ('noclip', None, {'clip': False}))
def build_multi_hist(ext, oracle, clip, half=None):
    bank = table_bank(TABLE_SIZES, 50, half)
    count = len(TABLE_SIZES)
    bank['hs'] = [F32([HSCALES[(k + j) % 5] for j in range(count)]) for k in range(5)]      # every slot's scale moves between sets
    inst = Inst(bank, None, None)
    if half:
        for i in range(count): inst.np[f'x{i}'] = [host(t.float()) for t in inst.bank[f'x{i}']]
    descs = table_descs(inst, TABLE_SIZES, TABLE_SLOTS)
    hist = torch.empty(count * BINS, dtype=torch.int32, device='cuda')

    def run(b):
        hist.zero_()
        if half: ext.Multi_Histogram_T_Half(descs, max(TABLE_SIZES), half, b['hs'], clip, hist, BINS)
        else: ext.Multi_Histogram_T(descs, max(TABLE_SIZES), b['hs'], clip, hist, BINS)
        return hist

    def check(inst, k, outs):
        h = outs[0].numpy().reshape(count, BINS)
        for i, s in enumerate(TABLE_SLOTS):
            same(h[s], oracle.histogram_t(inst.np[f'x{i}'][k], F32(inst.np['hs'][k][s]), BINS, clip), f'multi hist row {i} set {k}')
    inst._run, inst._check, inst.keep = run, check, descs
    return inst


@case('Multi_Histogram_T_Half', ('fp16', None, {'half': torch.float16, 'clip': True}), ('bf16', None, {'half': torch.bfloat16, 'clip': False}))
def build_multi_hist_half(ext, oracle, half, clip):
    return build_multi_hist(ext, oracle, clip, half)


# ------------------------------------------------------------------------------------------------------------------ radix select
SEL_CAP = 1 << 18                                                # the single-tensor entry's cap (select.cu kDefaultCap)
SAMPLE_KEYS = 16384


def select_sets(n, seed, cap):
    """Data sets whose selections take different routes: 0 randn (captured), 1 randn with NaN payloads, +-inf and +-0 (a guess hit after
    0), 2 randn x 50 (a miss), 3 a top-digit bucket of > cap close values (histogrammed to level 2), 4 a heavy tail (more keys beyond any
    remembered threshold than the buffer holds), 5 post-ReLU zeros and negated zeros (one-value buckets)."""
    r = np.random.RandomState(seed)
    out = [r.standard_normal(n).astype(F32), specials(r, r.standard_normal(n).astype(F32)), (r.standard_normal(n) * 50).astype(F32)]
    m = min(n // 2 - 1, cap + max(8, cap // 50))
    close = (F32(100.0).view(np.uint32) + r.randint(0, 1024, m).astype(np.uint32)).view(F32)     # both ranks inside these buckets
    x = np.concatenate([close, -close, r.standard_normal(n - 2 * m).astype(F32) * 10])
    out.append(x[r.permutation(n)])
    x = r.standard_normal(n).astype(F32)
    heavy = r.rand(n) < 0.7
    x[heavy] = r.uniform(1000, 2000, int(heavy.sum())).astype(F32) * np.where(r.rand(int(heavy.sum())) < 0.5, -1, 1)
    out.append(x)
    x = r.standard_normal(n).astype(F32)
    x[r.rand(n) < 0.45] = 0.0
    x[r.rand(n) < 0.45] = -0.0
    out.append(x)
    return out


def sel_expected(x, ranks):
    from test_gpu_select_paths import expected
    return expected(x, ranks)


def quantile_check(inst, k, outs, q):
    x = inst.bank['x'][k]
    want = inst.want(k, lambda k: sel_expected(x, list(inst.oracle.quantile_ranks(x.numel(), q))))
    same(outs[0].numpy(), want, f'quantile set {k}')


Q = 0.999


@case('Quantile_T', ('default', None, {}), ('select_p0_4_p1_2', ('select', 4 | (2 << 3)), {}),
      ('sampled', None, {'sampled': True}))
def build_quantile(ext, oracle, sampled=False, half=None, guess=False):
    if sampled:
        # n >= 2^23 without a guess: thresholds from a sample.  Set 1 plants large values at the sampled positions: the sampled threshold
        # then lies above all but a handful of elements and the speculation misses; sets 0 and 2 hit.
        n = (1 << 23) + 4099
        r = np.random.RandomState(60)
        xs = [r.standard_normal(n).astype(F32) for _ in range(3)]
        stride = n // SAMPLE_KEYS
        i = np.arange(SAMPLE_KEYS, dtype=np.uint64)
        pos = (i * np.uint64(stride) + ((i * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) % np.uint64(stride)).astype(np.int64)
        xs[1][pos] = r.uniform(100, 200, SAMPLE_KEYS).astype(F32)
        xs[2] *= 3
        q = 0.9999
    else:
        xs, q = select_sets(600000, 61, SEL_CAP), Q
    inst = Inst({'x': [dev(x, half) for x in xs]}, None, None)
    g = ext.Quantile_Guess_Init(1, inst.buf['x']) if guess else None
    torch.cuda.synchronize()

    def run(b):
        if guess: return ext.Quantile_T_Guess(b['x'], q, g)
        return ext.Quantile_T_Half(b['x'], q) if half else ext.Quantile_T(b['x'], q)
    inst._run, inst.guess, inst.q = run, g, q
    inst._check = lambda i, k, o: quantile_check(i, k, o, q)
    return inst


@case('Quantile_T_Guess', ('fp32', None, {}), ('bf16', None, {'half': torch.bfloat16}))
def build_quantile_guess(ext, oracle, half=None):
    return build_quantile(ext, oracle, half=half, guess=True)


@case('Quantile_T_Half', ('fp16', None, {'half': torch.float16}), ('bf16', None, {'half': torch.bfloat16}))
def build_quantile_half(ext, oracle, half):
    return build_quantile(ext, oracle, half=half)


@case('Isotone_T')
def build_isotone(ext, oracle):
    inst = Inst({'x': select_sets(600000, 62, SEL_CAP)}, lambda b: ext.Isotone_T(b['x']), None)
    inst._check = lambda i, k, o: same(o[0].numpy(), i.want(k, lambda k: oracle.isotone_t(i.np['x'][k], 'device')), f'isotone set {k}')
    return inst


MQ_CAP = 4096
MQ_SIZES = [300007, 20001, 0, 70001]                              # an n = 0 row: its outputs and guess words stay as they are
MQ_SLOTS = [1, 3, 0, 2]


@case('Multi_Quantile_T', ('plain', None, {}), ('guess', None, {'guess': True}))
def build_multi_quantile(ext, oracle, guess=False, half=None):
    bank = {}
    for i, n in enumerate(MQ_SIZES):
        bank[f'x{i}'] = [dev(x, half) for x in select_sets(max(n, 16), 70 + i, MQ_CAP)]
    inst = Inst(bank, None, None)
    count, stride = len(MQ_SIZES), 3
    descs = table_descs(inst, MQ_SIZES, MQ_SLOTS)
    out = torch.empty(count * stride, device='cuda')
    ws = torch.empty(ext.Multi_Quantile_Workspace_Bytes(count, MQ_CAP), dtype=torch.uint8, device='cuda')
    g = ext.Quantile_Guess_Init(count, out) if guess else None
    torch.cuda.synchronize()

    def run(b):
        if half: ext.Multi_Quantile_T_Half(descs, max(MQ_SIZES), half, Q, out, stride, ws, MQ_CAP, g)
        else: ext.Multi_Quantile_T(descs, max(MQ_SIZES), Q, out, stride, ws, MQ_CAP, g)
        return out

    def check(inst, k, outs):
        o = outs[0].numpy().reshape(count, stride)
        for i, (n, s) in enumerate(zip(MQ_SIZES, MQ_SLOTS)):
            if n == 0:
                same(o[s], np.full(stride, SENT, F32), f'n = 0 row set {k}')
                continue
            x = inst.bank[f'x{i}'][k]
            want = inst.want((k, i), lambda _: sel_expected(x, list(oracle.quantile_ranks(n, Q))))
            same(o[s, :2], want, f'multi quantile row {i} set {k}')
            assert o[s, 2] == SENT, 'a store outside the slot'
    inst._run, inst._check, inst.poison_list, inst.keep, inst.guess = run, check, [(out, SENT)], (descs, ws), g
    return inst


@case('Multi_Quantile_T_Half', ('fp16', None, {'half': torch.float16}), ('bf16_guess', None, {'half': torch.bfloat16, 'guess': True}))
def build_multi_quantile_half(ext, oracle, half, guess=False):
    return build_multi_quantile(ext, oracle, guess, half)


@case('Quantile_Guess_Init')
def build_guess_init(ext, oracle):
    like = torch.empty(1, device='cuda')
    inst = Inst({'dummy': [F32([k]) for k in range(3)]}, lambda b: ext.Quantile_Guess_Init(5, like), None)
    inst._check = lambda i, k, o: same(o[0].numpy().view(np.uint32), np.array(INIT_GUESS * 5, np.uint32), 'guess words')
    return inst


# ------------------------------------------------------------------------------------------------------------------ scale searches
def ranges_sets():
    """(min, max) rows: ordinary, signed zeros, NaN and +-inf ranges, reversed and extreme; each set a permutation with new values."""
    rows = [(-1.5, 2.0), (0.0, 3.0), (-0.0, 0.0), (NAN, NAN), (-INF, INF), (-INF, 1.0), (-1.0, INF), (NAN, 1.0), (-1.0, NAN), (-3e38, 3e38),
            (2.0, 5.0), (-5.0, -2.0), (1e-30, 1e-30), (-1e-42, 1e-42)]
    r = np.random.RandomState(80)
    sets = []
    for k in range(5):
        p = r.permutation(len(rows))
        sets.append(np.array([(rows[j][0] * (1 + k), rows[j][1] * (1 + k)) for j in p], F32))
    return sets


@case('MinMax_To_Scale_Offset', *[(f'stride{st}_{"sym" if sym else "asym"}_pow2{int(p2)}', None, {'stride': st, 'sym': sym, 'pow2': p2})
                                  for st in (1, 2) for sym in (True, False) for p2 in (False, True)])
def build_mm2so(ext, oracle, stride, sym, pow2):
    qmin, qmax = (-128, 127) if sym else (0, 255)
    inst = Inst({'mm': ranges_sets()}, None, None)

    def run(b):
        mm = b['mm']
        if stride == 1: return ext.MinMax_To_Scale_Offset(mm[:, 0].contiguous(), mm[:, 1].contiguous(), 1, qmin, qmax, sym, pow2, 1e-8)
        return ext.MinMax_To_Scale_Offset(mm.view(-1), mm.view(-1)[1:], 2, qmin, qmax, sym, pow2, 1e-8)

    def check(inst, k, outs):
        want = [oracle.minmax_to_scale_offset(float(a), float(b), qmin, qmax, sym, pow2, 1e-8, ieee=True) for a, b in inst.np['mm'][k]]
        same(outs[0].numpy(), np.array([w[0] for w in want], F32), f'scale set {k}', False)
        same(outs[1].numpy(), np.array([w[1] for w in want], F32), f'offset set {k}', False)
    inst._run, inst._check = run, check
    return inst


@case('Hist_Scale_From_MinMax', ('sym', None, {'sym': True}), ('asym', None, {'sym': False}))
def build_hist_scale(ext, oracle, sym):
    inst = Inst({'mm': ranges_sets()}, lambda b: ext.Hist_Scale_From_MinMax(b['mm'], sym, 4096), None)

    def check(inst, k, outs):
        want = [(builtins.max(abs(float(b)), abs(float(a))) if sym else float(b) - float(a)) / 4096 for a, b in inst.np['mm'][k]]
        same(outs[0].numpy(), np.array(want, F32), f'hist scale set {k}', False)
    inst._check = check
    return inst


def kl_hists(bins, seed, K=5, rows=3, sparse=False):
    """Histogram tables whose best candidate moves from set to set; `sparse`: mostly empty bins (empty merged groups: NaN candidates)."""
    r = np.random.RandomState(seed)
    sets = []
    for k in range(K):
        hs = []
        for j in range(rows):
            decay = bins / (1.0 + 3.0 * ((k + j) % 5))
            h = r.gamma(0.6 + 0.3 * j, 40.0, size=bins) * np.exp(-np.arange(bins) / decay)
            if sparse: h[r.rand(bins) < 0.9] = 0
            if (k + j) % 3 == 1: h[bins // (2 + k):] = 0
            hs.append(np.floor(h).astype(np.int32))
        sets.append(np.stack(hs))
    return sets


@case('KL_Search', *[(f'k{v}_{b}bit', ('kl_search', v), {'bits': b}) for v in (0, 1) for b in (8, 2)])
def build_kl(ext, oracle, bits):
    bins = 2048 if bits == 8 else 256
    hists = kl_hists(bins, 90 + bits, sparse=bits == 2)
    hss = [F32([[1e-3, 0.5, 2.0 ** -40][(k + j) % 3] for j in range(3)]) for k in range(5)]
    inst = Inst({'h': hists, 'hs': hss}, lambda b: ext.KL_Search(b['h'], bins, b['hs'], None, bits, False, 1e-8), None)
    qb = 2 ** (bits - 1)

    def check(inst, k, outs):
        scale, best = outs[0].numpy(), outs[1].numpy()
        ref = inst.want(k, lambda k: [oracle.kl_search(h, 1.0, bits, return_losses=True) for h in inst.np['h'][k]])
        for j, (_, _, wb, losses) in enumerate(ref):
            got = int(best[j])
            if got != wb:                                         # DESIGN.md §2 deviation 2: the argmin moves only on a numerical tie
                lg, lw = losses[got // qb - 1], losses[wb // qb - 1]
                assert (np.isnan(lg) and np.isnan(lw)) or abs(lg - lw) <= 1e-12 * builtins.max(1.0, abs(lw)), (k, j, got, wb, lg, lw)
                continue
            same(scale[j:j + 1], [oracle.kl_scale(wb, bins, float(inst.np['hs'][k][j]), bits, False, 1e-8)], f'KL row {j} set {k}', False)
    inst._check = check
    return inst


@case('MSE_Search', ('asym', None, {'sym': False}), ('sym', None, {'sym': True}))
def build_mse(ext, oracle, sym):
    bins, interval = 2048, 8
    qmin, qmax = (-128, 127) if sym else (0, 255)
    r = np.random.RandomState(100)
    base = [(r.gamma(0.6, 300.0, size=bins) * (r.rand(bins) > 0.3)).astype(np.int32), np.full(bins, 7, np.int32)]
    # vmin below, at and above 0 (different start counts), moving between rows from set to set; a flat histogram (ties)
    mmrows = [(-0.02, 3.0), (0.0, 3.0), (0.4, 3.0), (-2.0, 1.5)] if sym else [(-0.02, 3.0), (0.0, 3.0), (0.4, 3.0), (-0.05, 1.5)]
    hists, mms = [], []
    for k in range(5):
        hists.append(np.stack([base[(k + j) % 2] for j in range(3)]))
        mms.append(np.array([mmrows[(k + j) % 4] for j in range(3)], F32))
    inst = Inst({'h': hists, 'mm': mms}, lambda b: ext.MSE_Search(b['h'], bins, b['mm'], qmin, qmax, sym, False, 1e-8, interval), None)
    losses = {}

    def loss_of(h):
        def loss(_h, start, step, end):
            key = (h.tobytes(), start, step, end)
            if key not in losses: losses[key] = oracle.compute_mse_loss(np.ascontiguousarray(h, np.int64), start, step, end)
            return losses[key]
        return loss

    def check(inst, k, outs):
        want = []
        for j in range(3):
            lo32, hi32 = float(inst.np['mm'][k][j][0]), float(inst.np['mm'][k][j][1])
            hs = (builtins.max(abs(hi32), abs(lo32)) if sym else (hi32 - lo32)) / bins
            h = inst.np['h'][k][j]
            want.append(oracle.mse_search(h, hs, lo32, qmin, qmax, sym, False, interval, loss_of(h), 1e-8))
        same(outs[0].numpy(), np.array([w[0] for w in want], F32), f'MSE scale set {k}', False)
        same(outs[1].numpy(), np.array([w[1] for w in want], F32), f'MSE offset set {k}', False)
    inst._check = check
    return inst


# ------------------------------------------------------------------------------------------------------------------ training kernels
def train_sets(shape, seed, K=4):
    r = np.random.RandomState(seed)
    xs, dys = [], []
    for k in range(K):
        s = [0.05, 0.37, 3.1e-3, 17.0][k]
        x = (r.uniform(-140, 140, int(np.prod(shape))) * s).astype(F32)
        x[r.choice(x.size, 4, replace=False)] = (np.array([127.5, -128.5, 3.5, 0.0]) * s).astype(F32)
        xs.append(x.reshape(shape)); dys.append(r.standard_normal(int(np.prod(shape))).astype(F32).reshape(shape))
    return xs, dys


def train_params(C, K=4, floating=False):
    sc = [np.full(C, [0.05, 0.37, 3.1e-3, 17.0][k], F32) * np.linspace(1, 2, C, dtype=F32) for k in range(K)]
    of = [np.zeros(C, F32) if floating else np.array([[0.0, 3.0, -5.0, 0.5][(k + c) % 4] for c in range(C)], F32) for k in range(K)]
    return sc, of


@case('QuantizeTensor_LT_B', ('T', None, {'axis': None}))
def build_lsq(ext, oracle, axis, floating=False):
    import test_gpu_training_kernels as tk
    shape = (6, 8, 512)
    xs, dys = train_sets(shape, 110)
    C = 1 if axis is None else shape[axis]
    sc, of = train_params(C, floating=floating)
    inst = Inst({'x': xs, 'dy': dys, 's': sc, 'o': of}, None, None, exact=False)
    E, M, cmin, cmax = FP8
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def run(b):
        if floating:
            if axis is None: return ext.QuantizeTensor_FT_B(b['x'], b['s'], b['o'], b['dy'], E, M, cmin, cmax, 0)
            return ext.QuantizeTensor_FC_B(b['x'], b['s'], b['o'], b['dy'], E, M, cmin, cmax, 0, axis)
        if axis is None: return ext.QuantizeTensor_LT_B(b['x'], b['s'], b['o'], b['dy'], QMIN, QMAX, 0)
        return ext.QuantizeTensor_LC_B(b['x'], b['s'], b['o'], b['dy'], QMIN, QMAX, 0, axis)

    def check(inst, k, outs):
        x, dy, s, o = inst.np['x'][k], inst.np['dy'][k], inst.np['s'][k], inst.np['o'][k]
        if floating: wx, p, f = oracle.float_quant_backward(x, dy, s, o, E, M, cmin, cmax, 0, axis)
        else: wx, p, f = oracle.linear_quant_backward(x, dy, s, o, QMIN, QMAX, 0, axis)
        same(outs[0].numpy(), wx, f'grad_x set {k}')
        if axis is None:
            epc = tk.rows_of(x.size)
            groups, kk = [p.reshape(-1)], tk.chain_rows(epc, x.size // epc)
        else:
            epc, Cc = oracle.channel_geometry(x.shape, axis)
            ch = (np.arange(x.size) // epc) % Cc
            groups, kk = [p.reshape(-1)[ch == c] for c in range(Cc)], tk.chain_rows(epc, x.size // (epc * Cc))
        tk.check_sum(outs[1], groups, f, floating, kk, False, f'grad_s set {k}')
    inst._run, inst._check = run, check
    return inst


@case('QuantizeTensor_LC_B', ('C', None, {'axis': 1}))
def build_lsq_c(ext, oracle, axis):
    return build_lsq(ext, oracle, axis)


@case('QuantizeTensor_FT_B')
def build_fb_t(ext, oracle):
    return build_lsq(ext, oracle, None, floating=True)


@case('QuantizeTensor_FC_B')
def build_fb_c(ext, oracle):
    return build_lsq(ext, oracle, 1, floating=True)


@case('TensorClip_T', ('T', None, {'axis': None}))
def build_clip(ext, oracle, axis):
    shape = (6, 8, 513)
    r = np.random.RandomState(120)
    vs = [r.standard_normal(shape).astype(F32) * (k + 1) for k in range(4)]
    refs = [r.standard_normal(shape).astype(F32) for _ in range(4)]
    C = 1 if axis is None else shape[axis]
    lims = [r.rand(C).astype(F32) * (k + 0.5) for k in range(4)]
    inst = Inst({'v': vs, 'r': refs, 'l': lims}, None, None)

    def run(b):
        return ext.TensorClip_T(b['v'], b['r'], b['l']) if axis is None else ext.TensorClip_C(b['v'], b['r'], b['l'], axis)
    inst._run = run
    inst._check = lambda i, k, o: same(o[0].numpy(), oracle.tensor_clip(i.np['v'][k], i.np['r'][k], i.np['l'][k], axis), f'clip set {k}')
    return inst


@case('TensorClip_C', ('C', None, {'axis': 1}))
def build_clip_c(ext, oracle, axis):
    return build_clip(ext, oracle, axis)


@case('RoundingLoss_LT', ('T', None, {'axis': None}))
def build_rl(ext, oracle, axis, backward=False):
    import test_gpu_training_kernels as tk
    shape = (6, 8, 512)
    xs, _ = train_sets(shape, 130)
    C = 1 if axis is None else shape[axis]
    sc, of = train_params(C)
    dys = [F32([[1.0, -0.5, 3.0, 0.25][k]]) for k in range(4)]
    inst = Inst({'x': xs, 's': sc, 'o': of, 'dy': dys}, None, None, exact=backward)
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def run(b):
        if backward:
            if axis is None: return ext.RoundingLoss_LT_B(b['x'], b['dy'], b['s'], b['o'], QMIN, QMAX, 0)
            return ext.RoundingLoss_LC_B(b['x'], b['dy'], b['s'], b['o'], QMIN, QMAX, axis, 0)
        if axis is None: return ext.RoundingLoss_LT(b['x'], b['s'], b['o'], QMIN, QMAX, 0)
        return ext.RoundingLoss_LC(b['x'], b['s'], b['o'], QMIN, QMAX, axis, 0)

    def check(inst, k, outs):
        x, s, o = inst.np['x'][k], inst.np['s'][k], inst.np['o'][k]
        if backward:
            same(outs[0].numpy(), oracle.rounding_loss_backward(x, inst.np['dy'][k], s, o, QMIN, QMAX, 0, axis), f'RL grad set {k}')
            return
        p, d = oracle.rounding_loss(x, s, o, QMIN, QMAX, 0, axis)
        tk.check_sum(outs[0], [p.reshape(-1)], d, True, tk.chain_flat(x.size, sms), False, f'RL loss set {k}')
    inst._run, inst._check = run, check
    return inst


@case('RoundingLoss_LC', ('C', None, {'axis': 1}))
def build_rl_c(ext, oracle, axis):
    return build_rl(ext, oracle, axis)


@case('RoundingLoss_LT_B', ('T', None, {'axis': None}))
def build_rlb(ext, oracle, axis):
    return build_rl(ext, oracle, axis, backward=True)


@case('RoundingLoss_LC_B', ('C', None, {'axis': 1}))
def build_rlb_c(ext, oracle, axis):
    return build_rl(ext, oracle, axis, backward=True)


# ------------------------------------------------------------------------------------------------------------------ paired moments
@case('Multi_Paired_Moments', ('fp32', None, {'dtype': torch.float32}), ('fp16', None, {'dtype': torch.float16}),
      ('bf16', None, {'dtype': torch.bfloat16}))
def build_moments(ext, oracle, dtype):
    import layerwise_oracle as lo
    shapes = [(8, 70001), (32, 1000), (4, 3)]
    r = np.random.RandomState(140)
    bank = {}
    for i, sh in enumerate(shapes):
        ps, rs = [], []
        for k in range(4):
            p = (r.standard_normal(sh) * [1, 1e3, 1e-3, 1][k]).astype(F32)
            if k == 3: p = specials(r, p, 5).reshape(sh)
            ps.append(dev(p, dtype)); rs.append(dev((p + r.standard_normal(sh) * 0.01).astype(F32), dtype))
        bank[f'p{i}'], bank[f'r{i}'] = ps, rs
    inst = Inst(bank, None, None)
    rows, row0 = [], 0
    for i, sh in enumerate(shapes):
        rows.append([inst.buf[f'p{i}'].data_ptr(), inst.buf[f'r{i}'].data_ptr(), sh[0], sh[1], row0]); row0 += sh[0]
    descs = torch.tensor(rows, dtype=torch.int64, device='cuda')
    elems = sum(int(np.prod(s)) for s in shapes)
    out = torch.empty(row0, 4, dtype=torch.float64, device='cuda')
    ws = torch.empty(ext.Multi_Paired_Moments_Workspace_Bytes(row0, elems), dtype=torch.uint8, device='cuda')

    def run(b):
        ext.Multi_Paired_Moments(descs, elems, dtype, out, ws)
        return out

    def check(inst, k, outs):
        got, at = outs[0].numpy(), 0
        for i, sh in enumerate(shapes):
            p, rr = inst.bank[f'p{i}'][k], inst.bank[f'r{i}'][k]
            want, bound = lo.exact_moments(p, rr), lo.moments_bound(p, rr)
            assert lo.moments_agree(got[at:at + sh[0]], want, bound), (k, i, got[at:at + sh[0]][:2], want[:2])
            at += sh[0]
    inst._run, inst._check, inst.poison_list, inst.keep = run, check, [(out, NAN)], (descs, ws)
    return inst


# ------------------------------------------------------------------------------------------------------------------ fixtures and tests
@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


@pytest.fixture(scope='module')
def gate_cycles():
    """torch.cuda._sleep cycles for ~GATE_MS milliseconds, measured once with CUDA events."""
    torch.cuda._sleep(1000)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    probe = 20_000_000
    a.record(); torch.cuda._sleep(probe); b.record(); b.synchronize()
    return int(probe * GATE_MS / a.elapsed_time(b))


def build(ext, oracle, name, label):
    fn, kn, params = CASES[name][label]
    inst = fn(ext, oracle, **params)
    inst.oracle = oracle
    torch.cuda.synchronize()
    return inst, kn


@pytest.mark.parametrize('name,label', case_ids(), ids=[f'{n}-{lab}' for n, lab in case_ids()])
def test_side_stream_gate(ext, oracle, gate_cycles, name, label):
    inst, kn = build(ext, oracle, name, label)
    with knob(ext, kn):
        inst.load(0); pins = pinned_like(inst.run()); torch.cuda.synchronize()     # first launches load their modules outside the gate
        for gate_on_default, k in ((False, 1), (True, 2 % inst.K)):
            inst.load((k + 1) % inst.K); inst.poison(); torch.cuda.synchronize()
            s = torch.cuda.Stream()
            gc.disable()                                             # no collector pause inside the gated window
            try:
                with torch.cuda.stream(torch.cuda.current_stream() if gate_on_default else s):
                    torch.cuda._sleep(gate_cycles)
                    gate = torch.cuda.Event(); gate.record()
                with torch.cuda.stream(s):
                    inst.load(k)
                    outs = inst.run()
                assert not gate.query(), f'{name}: the call waited for the device'
                got = readback(outs, s, pins)
                if gate_on_default:
                    assert not gate.query(), 'the gate ended before the results were read: lengthen GATE_MS'
            finally:
                gc.enable()
            torch.cuda.synchronize()
            inst.check(k, got)


@pytest.mark.parametrize('name,label', case_ids(), ids=[f'{n}-{lab}' for n, lab in case_ids()])
def test_graph_replay_with_fresh_data(ext, oracle, name, label):
    inst, kn = build(ext, oracle, name, label)
    with knob(ext, kn):
        inst.load(0); torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            inst.run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = inst.run()
        first = None
        for k in [0] + list(range(1, inst.K)) + [0]:
            inst.load(k); inst.poison()
            graph.replay()
            torch.cuda.synchronize()
            got = [o.cpu() for o in outs]
            inst.check(k, got)
            if k == 0 and first is None:
                first = got
            elif k == 0 and inst.exact:
                for a, b in zip(first, got):
                    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f'{name}: replay of set 0 is not bit-identical'
        del graph


GUESS_SEQ = [0, 1, 2, 2, 4, 4]     # first call, hit, miss, hit (the same set again: its thresholds hold), heavy tail, hit


@pytest.mark.parametrize('name', ['Quantile_T_Guess', 'Multi_Quantile_T'])
def test_guess_words_carried_across_replays(ext, oracle, name):
    label = 'fp32' if name == 'Quantile_T_Guess' else 'guess'
    eager, _ = build(ext, oracle, name, label)
    seq = GUESS_SEQ
    init = eager.guess.clone()
    for k in seq:
        eager.load(k); eager.poison()
        out = eager.run()
        torch.cuda.synchronize()
        eager.check(k, [o.cpu() for o in out])
    words_eager = eager.guess.clone()

    inst, _ = build(ext, oracle, name, label)
    inst.load(0); torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        inst.run()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = inst.run()
    inst.guess.copy_(init)                                        # start from the init words, as the eager sequence did
    for k in seq:
        inst.load(k); inst.poison()
        graph.replay()
        torch.cuda.synchronize()
        inst.check(k, [o.cpu() for o in outs])
    assert torch.equal(inst.guess, words_eager), 'guess words after the replayed sequence differ from the eager sequence'
    assert not torch.equal(words_eager, init)


# ------------------------------------------------------------------------------------------------------------------ driver flows on a side stream
def flow_net(dtype=torch.float32):
    import netspec
    from ppq_b200.executor import TorchExecutor
    spec = netspec.SPECS['tinyres']
    model = netspec.SpecNet(spec, netspec.make_params(spec, 3)).cuda().to(dtype)
    data = [torch.from_numpy(x).cuda().to(dtype) for x in netspec.make_data('tinyres', 4, 8, 4)]
    ex = TorchExecutor(model, data[0], fuse_bn=False)
    ex.quantize_parameters()
    torch.cuda.synchronize()
    return ex, data


def config_bits(ex):
    """Every config's state, scale and offset bits, and every weight, in executor order."""
    def b(t):
        return None if t is None else t.detach().reshape(-1).cpu().view(torch.int16 if t.element_size() == 2 else torch.int32)
    rows = []
    for n, op in ex.quantable_operations():
        for c in ex._configs_of(op): rows.append((n, str(c.state), b(c._scale), b(c._offset)))
        if op.weight_cfg is not None: rows.append((n, b(op.module.weight.data)))
    return rows


def same_rows(a, b, what):
    assert len(a) == len(b), what
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert (u is None and v is None) or (isinstance(u, str) and u == v) or torch.equal(u, v), (what, x[0])


def on_side_stream(fn, gate_cycles):
    """fn() on a fresh side stream while the default stream sleeps ~GATE_MS: work the flow queues on the default stream runs late, so
    whatever the flow reads back on its own stream would be stale."""
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    torch.cuda._sleep(gate_cycles)
    with torch.cuda.stream(side):
        out = fn()
    torch.cuda.synchronize()
    return out


FLOWS = [(m, d, None, False) for m in ('minmax', 'kl', 'mse', 'percentile') for d in (True, False, 'auto')] + \
        [('kl', 'auto', 'ring', False), ('percentile', 'auto', 'ring', False), ('kl', 'auto', None, True), ('percentile', False, None, True)]


@pytest.mark.parametrize('method,deferred,to_device,half', FLOWS)
def test_calibrate_arena_on_a_side_stream(ext, gate_cycles, method, deferred, to_device, half):
    from ppq_b200.executor import calibrate_arena
    dtype = torch.bfloat16 if half else torch.float32

    def run(ex, data):
        batches = [d.cpu().pin_memory() for d in data] if to_device == 'ring' else data
        calibrate_arena(ex, batches, method=method, deferred=deferred, to_device=to_device, half_inputs=half)
    ex0, data0 = flow_net(dtype)
    run(ex0, data0); torch.cuda.synchronize()
    ex1, data1 = flow_net(dtype)
    on_side_stream(lambda: run(ex1, data1), gate_cycles)
    same_rows(config_bits(ex1), config_bits(ex0), f'calibrate_arena {method} deferred={deferred} {to_device} half={half}')


@pytest.mark.parametrize('method', ['minmax', 'kl', 'mse', 'percentile'])
def test_runtime_calibration_pass_on_a_side_stream(ext, gate_cycles, method):
    from ppq_b200.calibration import RuntimeCalibrationPass

    def run(ex, data):
        RuntimeCalibrationPass(method=method).optimize(graph=ex, dataloader=data, executor=ex, calib_steps=8)
    ex0, data0 = flow_net()
    run(ex0, data0); torch.cuda.synchronize()
    ex1, data1 = flow_net()
    on_side_stream(lambda: run(ex1, data1), gate_cycles)
    same_rows(config_bits(ex1), config_bits(ex0), f'RuntimeCalibrationPass {method}')


def test_error_analyses_on_a_side_stream(ext, gate_cycles):
    from ppq_b200.executor import calibrate_arena, graphwise_error_analyse, layerwise_error_analyse
    ex, data = flow_net()
    calibrate_arena(ex, data, method='kl')
    ex.align_quantization(); ex.bake_parameters()
    torch.cuda.synchronize()
    before = config_bits(ex)
    for graphs in (False, True):
        want = graphwise_error_analyse(ex, data[:3], graphs=graphs)
        got = on_side_stream(lambda: graphwise_error_analyse(ex, data[:3], graphs=graphs), gate_cycles)
        assert list(got) == list(want) and all(np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes() for k in want), (graphs, got, want)
    want = layerwise_error_analyse(ex, data, steps=2)
    got = on_side_stream(lambda: layerwise_error_analyse(ex, data, steps=2), gate_cycles)
    assert list(got) == list(want) and all(np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes() for k in want), (got, want)
    same_rows(config_bits(ex), before, 'configs after the analyses')
