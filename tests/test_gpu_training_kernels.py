"""The ten training-pass entry points (QuantizeTensor_LT_B / _LC_B, QuantizeTensor_FT_B / _FC_B, TensorClip_T / _C, RoundingLoss_LT /
_LC / _LT_B / _LC_B) against the oracle's scalar restatements (oracle/ppq_oracle.c), across every rounding policy and an unknown id,
4-bit, 8-bit and full int32 ranges, integer, half-integer and fractional offsets, six float formats with clip bounds on, off and beyond
the format's grid, special values in the input and in dy, and the launch geometries of train.cu.

Element-wise outputs must equal the oracle bit for bit.  The scalar reductions (grad_s, loss) are fp32 sums whose order the launch
decides, so they are held to |got - exact| <= (k + 1) * 2^-24 * sum|p_i| * |factor|: exact is the fp64 sum of the oracle's fp32
partials, k the longest addition chain the launch can form (elements per thread + 8 tree levels + the block sums that reach one
output), and the + 1 the scaling of each block sum.  Where every partial and every prefix sum is exact in fp32 and each block sum is
scaled exactly (a power-of-two normaliser, or one block sum per output), the result must be bit-exact: these cases see a wrong
partial whatever the summation order."""
import math

import numpy as np
import pytest
import torch

import refcuda

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0 ** -24
IMIN, IMAX = -2 ** 31, 2 ** 31 - 1
MODES = list(range(8)) + [11]                                  # 11: an unknown id, which rounds half away from zero
RANGES = [(0, 255), (-128, 127), (-8, 7), (0, 15), (IMIN, IMAX)]
OFFSETS = [0.0, 3.0, -5.0, 0.5, -0.5, 2.5, 3.5, 1.3]
# (E, M, a clip bound on the grid): E4M3 at 448 and 240, E5M2, E3M4, E2M1, E5M10
FORMATS = [(4, 3, 448.0), (4, 3, 240.0), (5, 2, 57344.0), (3, 4, 30.0), (2, 1, 6.0), (5, 10, 65504.0)]
TPB = 256
REF_K = 64                                                   # the reference's own reduction: 1024-thread trees, one atomic per block


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


@pytest.fixture(scope='module')
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture
def ref(request):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return refcuda.reference(request.node.nodeid)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).cuda()


def host(t):
    return t.detach().cpu().numpy()


def assert_same(got, want, what):
    """Bit-identical, except that any NaN matches any NaN (the device's canonical NaN is not x86's)."""
    g, w = np.asarray(host(got) if isinstance(got, torch.Tensor) else got, F32).reshape(-1), np.asarray(want, F32).reshape(-1)
    assert g.shape == w.shape, what
    bad = (g.view(np.int32) != w.view(np.int32)) & ~(np.isnan(g) & np.isnan(w))
    assert not bad.any(), (what, int(bad.sum()), np.flatnonzero(bad)[:5], g[bad][:5], w[bad][:5])


# ---- launch geometry of train.cu: the longest chain of fp32 additions behind one output ------------------------------------------
def rows_of(n):
    """Per-tensor backward rows: 8192 ... 256 elements when n is a multiple, else the whole tensor on one CTA (train.cu)."""
    for cand in (8192, 4096, 2048, 1024, 512, 256):
        if n % cand == 0:
            return cand
    return n


def chain_rows(epc, rows_per_output):
    return -(-epc // TPB) + 8 + rows_per_output


def chain_flat(n, sms):
    grid = max(1, min(-(-n // (TPB * 8)), sms * 8))
    return -(-n // (grid * TPB)) + 8 + grid


def check_sum(got, partials, scale, divide, k, exact, what):
    """got: the kernel's fp32 outputs, one per slot; partials: the oracle's fp32 terms of each slot."""
    got = np.asarray(host(got), F32).reshape(-1)
    assert len(got) == len(partials), what
    for c, (g, p) in enumerate(zip(got, partials)):
        p64 = np.asarray(p, np.float64)
        e = p64.sum()
        want = e / float(scale) if divide else e * float(scale)
        if not np.isfinite(want) or not np.isfinite(e):
            assert np.isnan(g) if np.isnan(want) else g == want, (what, c, g, want)
            continue
        if exact:
            assert g == F32(want), (what, c, float(g), float(F32(want)))
            continue
        mag = np.abs(p64).sum() / float(scale) if divide else np.abs(p64).sum() * abs(float(scale))
        assert abs(float(g) - want) <= (k + 1) * U * mag * 1.0001 + 1e-45, (what, c, float(g), want, k, mag)


def exactly_summable(partials):
    """Every partial a multiple of a common power of two (the lowest set bit among them), and the sum of their magnitudes below
    2^24 such units: every partial sum, in any order, is then exact in fp32."""
    p = np.asarray(partials, np.float64).reshape(-1)
    if not np.isfinite(p).all():
        return False
    nz = p[p != 0]
    if nz.size == 0:
        return True
    m, e = np.frexp(nz)
    mi = np.abs(np.ldexp(m, 53)).astype(np.int64)
    unit = np.ldexp((mi & -mi).astype(np.float64), e - 53).min()
    return np.abs(nz).sum() / unit < 2.0 ** 24


# ---- inputs ------------------------------------------------------------------------------------------------------------------------
def int_quotients(r, n, qmin, qmax, o):
    """x / s values: uniform over the range and a margin, exact ties k + 1/2 and their fp32 neighbours, the clip boundaries
    (qmax - o) +- 1/2 and +- one ulp, quotients that saturate the int32 conversion."""
    lo, hi = max(float(qmin) - o, -3e9), min(float(qmax) - o, 3e9)
    t = r.uniform(lo - 3, hi + 3, n)
    m = max(1, n // 8)
    ties = (np.floor(r.uniform(lo - 2, hi + 2, m)) + 0.5).astype(F32)
    t[:m] = ties
    if n >= 3 * m:
        t[m:2 * m], t[2 * m:3 * m] = np.nextafter(ties, F32(np.inf)), np.nextafter(ties, F32(-np.inf))
    edges = []
    for b in (hi, lo, hi + 0.5, lo - 0.5):
        fb = F32(b)
        edges += [fb, np.nextafter(fb, F32(np.inf)), np.nextafter(fb, F32(-np.inf))]
    edges += [3e12, -3e12]
    k = min(len(edges), n)
    idx = r.choice(n, k, replace=False)
    t[idx] = edges[:k]
    return t.astype(F32)


def with_specials(r, x):
    x = x.copy()
    sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan], F32)
    k = min(len(sp), x.size)
    x.reshape(-1)[r.choice(x.size, k, replace=False)] = sp[:k]
    return x


def fp_quotients(r, n, E, M, cmax):
    """x / s values for FP(E, M): log-uniform magnitudes from below the smallest sub-normal to beyond the clip, grid ties, the
    clip bound, cmax + 1 and the points between."""
    k = (1 << (E - 1)) + M - 2
    mags = np.exp2(r.uniform(-k - 2, math.log2(cmax) + 1.5, n))
    t = mags * np.where(r.rand(n) < 0.5, -1.0, 1.0)
    m = max(1, n // 6)
    # ties on the normal grid: a value with M mantissa bits plus one half-ulp bit
    e = np.floor(r.uniform(-k + M, math.log2(cmax), m))
    mant = np.floor(r.uniform(0, 2 ** M, m))
    t[:m] = np.exp2(e) * (1 + (mant + 0.5) / 2 ** M) * np.where(r.rand(m) < 0.5, -1, 1)
    t[m:2 * m] = np.floor(r.uniform(-8, 8, m)) * 2.0 ** -k + 2.0 ** -(k + 1)      # sub-normal ties
    edges = [cmax, cmax + 0.5, cmax + 1, cmax + 1.5, cmax + 2, np.nextafter(F32(cmax + 1), F32(np.inf)), -cmax, -cmax - 1, -cmax - 1.5]
    j = min(len(edges), n)
    t[r.choice(n, j, replace=False)] = edges[:j]
    return t.astype(F32)


# ---- LSQ backward ------------------------------------------------------------------------------------------------------------------
def run_lsq(ext, oracle, sms, x, dy, s, o, qmin, qmax, mode, axis, what, exact=False, call=None):
    if axis is None:
        gx, gs = (call or ext.QuantizeTensor_LT_B)(dev(x), dev(s), dev(o), dev(dy), qmin, qmax, mode)
        wx, p, f = oracle.linear_quant_backward(x, dy, s, o, qmin, qmax, mode)
        epc = rows_of(x.size)
        groups, k = [p.reshape(-1)], chain_rows(epc, x.size // epc)
    else:
        gx, gs = (call or ext.QuantizeTensor_LC_B)(dev(x), dev(s), dev(o), dev(dy), qmin, qmax, mode, axis)
        wx, p, f = oracle.linear_quant_backward(x, dy, s, o, qmin, qmax, mode, axis)
        epc, C = oracle.channel_geometry(x.shape, axis)
        ch = (np.arange(x.size) // epc) % C
        groups, k = [p.reshape(-1)[ch == c] for c in range(C)], chain_rows(epc, x.size // (epc * C))
    assert_same(gx, wx, what + ' grad_x')
    check_sum(gs, groups, f, False, k, exact, what + ' grad_s')
    return gx, gs


@pytest.mark.parametrize('qmin,qmax', RANGES)
def test_lsq_backward_modes_offsets(ext, oracle, sms, qmin, qmax):
    r = np.random.RandomState(qmax & 0xffff)
    for mode in MODES:
        for off in OFFSETS:
            s = F32(r.choice([0.25, 0.37, 3.1e-3, 17.0]))
            x = (int_quotients(r, 768, qmin, qmax, round(off)) * s).astype(F32)
            dy = r.randn(768).astype(F32)
            run_lsq(ext, oracle, sms, x, dy, [s], [off], qmin, qmax, mode, None, f'LT {qmin}..{qmax} mode {mode} o {off}')
            xc, dyc = x.reshape(4, 3, 64), dy.reshape(4, 3, 64)
            sc = np.array([s, s * 2, 0.11], F32); oc = np.array([off, -off, 2.5], F32)
            run_lsq(ext, oracle, sms, xc, dyc, sc, oc, qmin, qmax, mode, 1, f'LC {qmin}..{qmax} mode {mode} o {off}')
        x = with_specials(r, (int_quotients(r, 300, qmin, qmax, 0) * F32(0.5)).astype(F32))
        dy = with_specials(r, r.randn(300).astype(F32))
        run_lsq(ext, oracle, sms, x, dy, [0.5], [0.0], qmin, qmax, mode, None, f'LT specials mode {mode}')
        run_lsq(ext, oracle, sms, x.reshape(3, 100), dy.reshape(3, 100), [0.5, 1e-30, 3e30], [1.0, 0.5, -2.5], qmin, qmax, mode, 0,
                f'LC specials mode {mode}')


LSQ_SHAPES = [([1], None), ([255], None), ([256], None), ([768], None), ([8192 * 3], None), ([10007], None), ([(1 << 24) + 3], None),
              ([8, 16, 5, 5], 0), ([4, 16, 7, 7], 1), ([2, 9, 300], -1), ([6, 2, 4, 3], 3), ([64, 1], 0), ([3, 1, 5], 1), ([513, 7], 1)]


@pytest.mark.parametrize('shape,axis', LSQ_SHAPES)
def test_lsq_backward_geometry(ext, oracle, sms, shape, axis):
    r = np.random.RandomState(len(shape) + sum(shape) % 97)
    n = int(np.prod(shape))
    mode = int(r.choice(MODES))
    C = 1 if axis is None else shape[axis]
    s = (r.rand(C) * 0.1 + 0.02).astype(F32)
    o = r.choice([0.0, 2.5, -3.0, 0.5], C).astype(F32)
    x = (int_quotients(r, n, -128, 127, 0).reshape(shape) * s.max()).astype(F32)
    dy = r.randn(*shape).astype(F32)
    run_lsq(ext, oracle, sms, x, dy, s, o, -128, 127, mode, axis, f'{shape} axis {axis} mode {mode}')


def test_lsq_backward_layouts(ext, oracle, sms):
    """[1, C, 1, 1] scale views, transposed value and dy, a negative axis: the binding makes them dense in the reference's order."""
    r = np.random.RandomState(11)
    x = (int_quotients(r, 2 * 8 * 6 * 5, 0, 255, 3) * F32(0.1)).reshape(2, 8, 6, 5).astype(F32)
    dy = r.randn(2, 8, 6, 5).astype(F32)
    s = (r.rand(8) * 0.1 + 0.05).astype(F32); o = np.array([3, 2.5, 0.5, -1, 3.5, 0, 7, 1.3], F32)
    tx, tdy = dev(x), dev(dy)
    for view, axis in (((1, 8, 1, 1), 1), ((8,), -3)):
        gx, gs = ext.QuantizeTensor_LC_B(tx, dev(s).view(view), dev(o).view(view), tdy, 0, 255, 4, axis)
        wx, p, f = oracle.linear_quant_backward(x, dy, s, o, 0, 255, 4, 1)
        assert_same(gx, wx, f'view {view}')
        check_sum(gs, [p[:, c].reshape(-1) for c in range(8)], f, False, chain_rows(30, 2), False, f'view {view}')
    xt, dyt = tx.transpose(1, 3), tdy.transpose(1, 3)                  # non-contiguous [2, 5, 6, 8], channel axis 3
    gx, gs = ext.QuantizeTensor_LC_B(xt, dev(s), dev(o), dyt, 0, 255, 6, 3)
    xn, dyn = host(xt.contiguous()), host(dyt.contiguous())
    wx, p, f = oracle.linear_quant_backward(xn, dyn, s, o, 0, 255, 6, 3)
    assert_same(gx, wx, 'transposed LC')
    check_sum(gs, [p[..., c].reshape(-1) for c in range(8)], f, False, chain_rows(1, 60), False, 'transposed LC')
    gx, gs = ext.QuantizeTensor_LT_B(xt, dev(s[:1]), dev(o[:1]), dyt, 0, 255, 1)
    wx, p, f = oracle.linear_quant_backward(xn, dyn, s[:1], o[:1], 0, 255, 1)
    assert_same(gx, wx, 'transposed LT')
    check_sum(gs, [p.reshape(-1)], f, False, chain_rows(x.size, 1), False, 'transposed LT')


def dyadic_quotients(r, n, lo, hi):
    """x / s as multiples of 1/8 inside and around [lo, hi]: every LSQ partial is a multiple of dy / 8."""
    return (np.floor(r.uniform(lo - 2, hi + 2, n) * 8) / 8).astype(F32)


@pytest.mark.parametrize('n,qmin,qmax,axis_shape', [
    (1, 0, 255, None), (200, -8, 7, None), (256, 0, 15, None),                      # one CTA: any normaliser
    (4096, -8, 8, None), (16384, 0, 4, None), (1 << 16, -32, 32, None),             # n * (qmax - qmin) a power of 4
    (4096, -16, 16, (4, 16, 64)), (1024, -4, 4, (1024,)), (65536, 0, 16, (16, 4096))])   # n * qmax a power of 4, or one row per channel
def test_lsq_backward_exact_sums(ext, oracle, sms, n, qmin, qmax, axis_shape):
    r = np.random.RandomState(n % 1000 + qmax)
    for mode in (0, 1, 6, 11):
        s, dy_unit = F32(2.0 ** -3), F32(2.0 ** -1)
        if axis_shape is None:
            x = dyadic_quotients(r, n, qmin, qmax) * s
            dy = (np.floor(r.uniform(-4, 4, n)) * dy_unit).astype(F32)
            _, p, f = oracle.linear_quant_backward(x, dy, [s], [2.0], qmin, qmax, mode)
            assert exactly_summable(p)
            run_lsq(ext, oracle, sms, x, dy, [s], [2.0], qmin, qmax, mode, None, f'exact LT n {n} mode {mode}', exact=True)
        else:
            shape = list(axis_shape)
            axis = 1 if len(shape) > 1 else 0
            C = shape[axis]
            sc = (2.0 ** r.randint(-4, 2, C)).astype(F32)
            x = dyadic_quotients(r, n, qmin, qmax).reshape(shape) * (sc.reshape([-1] + [1] * (len(shape) - axis - 1)))
            dy = (np.floor(r.uniform(-4, 4, n)) * dy_unit).reshape(shape).astype(F32)
            oc = np.floor(r.uniform(-3, 3, C)).astype(F32)
            _, p, f = oracle.linear_quant_backward(x, dy, sc, oc, qmin, qmax, mode, axis)
            assert exactly_summable(p)
            run_lsq(ext, oracle, sms, x.astype(F32), dy, sc, oc, qmin, qmax, mode, axis, f'exact LC {shape} mode {mode}', exact=True)


# ---- float backward ----------------------------------------------------------------------------------------------------------------
def tmax_of(E, M):
    return 2.0 ** (1 << (E - 1)) * (2 - 2.0 ** -M)


def run_fb(ext, oracle, x, dy, s, o, E, M, cmin, cmax, mode, axis, what, exact=False, call=None):
    if axis is None:
        gx, gs = (call or ext.QuantizeTensor_FT_B)(dev(x), dev(s), dev(o), dev(dy), E, M, cmin, cmax, mode)
        wx, p, d = oracle.float_quant_backward(x, dy, s, o, E, M, cmin, cmax, mode)
        epc = rows_of(x.size)
        groups, k = [p.reshape(-1)], chain_rows(epc, x.size // epc)
    else:
        gx, gs = (call or ext.QuantizeTensor_FC_B)(dev(x), dev(s), dev(o), dev(dy), E, M, cmin, cmax, mode, axis)
        wx, p, d = oracle.float_quant_backward(x, dy, s, o, E, M, cmin, cmax, mode, axis)
        epc, C = oracle.channel_geometry(x.shape, axis)
        ch = (np.arange(x.size) // epc) % C
        groups, k = [p.reshape(-1)[ch == c] for c in range(C)], chain_rows(epc, x.size // (epc * C))
    assert_same(gx, wx, what + ' grad_x')
    check_sum(gs, groups, d, True, k, exact, what + ' grad_s')


@pytest.mark.parametrize('E,M,grid_max', FORMATS)
def test_float_backward_formats_clips_modes(ext, oracle, E, M, grid_max):
    r = np.random.RandomState(E * 16 + M + int(grid_max) % 7)
    tmax = tmax_of(E, M)
    clips = {'on grid': grid_max, 'off grid': float(F32(grid_max * 1.0 + grid_max * 2.0 ** -(M + 2))), 'beyond tmax': tmax * 1.5,
             'tmax': tmax}
    for tag, cmax in clips.items():
        for mode in MODES:
            for s, o in ((0.5, 0.0), (0.37, 1.5), (2.0 ** -20, -3.0), (3e4, 0.25)):
                t = fp_quotients(r, 512, E, M, min(cmax, tmax))
                x = (t * F32(s)).astype(F32)
                dy = r.randn(512).astype(F32)
                run_fb(ext, oracle, x, dy, [s], [o], E, M, -cmax, cmax, mode, None, f'FT E{E}M{M} {tag} mode {mode} s {s} o {o}')
            x = (fp_quotients(r, 512, E, M, min(cmax, tmax)) * F32(0.75)).astype(F32).reshape(2, 4, 64)
            dy = with_specials(r, r.randn(2, 4, 64).astype(F32))
            run_fb(ext, oracle, with_specials(r, x), dy, np.array([0.75, 0.5, 1e-3, 6.0], F32), np.array([0, 1.5, -2, 0.3], F32),
                   E, M, -cmax, cmax, mode, 1, f'FC E{E}M{M} {tag} mode {mode}')


@pytest.mark.parametrize('shape,axis', [([1], None), ([255], None), ([768], None), ([8192 * 3], None), ([10007], None),
                                        ([(1 << 24) + 3], None), ([16, 3, 32], 0), ([5, 7, 1], -2), ([3, 300], 1), ([40, 1], 0)])
def test_float_backward_geometry(ext, oracle, shape, axis):
    r = np.random.RandomState(sum(shape) % 101)
    n = int(np.prod(shape))
    C = 1 if axis is None else shape[axis]
    s = (2.0 ** r.randint(-3, 3, C)).astype(F32)
    x = (fp_quotients(r, n, 4, 3, 448.0).reshape(shape) * s.max()).astype(F32)
    dy = r.randn(*shape).astype(F32)
    run_fb(ext, oracle, x, dy, s, np.zeros(C, F32), 4, 3, -448.0, 448.0, int(r.choice(MODES)), axis, f'{shape} axis {axis}')


@pytest.mark.parametrize('n,cmax,axis_shape', [(1, 448.0, None), (255, 448.0, None), (1024, 256.0, None), (1 << 16, 64.0, None),
                                               (4096, 16.0, (4, 1024)), (768, 448.0, (3, 256))])
def test_float_backward_exact_sums(ext, oracle, n, cmax, axis_shape):
    """Power-of-two scale and dy, quotients on a coarse dyadic grid, n * cmax a power of 4 (or one row per output)."""
    r = np.random.RandomState(n % 997)
    for mode in (0, 2, 7):
        t = (np.floor(r.uniform(-cmax - 4, cmax + 4, n) * 4) / 4).astype(F32)
        dy = (np.floor(r.uniform(-4, 4, n)) / 2).astype(F32)
        if axis_shape is None:
            s = F32(0.5)
            _, p, _ = oracle.float_quant_backward(t * s, dy, [s], [0.0], 4, 3, -cmax, cmax, mode)
            assert exactly_summable(p)
            run_fb(ext, oracle, t * s, dy, [s], [0.0], 4, 3, -cmax, cmax, mode, None, f'exact FT n {n} mode {mode}', exact=True)
        else:
            C = axis_shape[0]
            sc = (2.0 ** r.randint(-2, 2, C)).astype(F32)
            x = (t.reshape(axis_shape) * sc[:, None]).astype(F32)
            oc = np.floor(r.uniform(-2, 2, C)).astype(F32)
            _, p, _ = oracle.float_quant_backward(x, dy.reshape(axis_shape), sc, oc, 4, 3, -cmax, cmax, mode, 0)
            assert exactly_summable(p)
            run_fb(ext, oracle, x, dy.reshape(axis_shape), sc, oc, 4, 3, -cmax, cmax, mode, 0, f'exact FC {axis_shape} mode {mode}',
                   exact=True)


# ---- TensorClip ----------------------------------------------------------------------------------------------------------------------
def test_tensor_clip(ext, oracle):
    r = np.random.RandomState(5)
    sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e38, -1e38], F32)
    for shape, axis in (([1], 0), ([255], 0), ([10007], 0), ([8192 * 3 + 1], 0), ([5, 12, 13, 4], 1), ([3, 7, 1], -1), ([4, 6, 5], 2),
                        ([1, 9], 0), ([2, 1, 3], 1)):
        n = int(np.prod(shape))
        v = r.randn(*shape).astype(F32)
        ref_ = r.randn(*shape).astype(F32)
        v.reshape(-1)[r.choice(n, min(n, 7), replace=False)] = sp[:min(n, 7)]
        ref_.reshape(-1)[r.choice(n, min(n, 7), replace=False)] = sp[:min(n, 7)]
        ref_.reshape(-1)[:min(n, 3)] = v.reshape(-1)[:min(n, 3)]                 # v on both bounds when the limit is 0
        C = shape[axis]
        for lim in (np.array([0.5], F32), np.array([0.0], F32), np.array([-0.25], F32), np.array([np.nan], F32), np.array([np.inf], F32)):
            assert_same(ext.TensorClip_T(dev(v), dev(ref_), dev(lim)), oracle.tensor_clip(v, ref_, lim), f'T {shape} {lim}')
        limc = r.randn(C).astype(F32)
        limc[:1] = 0.0
        if C > 2: limc[2] = np.nan
        assert_same(ext.TensorClip_C(dev(v), dev(ref_), dev(limc), axis), oracle.tensor_clip(v, ref_, limc, axis), f'C {shape} {axis}')
    v, ref_ = dev(r.randn(6, 5).astype(F32)), dev(r.randn(6, 5).astype(F32))
    lim = r.rand(6).astype(F32)
    got = ext.TensorClip_C(v.t(), ref_.t(), dev(lim).view(1, 6), 1)
    assert_same(got, oracle.tensor_clip(host(v.t().contiguous()), host(ref_.t().contiguous()), lim, 1), 'transposed')


# ---- RoundingLoss --------------------------------------------------------------------------------------------------------------------
def run_rl(ext, oracle, sms, x, s, o, qmin, qmax, mode, axis, dy0, what, exact=False, wrappers=False):
    if axis is None:
        loss = ext.RoundingLoss_LT(dev(x), dev(s), dev(o), qmin, qmax, mode)
        grad = ext.RoundingLoss_LT_B(dev(x), dev([dy0]), dev(s), dev(o), qmin, qmax, mode)
    else:
        loss = ext.RoundingLoss_LC(dev(x), dev(s), dev(o), qmin, qmax, axis, mode)
        grad = ext.RoundingLoss_LC_B(dev(x), dev([dy0]), dev(s), dev(o), qmin, qmax, axis, mode)
    p, d = oracle.rounding_loss(x, s, o, qmin, qmax, mode, axis)
    assert_same(grad, oracle.rounding_loss_backward(x, [dy0], s, o, qmin, qmax, mode, axis), what + ' grad')
    check_sum(loss, [p.reshape(-1)], d, True, chain_flat(x.size, sms), exact, what + ' loss')


@pytest.mark.parametrize('qmin,qmax', RANGES)
def test_rounding_loss_modes_offsets(ext, oracle, sms, qmin, qmax):
    r = np.random.RandomState((qmax & 0xfff) + 1)
    for mode in MODES:
        for off in OFFSETS:
            s = F32(r.choice([0.25, 0.37, 3.1e-3, 17.0]))
            x = (int_quotients(r, 640, qmin, qmax, round(off)) * s).astype(F32)
            run_rl(ext, oracle, sms, x, [s], [off], qmin, qmax, mode, None, F32(0.7), f'LT {qmin}..{qmax} mode {mode} o {off}')
            # per channel, with the clip bounds of the UNROUNDED offset planted: they differ from the rounded ones for half-integers
            sc = np.array([s, 0.5, 0.11, 2.0], F32); oc = np.array([off, off + 1, -off, 0.5], F32)
            xc = x.reshape(4, 160).copy()
            for c in range(4):
                xc[c, :2] = sc[c] * (F32(qmax) - oc[c]), sc[c] * (F32(qmin) - oc[c])
                xc[c, 2:4] = np.nextafter(xc[c, :2], F32(np.inf))
            run_rl(ext, oracle, sms, xc, sc, oc, qmin, qmax, mode, 0, F32(-1.25), f'LC {qmin}..{qmax} mode {mode} o {off}')
        x = with_specials(r, (int_quotients(r, 300, qmin, qmax, 0) * F32(0.5)).astype(F32))
        for dy0 in (F32(0.0), F32(-0.0), F32(np.inf), F32(np.nan)):
            run_rl(ext, oracle, sms, x, [0.5], [0.5], qmin, qmax, mode, None, dy0, f'LT specials mode {mode} dy {dy0}')
            run_rl(ext, oracle, sms, x.reshape(3, 100), [0.5, 1e-30, 3e30], [2.5, -0.5, 1.0], qmin, qmax, mode, 0, dy0,
                   f'LC specials mode {mode} dy {dy0}')


@pytest.mark.parametrize('shape,axis', [([1], None), ([255], None), ([256], None), ([768], None), ([8192 * 3], None),
                                        ([1000003], None), ([(1 << 24) + 3], None), ([8, 16, 5, 5], 0), ([4, 16, 7, 7], 1),
                                        ([2, 9, 300], -1), ([64, 1], 0), ([3, 1, 5], 1), ([1024, 3, 3], 2)])
def test_rounding_loss_geometry(ext, oracle, sms, shape, axis):
    r = np.random.RandomState(sum(shape) % 89)
    n = int(np.prod(shape))
    C = 1 if axis is None else shape[axis]
    s = (r.rand(C) * 0.1 + 0.02).astype(F32)
    o = r.choice([0.0, 2.5, -3.5, 0.5], C).astype(F32)
    x = (int_quotients(r, n, -128, 127, 0).reshape(shape) * s.max()).astype(F32)
    run_rl(ext, oracle, sms, x, s, o, -128, 127, int(r.choice(MODES)), axis, F32(0.3), f'{shape} axis {axis}')


@pytest.mark.parametrize('n', [1, 7, 256, 2048, 4096, 1 << 18])
def test_rounding_loss_exact_sums(ext, oracle, sms, n):
    """Quotients on a 1/8 grid and a power-of-two scale: every |deq - v| is a multiple of s / 8.  One CTA (n <= 2048) or n a power
    of 4 (sqrtf(n) a power of two): bit-exact."""
    r = np.random.RandomState(n % 991)
    for mode in (0, 3, 7, 11):
        s = F32(0.25)
        x = (dyadic_quotients(r, n, -8, 7) * s).astype(F32)
        p, _ = oracle.rounding_loss(x, [s], [0.0], -8, 7, mode)
        assert exactly_summable(p)
        run_rl(ext, oracle, sms, x, [s], [0.0], -8, 7, mode, None, F32(0.5), f'exact n {n} mode {mode}', exact=True)
        run_rl(ext, oracle, sms, x.reshape(1, -1), [s], [1.0], -8, 7, mode, 0, F32(0.5), f'exact LC n {n} mode {mode}', exact=True)


# ---- single-element tensors: one partial, so the result is the normaliser applied once -------------------------------------------
def test_single_element_reductions_are_bit_exact(ext, oracle, sms):
    r = np.random.RandomState(17)
    cases = 0
    for qmin, qmax in RANGES + [(-127, 0), (-2, 1), (0, 3), (-64, 63)]:
        for off in (0.0, 2.5, -1.0):
            for t in (0.0, 0.3, -0.7, 2.5, qmax - round(off) + 0.75, qmin - round(off) - 2.0, 1e11):   # 0: a zero sum, NaN for a NaN factor
                for s in (0.37, 0.5, 3e-3):
                    x = np.array([F32(t) * F32(s)], F32)
                    dy = np.array([r.randn()], F32)
                    run_lsq(ext, oracle, sms, x, dy, [s], [off], qmin, qmax, int(r.choice(MODES)), None, f'LT 1 {qmin}..{qmax} {t}', exact=True)
                    run_lsq(ext, oracle, sms, x, dy, [s], [off], qmin, qmax, 0, 0, f'LC 1 {qmin}..{qmax} {t}', exact=True)
                    run_rl(ext, oracle, sms, x, [s], [off], qmin, qmax, 0, None, F32(1.0), f'RL 1 {qmin}..{qmax} {t}', exact=True)
                    run_rl(ext, oracle, sms, x, [s], [off], qmin, qmax, 0, 0, F32(1.0), f'RLC 1 {qmin}..{qmax} {t}', exact=True)
                    cases += 1
    for E, M, cmax in FORMATS:
        for cm in (cmax, cmax * 0.7, tmax_of(E, M) * 2):
            for u in (0.3, -1.7, cm * 0.9, cm + 0.5, cm + 3, -cm - 3):
                for s in (0.37, 0.5):
                    x = np.array([F32(u) * F32(s)], F32)
                    dy = np.array([r.randn()], F32)
                    run_fb(ext, oracle, x, dy, [s], [0.0], E, M, -cm, cm, 0, None, f'FT 1 E{E}M{M} {cm} {u}', exact=True)
                    run_fb(ext, oracle, x, dy, [s], [0.5], E, M, -cm, cm, 0, 0, f'FC 1 E{E}M{M} {cm} {u}', exact=True)
    assert cases > 300


# ---- the callers -------------------------------------------------------------------------------------------------------------------
def test_ffi_wrappers_argument_order(ext, oracle, sms):
    """The wrappers take (..., channel_axis, rounding) in Python and pass (..., rounding, channel_axis) to the extension.  On a
    [4, 8, 8] tensor with axis 2 and mode 1 a swapped order still runs (axis 1 also has 8 channels, mode 2 is valid) but gives
    other channels and other ties."""
    from ppq_b200.ffi import CUDA
    r = np.random.RandomState(23)
    x = (dyadic_quotients(r, 256, -8, 7) * F32(0.25)).reshape(4, 8, 8).astype(F32)
    x.reshape(-1)[::3] = (np.floor(r.uniform(-8, 7, x.size // 3 + 1)) + 0.5)[:len(x.reshape(-1)[::3])] * F32(0.25)
    dy = r.randn(4, 8, 8).astype(F32)
    s = (r.rand(8) * 0.1 + 0.2).astype(F32); o = np.array([0, 1, -1, 2, 0.5, 3, -2, 1], F32)
    gx, gs = CUDA.LinearQuantize_C_B(dev(x), dev(s), dev(o), dev(dy), -8, 7, 2, 1)
    wx, p, f = oracle.linear_quant_backward(x, dy, s, o, -8, 7, 1, 2)
    assert_same(gx, wx, 'LinearQuantize_C_B grad_x')
    check_sum(gs, [p[:, :, c].reshape(-1) for c in range(8)], f, False, chain_rows(1, 32), False, 'LinearQuantize_C_B grad_s')
    gx, gs = CUDA.FloatingQuantize_C_B(dev(x), dev(s), dev(o), dev(dy), 4, 3, -6.0, 6.0, 2, 1)
    wx, p, d = oracle.float_quant_backward(x, dy, s, o, 4, 3, -6.0, 6.0, 1, 2)
    assert_same(gx, wx, 'FloatingQuantize_C_B grad_x')
    check_sum(gs, [p[:, :, c].reshape(-1) for c in range(8)], d, True, chain_rows(1, 32), False, 'FloatingQuantize_C_B grad_s')
    gx, gs = CUDA.LinearQuantize_T_B(dev(x), dev(s[:1]), dev(o[:1]), dev(dy), -8, 7, 4)
    wx, p, f = oracle.linear_quant_backward(x, dy, s[:1], o[:1], -8, 7, 4)
    assert_same(gx, wx, 'LinearQuantize_T_B')
    g = CUDA.RoundingLoss_LC_B(dev(x), dev([0.5]), dev(s), dev(o), 2, -8, 7, 1)
    assert_same(g, oracle.rounding_loss_backward(x, [0.5], s, o, -8, 7, 1, 2), 'RoundingLoss_LC_B')
    loss = CUDA.RoundingLoss_LC(dev(x), dev(s), dev(o), 2, -8, 7, 6)
    p, d = oracle.rounding_loss(x, s, o, -8, 7, 6, 2)
    check_sum(loss, [p.reshape(-1)], d, True, chain_flat(x.size, sms), False, 'RoundingLoss_LC')


def test_culsq_autograd_non_default_mode(ext, oracle, sms):
    from ppq_b200.core import RoundingPolicy
    from ppq_b200.qfunction import CuLSQ_LC, CuLSQ_LT
    r = np.random.RandomState(29)
    xn = (int_quotients(r, 6 * 8 * 16, 0, 255, 3) * F32(0.11)).reshape(6, 8, 16).astype(F32)
    w = r.randn(6, 8, 16).astype(F32)
    x = dev(xn).requires_grad_()
    s = dev([0.11]).requires_grad_(); o = dev([2.5])
    (CuLSQ_LT.apply(x, s, o, 0, 255, RoundingPolicy.ROUND_HALF_UP) * dev(w)).sum().backward()
    wx, p, f = oracle.linear_quant_backward(xn, w, [0.11], [2.5], 0, 255, int(RoundingPolicy.ROUND_HALF_UP.value))
    assert_same(x.grad, wx, 'CuLSQ_LT grad_x')
    check_sum(s.grad, [p.reshape(-1)], f, False, chain_rows(xn.size, 1), False, 'CuLSQ_LT grad_s')
    x2 = dev(xn).requires_grad_()
    sc = dev((r.rand(8) * 0.2 + 0.05).astype(F32)).requires_grad_(); oc = dev(np.array([0, 0.5, -0.5, 1.5, 2, -3, 4, 0], F32))
    (CuLSQ_LC.apply(x2, sc, oc, 1, -128, 127, RoundingPolicy.ROUND_HALF_TOWARDS_ZERO) * dev(w)).sum().backward()
    wx, p, f = oracle.linear_quant_backward(xn, w, host(sc.detach()), host(oc), -128, 127, int(RoundingPolicy.ROUND_HALF_TOWARDS_ZERO.value), 1)
    assert_same(x2.grad, wx, 'CuLSQ_LC grad_x')
    check_sum(sc.grad, [p[:, c].reshape(-1) for c in range(8)], f, False, chain_rows(16, 6), False, 'CuLSQ_LC grad_s')


# ---- the reference's own kernels on the new modes, offsets and formats (recorded, tests/refcuda.py) ----------------------------------
def test_reference_kernels_agree_with_the_oracle(ext, oracle, sms, ref):
    """Pins the oracle to the reference's CUDA build for rounding modes 1-7, half-integer offsets, 4-bit ranges and the float formats.
    Reductions are compared only where the reference's own is well defined: LT_B with n a multiple of its 1024-thread block, FT_B
    within 2560 blocks of 1024."""
    r = np.random.RandomState(31)
    n = 4096
    for mode in range(8):
        for (qmin, qmax), off in (((0, 255), 2.5), ((-8, 7), -0.5), ((0, 15), 3.5), ((-128, 127), 1.3)):
            s = F32(0.37)
            x = (int_quotients(r, n, qmin, qmax, round(off)) * s).astype(F32)
            dy = r.randn(n).astype(F32)
            rx, rs = ref.QuantizeTensor_LT_B(dev(x), dev([s]), dev([off]), dev(dy), qmin, qmax, mode)
            wx, p, f = oracle.linear_quant_backward(x, dy, [s], [off], qmin, qmax, mode)
            assert_same(rx, wx, f'ref LT_B mode {mode}')
            check_sum(rs, [p], f, False, REF_K, False, f'ref LT_B mode {mode}')
            xc, dyc = x.reshape(4, 8, 128), dy.reshape(4, 8, 128)
            sc = (r.rand(8) * 0.3 + 0.05).astype(F32); oc = np.full(8, off, F32)
            rx, rs = ref.QuantizeTensor_LC_B(dev(xc), dev(sc), dev(oc), dev(dyc), qmin, qmax, mode, 1)
            wx, p, f = oracle.linear_quant_backward(xc, dyc, sc, oc, qmin, qmax, mode, 1)
            assert_same(rx, wx, f'ref LC_B mode {mode}')
            check_sum(rs, [p[:, c].reshape(-1) for c in range(8)], f, False, 1 + 10 + 4, False, f'ref LC_B mode {mode}')
            dy0 = F32(0.7)
            assert_same(ref.RoundingLoss_LT_B(dev(x), dev([dy0]), dev([s]), dev([off]), qmin, qmax, mode),
                        oracle.rounding_loss_backward(x, [dy0], [s], [off], qmin, qmax, mode), f'ref RL_LT_B mode {mode}')
            assert_same(ref.RoundingLoss_LC_B(dev(xc), dev([dy0]), dev(sc), dev(oc), qmin, qmax, 1, mode),
                        oracle.rounding_loss_backward(xc, [dy0], sc, oc, qmin, qmax, mode, 1), f'ref RL_LC_B mode {mode}')
            p, d = oracle.rounding_loss(x, [s], [off], qmin, qmax, mode)
            check_sum(ref.RoundingLoss_LT(dev(x), dev([s]), dev([off]), qmin, qmax, mode), [p], d, True, REF_K, False, 'ref RL_LT')
            p, d = oracle.rounding_loss(xc, sc, oc, qmin, qmax, mode, 1)
            check_sum(ref.RoundingLoss_LC(dev(xc), dev(sc), dev(oc), qmin, qmax, 1, mode), [p.reshape(-1)], d, True, REF_K, False,
                      'ref RL_LC')
        for E, M, cmax in FORMATS:
            for cm in (cmax, float(F32(cmax * 0.93)), tmax_of(E, M) * 1.5):
                x = (fp_quotients(r, n, E, M, min(cm, tmax_of(E, M))) * F32(0.5)).astype(F32)
                dy = r.randn(n).astype(F32)
                rx, rs = ref.QuantizeTensor_FT_B(dev(x), dev([0.5]), dev([0.25]), dev(dy), E, M, -cm, cm, mode)
                wx, p, d = oracle.float_quant_backward(x, dy, [0.5], [0.25], E, M, -cm, cm, mode)
                assert_same(rx, wx, f'ref FT_B E{E}M{M} {cm} mode {mode}')
                check_sum(rs, [p], d, True, REF_K, False, f'ref FT_B E{E}M{M} {cm} mode {mode}')
                xc, dyc = x.reshape(4, 1024), dy.reshape(4, 1024)
                sc = np.array([0.5, 0.25, 2.0, 0.37], F32); oc = np.array([0, 1, -0.5, 0.25], F32)
                rx, rs = ref.QuantizeTensor_FC_B(dev(xc), dev(sc), dev(oc), dev(dyc), E, M, -cm, cm, mode, 0)
                wx, p, d = oracle.float_quant_backward(xc, dyc, sc, oc, E, M, -cm, cm, mode, 0)
                assert_same(rx, wx, f'ref FC_B E{E}M{M} {cm} mode {mode}')
                check_sum(rs, [p[c] for c in range(4)], d, True, REF_K, False, f'ref FC_B E{E}M{M} {cm} mode {mode}')
    v, rr = r.randn(8, 512).astype(F32), r.randn(8, 512).astype(F32)
    v[0, :5] = [0.0, -0.0, np.inf, -np.inf, np.nan]
    lim = r.randn(8).astype(F32)
    assert_same(ref.TensorClip_T(dev(v), dev(rr), dev(lim[:1])), oracle.tensor_clip(v, rr, lim[:1]), 'ref TensorClip_T')
    assert_same(ref.TensorClip_C(dev(v), dev(rr), dev(lim), 0), oracle.tensor_clip(v, rr, lim, 0), 'ref TensorClip_C')
