"""The fp32 fake-quant launch routes, restated on the host: which kernel `launch_channel` / `launch_tensor` (ppq_b200/csrc/fakequant.cu)
picks for a shape, an alignment, an output type and a variant, which operator the C entries instantiate for a rounding id and clip range,
and the host predicate `float_fast_path_ok` that sends a float format to the branch-free FloatOp.

tests/test_gpu_fakequant_routes.py runs every case of ROUTE_CASES on the device, checks with the profiler that the kernel it names is the
one that ran, and compares the output with the oracle bit for bit.  The tests here need no GPU: they check that the case table reaches
every (route x operator family x output type) cell, and that the predicate twin agrees with an independent definition of "both clip
bounds lie on the format's normal grid", and with the oracle: where it says yes, clamp-then-round equals the reference's slow path.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

H100_SMS = 132

# ---- the dispatch, restated ---------------------------------------------------------------------------------------------------
CHANNEL_ROUTES = ('seg', 'table4', 'vec', 'last', 'ragged', 'generic')
TENSOR_ROUTES = ('vec8', 'vec', 'scalar')
FAMILIES = ('lin', 'lin_dyn', 'float_fast', 'float_slow')      # LinearOp<0..7>, LinearOp<-1>, FloatOp<M, true>, FloatOp<0|-1, false>
OUT_BYTES = {'float': 4, 'int32': 4, 'int8': 1}


def grid_for(work, threads, per_thread, ctas_per_sm, sms=H100_SMS):
    """common.cuh:201-208."""
    per_cta = threads * per_thread
    return max(1, min((work + per_cta - 1) // per_cta, sms * ctas_per_sm))


def channel_route(n, epc, C, x_al, y_al, variant=0, sms=H100_SMS):
    """launch_channel, fakequant.cu:650-699.  x_al: x is 16-byte aligned; y_al: y is aligned to 4 output elements (out_aligned)."""
    al = x_al and y_al
    if epc % 4 == 0 and al:
        n4 = n // 4
        if n4 <= 0x1fffffff and epc // 4 >= 128:                        # :663
            return 'seg'
        if n <= 0x7fffffff and variant == 0:                           # :669
            return 'table4'
        if n4 <= 0x7fffffff:                                           # :674
            return 'vec'
    if epc == 1 and C % 4 == 0 and al:                                 # :681-688
        if grid_for(n // 4, 256, 4, 8, sms) * 256 >= C // 4:
            return 'last'
    if epc >= 4 and al and n <= 0x7fffffff and variant == 0:           # :690
        return 'ragged'
    return 'generic'                                                   # :695


def tensor_route(n, x_al, y_al, light, out_bytes):
    """launch_tensor, fakequant.cu:633-648 (Op::kLight: LinearOp<0> and every FloatOp<M, true>)."""
    vec = x_al and y_al
    if vec and light and out_bytes == 4 and n >= 1 << 25:              # :638
        return 'vec8'
    return 'vec' if vec else 'scalar'


def family(op, mode, fmt=None):
    """The operator an entry instantiates (fakequant.cu:747-943).  op: LT / LC (float out), QT / QC (toInt), FT / FC.
    LT / LC: PPQB_DISPATCH_MODE, ids 0..7 compile-time, anything else LinearOp<-1>.  toInt: only HALF_EVEN is compile-time.
    FT / FC: the fast FloatOp when the predicate holds and the id is 0..7, else FloatOp<0, false> / FloatOp<-1, false>."""
    if op in ('LT', 'LC'):
        return 'lin' if 0 <= mode <= 7 else 'lin_dyn'
    if op in ('QT', 'QC'):
        return 'lin' if mode == 0 else 'lin_dyn'
    E, M, cmin, cmax = fmt
    return 'float_fast' if float_fast_path_ok(E, M, cmin, cmax) and 0 <= mode <= 7 else 'float_slow'


def is_light(op, mode, fam):
    return fam == 'float_fast' or (fam == 'lin' and mode == 0)


# ---- float_fast_path_ok, restated (fakequant.cu:701-712) --------------------------------------------------------------------------
def _f2u(f):
    return int(np.float32(f).view(np.uint32))


def _u2f(u):
    return np.uint32(u & 0xFFFFFFFF).view(np.float32)


def fp_tmax(E, M):
    """2^emax * (2 - 2^-M), emax = 2^(E-1): the largest value the rounding can produce (E4M3: 480)."""
    return _u2f((((1 << (E - 1)) + 127) << 23) + (~(0x007FFFFF >> M) & 0x007FFFFF))


def float_fast_path_ok(E, M, cmin, cmax):
    emin = -(1 << (E - 1)) + 1
    tmax = fp_tmax(E, M)
    cmin, cmax = np.float32(cmin), np.float32(cmax)
    hi = cmax if cmax < tmax else tmax
    lo = cmin if cmin > -tmax else -tmax
    thresh = (emin + 1 + 127) << 23
    half_minus1 = (1 << (22 - M)) - 1
    keep = ~((1 << (23 - M)) - 1) & 0xFFFFFFFF
    hb, lb = _f2u(hi) & 0x7FFFFFFF, _f2u(lo) & 0x7FFFFFFF
    return bool(hi > 0 and lo < 0 and hb >= thresh and lb >= thresh
                and ((hb + half_minus1) & keep) == hb and ((lb + half_minus1) & keep) == lb)


def on_normal_grid(v, E, M):
    """Independent definition: v is a normal number of FP(E, M) -- |v| >= 2^(emin + 1) and v = m * 2^e with M fraction bits."""
    v = float(v)
    if not math.isfinite(v) or v == 0:
        return False
    emin = -(1 << (E - 1)) + 1
    m, e = math.frexp(abs(v))                                          # |v| = m * 2^e, m in [0.5, 1)
    return e - 1 >= emin + 1 and (Fraction(m) * 2 ** (M + 1)).denominator == 1


FORMATS = ((4, 3), (5, 2), (3, 4), (2, 1), (5, 10))


def fp_grid_point(E, M):
    """A normal grid point below the format maximum with a non-zero mantissa (E4M3: 144), and its grid neighbour above."""
    e = max(1, (1 << (E - 1)) - 1)
    g = 2.0 ** e * (1 + 2.0 ** -M)
    return np.float32(g), np.float32(g + 2.0 ** (e - M))


def boundary_clips(E, M):
    """The clip pairs of the fast-path boundary: at and beyond the format maximum, on a grid point, one float ulp either side, between two
    grid points, one-sided, cmin > 0, asymmetric, inside the subnormal range.  (cmin, cmax, fast path expected)."""
    t = fp_tmax(E, M)
    g, g2 = fp_grid_point(E, M)
    up, dn = np.nextafter(g, np.float32(np.inf)), np.nextafter(g, np.float32(-np.inf))
    mid = np.float32((float(g) + float(g2)) / 2)
    sub = np.float32(2.0 ** (-(1 << (E - 1)) + 1))                    # 2^emin: below the normal threshold 2^(emin + 1)
    beyond = np.float32(float(t) * 1.04)
    return [(-t, t, True), (-beyond, beyond, True), (-g, g, True), (-up, up, False), (-dn, dn, False), (-mid, mid, False),
            (-g, up, False), (np.float32(0), t, False), (-t, np.float32(0), False), (g, t, False), (-t, g, True), (-t, mid, False),
            (-sub, sub, False), (-sub, t, False)]


# ---- the case table -------------------------------------------------------------------------------------------------------------
# Per-channel geometries: (outer, C, epc, x offset in floats, y offset in elements, variant) chosen at each route's edges.
CHANNEL_GEOMS = [
    (1, 4, 512, 0, 0, 0), (3, 5, 516, 0, 0, 0), (2, 3, 4100, 4, 0, 0), (3, 1, 516, 0, 4, 0), (1, 47, 512, 0, 0, 0),    # seg
    (1, 4, 4, 0, 0, 0), (3, 47, 8, 0, 0, 0), (2, 7, 508, 0, 0, 0), (1, 768, 12, 4, 0, 0), (3, 1, 4, 0, 0, 0),            # table4
    (1, 4, 4, 0, 0, 1), (3, 47, 8, 0, 0, 1), (2, 7, 508, 0, 0, 1), (1, 768, 12, 0, 4, 1),                               # vec
    (197, 768, 1, 0, 0, 0), (5, 4, 1, 0, 0, 0), (3, 48, 1, 4, 0, 1),                                                    # last
    (3, 47, 9, 0, 0, 0), (1, 5, 511, 0, 0, 0), (2, 7, 513, 0, 0, 0), (1, 768, 9, 0, 0, 0), (3, 4, 5, 0, 0, 0),           # ragged
    (3, 47, 9, 0, 0, 1), (1, 5, 511, 0, 0, 1), (2, 400000, 1, 0, 0, 0), (3, 47, 1, 0, 0, 0), (2, 7, 3, 0, 0, 0),         # generic
    (1, 4, 9, 1, 0, 0), (3, 5, 516, 2, 0, 0), (1, 4, 512, 3, 0, 0), (3, 47, 8, 0, 1, 0), (1, 5, 12, 0, 2, 0), (2, 3, 2, 0, 0, 0),
]
TENSOR_GEOMS = [(1, 0, 0), (3, 0, 0), (4099, 0, 0), (70001, 0, 0), (4099, 1, 0), (70001, 3, 0), (4100, 0, 1), (5, 2, 0)]


def y_aligned(y_off, out):
    """Output bases are allocation-aligned (>= 256 bytes) plus y_off elements; out_aligned wants 4 elements' worth of bytes."""
    return (y_off * OUT_BYTES[out]) % (4 * OUT_BYTES[out]) == 0


E4M3_FAST, E4M3_SLOW = (4, 3, -448.0, 448.0), (4, 3, -300.0, 300.0)
# (op, mode, output type, float format): one per (family x output type) cell
OPERATOR_CELLS = [('LC', 3, 'float', None), ('LC', 11, 'float', None), ('QC', 0, 'int32', None), ('QC', 0, 'int8', None),
                  ('QC', 4, 'int32', None), ('QC', 11, 'int8', None), ('FC', 1, 'float', E4M3_FAST), ('FC', 11, 'float', E4M3_SLOW)]


def _channel_cases():
    out = []
    for outer, C, epc, xo, yo, var in CHANNEL_GEOMS:
        n = outer * C * epc
        for op, mode, ot, fmt in OPERATOR_CELLS:
            fam = family(op, mode, fmt)
            route = channel_route(n, epc, C, xo % 4 == 0, y_aligned(yo, ot), var)
            out.append(dict(kind='C', op=op, mode=mode, out=ot, fmt=fmt, outer=outer, C=C, epc=epc, x_off=xo, y_off=yo, variant=var,
                            route=route, family=fam))
    return out


def _tensor_cases():
    out = []
    big = [(2 ** 25 + 3, 0, 0), (2 ** 25 + 151, 0, 0), (2 ** 25 + 3, 1, 0)]      # the 8-deep loop, its partial last segment, the scalar loop
    for n, xo, yo in TENSOR_GEOMS + big:
        cells = [('LT', 0, 'float', None), ('LT', 5, 'float', None), ('LT', 11, 'float', None), ('QT', 0, 'int32', None), ('QT', 0, 'int8', None),
                 ('QT', 1, 'int32', None), ('QT', 11, 'int8', None), ('FT', 0, 'float', E4M3_FAST), ('FT', 6, 'float', E4M3_SLOW)]
        if n > 1 << 25:
            cells = [c for c in cells if (c[0], c[1]) in (('LT', 0), ('QT', 0), ('FT', 0)) and c[2] != 'int8']
        for op, mode, ot, fmt in cells:
            fam = family(op, mode, fmt)
            route = tensor_route(n, xo % 4 == 0, y_aligned(yo, ot), is_light(op, mode, fam), OUT_BYTES[ot])
            out.append(dict(kind='T', op=op, mode=mode, out=ot, fmt=fmt, n=n, x_off=xo, y_off=yo, route=route, family=fam))
    return out


ROUTE_CASES = _channel_cases() + _tensor_cases()


def case_id(c):
    geo = f'{c["outer"]}x{c["C"]}x{c["epc"]}v{c["variant"]}' if c['kind'] == 'C' else f'n{c["n"]}'
    return f'{c["op"]}-{c["route"]}-{c["family"]}-{c["out"]}-m{c["mode"]}-{geo}-x{c["x_off"]}y{c["y_off"]}'


# ---- tests ----------------------------------------------------------------------------------------------------------------------
def test_channel_cases_cover_every_route_family_and_output_cell():
    have = {(c['route'], c['family'], c['out']) for c in ROUTE_CASES if c['kind'] == 'C'}
    want = {(r, f, o) for r in CHANNEL_ROUTES for f in FAMILIES for o in OUT_BYTES
            if (o == 'float') or f in ('lin', 'lin_dyn')}                 # the float operators only emit floats
    assert want - have == set(), sorted(want - have)


def test_tensor_cases_cover_every_route_family_and_output_cell():
    have = {(c['route'], c['family'], c['out']) for c in ROUTE_CASES if c['kind'] == 'T'}
    want = set()
    for r in TENSOR_ROUTES:
        for f in FAMILIES:
            for o in OUT_BYTES:
                if o != 'float' and f not in ('lin', 'lin_dyn'):
                    continue
                if r == 'vec8' and (f == 'lin_dyn' or f == 'float_slow' or OUT_BYTES[o] != 4):
                    continue                                           # only light operators with 4-byte outputs take the 8-deep loop
                want.add((r, f, o))
    assert want - have == set(), sorted(want - have)


def test_route_edges_sit_on_both_sides_of_each_threshold():
    """The geometries straddle the thresholds they are meant to: epc 508/512 around the segment kernel, epc 4 (the smallest table row),
    a channel-last shape with fewer threads than channel groups, rows crossing the 4096-element tile and the 512-element segment."""
    r = {(o, C, e, xo, yo, v): channel_route(o * C * e, e, C, xo % 4 == 0, yo % 4 == 0, v) for o, C, e, xo, yo, v in CHANNEL_GEOMS}
    assert r[(2, 7, 508, 0, 0, 0)] == 'table4' and r[(1, 4, 512, 0, 0, 0)] == 'seg' and r[(1, 5, 511, 0, 0, 0)] == 'ragged'
    assert r[(1, 4, 4, 0, 0, 0)] == 'table4' and r[(3, 4, 5, 0, 0, 0)] == 'ragged' and r[(2, 7, 3, 0, 0, 0)] == 'generic'
    assert r[(2, 400000, 1, 0, 0, 0)] == 'generic' and r[(197, 768, 1, 0, 0, 0)] == 'last'
    assert grid_for(2 * 400000 // 4, 256, 4, 8) * 256 < 400000 // 4          # the channel-last fallback: threads < C / 4
    assert 4096 % 12 and 768 * 12 > 2 * 4096 and 4096 % 9 and 768 * 9 > 4096  # table rows straddle the tile
    assert 516 % 512 and 4100 % 512 and (2 * 4100) % 512                      # segment rows straddle the 512-element segment
    assert channel_route(8, 4, 2, True, True, 1) == 'vec' and channel_route(9 * 4, 9, 4, True, True, 1) == 'generic'


def test_ragged_tail_lies_in_one_row():
    """The ragged table kernel's scalar tail (the <= 3 elements after the last whole vector) never reaches a row end before the tensor's
    end: launch_channel refuses n % epc != 0 and the table route needs epc >= 4.  So the tail's re-bind to the next row is unreachable,
    and a kernel change there cannot be seen by any output."""
    for epc in range(4, 40):
        for rows in range(1, 20):
            n = rows * epc
            tail0 = n // 4 * 4
            assert all(e // epc == (n - 1) // epc for e in range(tail0, n))


@pytest.mark.parametrize('E,M', FORMATS)
def test_fast_path_twin_matches_grid_definition(E, M):
    """The predicate is true exactly when max(cmin, -tmax) < 0 < min(cmax, tmax) and both are normal grid points -- checked on the
    boundary clips and on every float32 within 3 ulps of 64 grid points and midpoints of the format."""
    t = fp_tmax(E, M)

    def indep(cmin, cmax):
        hi, lo = min(np.float32(cmax), t), max(np.float32(cmin), -t)
        return bool(hi > 0 and lo < 0 and on_normal_grid(hi, E, M) and on_normal_grid(lo, E, M))

    for cmin, cmax, fast in boundary_clips(E, M):
        assert float_fast_path_ok(E, M, cmin, cmax) == fast == indep(cmin, cmax), (E, M, cmin, cmax)
    emin = -(1 << (E - 1)) + 1
    pts = set()
    for e in np.linspace(emin - 1, (1 << (E - 1)), 16).astype(int):
        for k in (0, 1, (1 << M) - 1, 1 << max(M - 1, 0)):
            pts.add(np.float32(2.0 ** int(e) * (1 + k * 2.0 ** -M)))
            pts.add(np.float32(2.0 ** int(e) * (1 + (k + 0.5) * 2.0 ** -M)))
    for p in sorted(pts):
        v = p
        for _ in range(3):
            v = np.nextafter(v, np.float32(-np.inf))
        for _ in range(7):
            for cmin, cmax in ((-v, v), (-t, v), (-v, t)):
                assert float_fast_path_ok(E, M, cmin, cmax) == indep(cmin, cmax), (E, M, cmin, cmax)
            v = np.nextafter(v, np.float32(np.inf))


@pytest.mark.parametrize('E,M', FORMATS)
def test_oracle_float_dequantise_returns_the_canonical_nan(oracle, E, M):
    """Under ROUND_DOWN a NaN input keeps a NaN grid value with a payload; the GPU's (q - o) * s returns the canonical 0x7FFFFFFF for it
    (the reference's FT / FC kernels do), so the oracle must too, per tensor and per channel."""
    x = np.float32([np.nan, 1.0, -np.nan])
    for s, o in ((1.0, 0.0), (0.3, 2.5)):
        y = oracle.float_quant_t(x, s, o, E, M, -float(fp_tmax(E, M)), float(fp_tmax(E, M)), 7)
        assert y.view(np.uint32)[0] == 0x7FFFFFFF and y.view(np.uint32)[2] == 0x7FFFFFFF, [hex(v) for v in y.view(np.uint32)]
    y = oracle.float_quant_c(x.reshape(3, 1), np.float32([0.3]), np.float32([2.5]), 1, E, M, -6.0, 6.0, 7)
    assert y.view(np.uint32)[0] == 0x7FFFFFFF


def _fast_grid(x, s, E, M, cmin, cmax):
    """FloatOp<HALF_EVEN, true>::grid on u = x / s (ops.cuh:107-122), in numpy: clamp, then round the magnitude's discarded bits half-down in
    the normal range and ties-to-even on the sub-normal grid.  A NaN quotient is the device's canonical 0x7FFFFFFF."""
    u = (x / np.float32(s)).astype(np.float32)
    u = np.where(np.isnan(u), np.uint32(0x7FFFFFFF).view(np.float32), u)
    t = fp_tmax(E, M)
    hi, lo = min(np.float32(cmax), t), max(np.float32(cmin), -t)
    uc = np.where(np.isnan(u), u, np.minimum(np.maximum(u, lo), hi)).astype(np.float32)
    k = (1 << (E - 1)) + M - 2
    magic = np.float32(1.5 * 2.0 ** (23 - k))
    sub = ((uc + magic).astype(np.float32) - magic).astype(np.float32)
    nb = ((uc.view(np.uint32).astype(np.uint64) + ((1 << (22 - M)) - 1)) & (~((1 << (23 - M)) - 1) & 0xFFFFFFFF)).astype(np.uint32)
    thresh = np.float32(2.0 ** (-(1 << (E - 1)) + 2))
    return np.where(np.abs(uc) < thresh, sub, nb.view(np.float32))


@pytest.mark.parametrize('E,M', FORMATS)
def test_fast_path_equals_oracle_exactly_where_the_predicate_holds(oracle, E, M):
    """Where the predicate holds, clamp-then-round (what the fast kernel computes) equals the reference's slow path on a dense sweep of
    the format's range, the clip bounds' neighbours and the specials.  Where a clip bound is off the grid it does not, so the predicate
    is what keeps the fast kernel off those clips."""
    r = np.random.RandomState(E * 16 + M)
    t = float(fp_tmax(E, M))
    x = np.concatenate([(r.standard_normal(20000) * t / 3).astype(np.float32),
                        (r.standard_normal(4000) * 2.0 ** (-(1 << (E - 1)) + 1)).astype(np.float32),
                        np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, t, -t, 3e38, -3e38])])
    for cmin, cmax, fast in boundary_clips(E, M):
        xs = np.concatenate([x, np.float32([cmin, cmax]), np.nextafter(np.float32([cmin, cmax]), np.float32(np.inf)),
                             np.nextafter(np.float32([cmin, cmax]), np.float32(-np.inf))]).astype(np.float32)
        want = oracle.float_quant_t(xs, 1.0, 0.0, E, M, float(cmin), float(cmax), 0)
        got = _fast_grid(xs, 1.0, E, M, cmin, cmax)
        same = np.array_equal(got.view(np.uint32), want.view(np.uint32))
        if fast:
            assert same, (E, M, cmin, cmax, np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))[:5])
        elif float(cmin) == -float(cmax) and float(cmax) >= 2.0 ** (-(1 << (E - 1)) + 2):
            assert not same, (E, M, cmin, cmax)                        # symmetric, normal, off the grid
