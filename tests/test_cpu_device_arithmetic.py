"""CPU twins of the three arithmetic shortcuts the sm_90a kernels take (ppq_b200/csrc/common.cuh, ops.cuh), checked here without a GPU:

  1. ExactDiv: x / s through a hoisted reciprocal and two Markstein corrections == the IEEE fp32 quotient (exact rational arithmetic);
  2. the "+ .5" rounding modes evaluated in fp32 (floor / ceil + fraction test) == the reference's double formulation (the oracle);
  3. FloatOp<.., FAST>: clamp -> signed add of half-1 -> mask / magic-add sub-normal rounding == QuantizeScalarFloating (the oracle).

The GPU parity tests prove the kernels; these prove the *algorithms*, so a change to either side shows up on the CPU suite first."""
from fractions import Fraction

import numpy as np

F32_MIN_EXP = -149


def rn32(fr: Fraction) -> np.float32:
    """Correctly rounded (ties to even) float32 of an exact rational (single rounding, sub-normals included, no overflow expected)."""
    if fr == 0: return np.float32(0.0)
    sign = -1 if fr < 0 else 1
    a = abs(fr)
    e = a.numerator.bit_length() - a.denominator.bit_length()           # 2^(e-1) <= a < 2^(e+1)
    if a < Fraction(2) ** e: e -= 1                                       # now 2^e <= a < 2^(e+1)
    ulp_exp = max(e - 23, F32_MIN_EXP)
    m = a / (Fraction(2) ** ulp_exp)
    n = m.numerator // m.denominator
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and (n & 1)): n += 1
    return np.float32(sign * float(n) * 2.0 ** ulp_exp)                  # n < 2^25 and the power of two are exact in double -> exact product


def fr(x) -> Fraction:
    return Fraction(float(x))


def fma32(a, b, c) -> np.float32:
    return rn32(fr(a) * fr(b) + fr(c))


def markstein(x: np.float32, s: np.float32) -> np.float32:
    r = np.float32(1.0) / s                                               # == __frcp_rn(s): IEEE division is correctly rounded
    q0 = rn32(fr(x) * fr(r))
    e0 = fma32(-q0, s, x)
    q1 = fma32(e0, r, q0)
    e1 = fma32(-q1, s, x)
    return fma32(e1, r, q1)


def test_markstein_division_is_the_ieee_quotient():
    r = np.random.RandomState(2026)
    n_checked = 0
    with np.errstate(all='ignore'):
        for it in range(6000):
            s = np.float32(r.uniform(1, 2) * 2.0 ** r.randint(-59, 60) * (1 if r.rand() < 0.9 else -1))
            kind = it % 4
            if kind == 0: x = np.float32(r.standard_normal() * 10.0 ** r.uniform(-6, 6))
            elif kind == 1: x = np.float32((r.randint(-300, 300) + 0.5)) * s                     # quotient next to a rounding tie
            elif kind == 2: x = np.nextafter(np.float32((r.randint(-300, 300) + 0.5)) * s, np.float32(r.choice([-np.inf, np.inf])))
            else: x = np.float32(r.randint(-2 ** 24, 2 ** 24)) * np.float32(2.0 ** r.randint(-20, 20))
            want = x / s
            if not np.isfinite(want) or abs(float(want)) >= 2.0 ** 31 or (want != 0 and abs(float(want)) < 2.0 ** -40): continue    # slow-path domain
            if abs(float(x)) < 2.0 ** -100 and x != 0: continue                                    # residuals could underflow: harmless, see common.cuh
            got = markstein(np.float32(x), s)
            assert got.view(np.uint32) == np.float32(want).view(np.uint32) or (got == 0 and want == 0), (it, float(x), float(s), float(got), float(want))
            n_checked += 1
    assert n_checked > 4000


def sat_i32(a):
    a = np.where(np.isnan(a), 0.0, a.astype(np.float64))
    return np.clip(a, -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)


def dev_half_up(v):   return sat_i32(np.floor(v)) + ((v - np.floor(v)).astype(np.float32) >= np.float32(0.5))
def dev_half_down(v): return sat_i32(np.ceil(v)) - ((np.ceil(v) - v).astype(np.float32) >= np.float32(0.5))


def dev_round(v, mode):
    if mode == 1: return dev_half_up(v)
    if mode == 2: return dev_half_down(v)
    if mode == 3: return np.where(v > 0, dev_half_down(v), dev_half_up(v))
    return np.where(v > 0, dev_half_up(v), dev_half_down(v))               # 4 (far from zero) and 5 (round()): the same function


def test_fp32_rounding_formulation_equals_the_double_one(oracle):
    r = np.random.RandomState(7)
    h = np.arange(-3000, 3000, dtype=np.float32) + np.float32(0.5)
    tiny = np.float32([-1e-30, 1e-30, -1e-45, 1e-45, -0.49999997, 0.49999997, -0.50000006, 0.50000006, -0.5, 0.5, -0.0, 0.0,
                       -(0.5 - 2.0 ** -25), 0.5 - 2.0 ** -25, -0.99999994, 0.99999994, -1.0000001, 1.0000001, -0.25 - 2.0 ** -26])
    big = np.float32([2 ** 23 - 0.5, 2 ** 23 + 1, 2 ** 22 + 0.5, -(2 ** 22 + 0.5), -(2 ** 23 - 0.5), 2 ** 24 + 2, 2147483520.0, -2147483520.0,
                      2 ** 31, -2 ** 31, -2147483904.0, 3e38, -3e38, np.inf, -np.inf, np.nan, 4194303.5, -4194303.5, 8388607.5, -8388607.5])
    rnd = (r.standard_normal(400000) * np.exp(r.uniform(-25, 25, 400000))).astype(np.float32)
    x = np.concatenate([h, np.nextafter(h, np.float32(np.inf)), np.nextafter(h, np.float32(-np.inf)), tiny, big, rnd, -rnd])
    with np.errstate(all='ignore'):
        for mode in (1, 2, 3, 4, 5):
            want = oracle.linear_quant_t(x, np.float32(1.0), 0, -2 ** 31, 2 ** 31 - 1, mode, return_int=True)[1].astype(np.int64)
            got = dev_round(x, mode)
            bad = np.flatnonzero(want != got)
            assert bad.size == 0, (mode, x[bad[:4]], want[bad[:4]], got[bad[:4]])


def fp_fast_twin(x, s, E, M, cmin, cmax):
    """FloatOp<HALF_EVEN, FAST>::grid + dequant with offset 0 in numpy: bit for bit what ops.cuh does."""
    u = (x / np.float32(s)).astype(np.float32)
    emin, emax = -(1 << (E - 1)) + 1, 1 << (E - 1)
    top = (~(0x007FFFFF >> M)) & 0x007FFFFF
    tmax = np.array([((emax + 127) << 23) + top], np.uint32).view(np.float32)[0]
    hi, lo = np.float32(min(cmax, tmax)), np.float32(max(cmin, -tmax))
    k = (1 << (E - 1)) + M - 2
    magic = np.array([((127 + 23 - k) << 23) | 0x00400000], np.uint32).view(np.float32)[0]
    thresh = np.array([(emin + 1 + 127) << 23], np.uint32).view(np.float32)[0]
    half_minus1, keep = np.uint32((1 << (22 - M)) - 1), np.uint32((~((1 << (23 - M)) - 1)) & 0xFFFFFFFF)
    nan = np.isnan(u)
    uc = np.minimum(np.maximum(u, lo), hi)
    uc_bits = np.where(nan, np.uint32(0x7FFFFFFF), uc.view(np.uint32))    # min.NaN / max.NaN return the canonical NaN
    nb = ((uc_bits.astype(np.uint64) + half_minus1) & 0xFFFFFFFF).astype(np.uint32) & keep
    sub = ((uc + magic).astype(np.float32) - magic).astype(np.float32)
    q = np.where(np.abs(uc) < thresh, sub, nb.view(np.float32))
    q = np.where(nan, nb.view(np.float32), q)
    return (q * np.float32(s)).astype(np.float32)


def test_fp8_fast_path_twin_equals_the_reference_algorithm(oracle):
    r = np.random.RandomState(11)
    x = (r.standard_normal(300000) * np.exp(r.uniform(-12, 8, 300000))).astype(np.float32)
    x[::3] = x[::3].astype(np.float16).astype(np.float32)                  # tie-rich
    sp = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, 464.0, 480.0, 448.0, 1.1875, 1.4375, 2.375, 19.0, -1.1875, 1.5 * 2 ** -9,
                     2.5 * 2 ** -9, 2 ** -10, -2 ** -11, 2 ** -6, 2 ** -6 * (1 - 2 ** -24), 3e38, -3e38, 57344.0, 61440.0, 65504.0])
    x[:sp.size] = sp
    with np.errstate(all='ignore'):
        for (E, M, cmin, cmax) in ((4, 3, -448.0, 448.0), (5, 2, -57344.0, 57344.0), (4, 3, -240.0, 240.0), (5, 10, -65504.0, 65504.0), (3, 4, -30.0, 30.0)):
            for s in (1.0, 0.125, 4.0, 0.3):
                want = oracle.float_quant_t(x, np.float32(s), 0.0, E, M, cmin, cmax, 0)
                got = fp_fast_twin(x, s, E, M, cmin, cmax)
                bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
                assert bad.size == 0, (E, M, s, x[bad[:4]], got[bad[:4]], want[bad[:4]])


def test_radix_select_raw_prefix_filter_has_no_false_negatives():
    """select.cu passes 1-2 reject elements on the raw bits before computing the order-preserving key.  Twin of order_key / raw_of / hit:
    every element whose key matches a chosen prefix must pass the filter (false positives are allowed: the exact test follows)."""
    r = np.random.RandomState(5)
    b = r.randint(0, 2 ** 32, size=400000, dtype=np.uint64).astype(np.uint32)
    b[:8] = np.uint32([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x00000001, 0x80000001])
    bz = np.where(b == 0x80000000, np.uint32(0), b)                       # -0.0 shares +0.0's key
    key = np.where(bz & 0x80000000, ~bz, bz | np.uint32(0x80000000)).astype(np.uint32)
    for pmask in (np.uint32(0xFFE00000), np.uint32(0xFFFFFC00)):
        prefixes = [np.uint32(0x80000000), np.uint32(0x7FFFFFFF) & pmask,      # the bucket of +0 (takes -0.0 too) and the bucket just below it
                    key[17] & pmask, key[99] & pmask, key[12345] & pmask, key[5] & pmask, key[1] & pmask]
        for p0 in prefixes:
            for p1 in (prefixes[0], prefixes[2], p0):
                def raw_of(p): return (p & np.uint32(0x7FFFFFFF)) if (p & 0x80000000) else (~p & pmask)
                c0, c1 = raw_of(p0), raw_of(p1)
                c2 = np.uint32(0x80000000) if (p0 == 0x80000000 or p1 == 0x80000000) else c0
                t = b & pmask
                hit = (t == c0) | (t == c1) | (t == c2)
                exact = ((key & pmask) == p0) | ((key & pmask) == p1)
                assert not np.any(exact & ~hit), (hex(int(pmask)), hex(int(p0)), hex(int(p1)))
                assert (hit & ~exact).sum() <= 2 + (b == 0x80000000).sum() + ((b & pmask) == 0x80000000).sum()      # only the -0.0 pattern's bucket


def test_raw_bit_float_atomics_give_min_and_max_for_mixed_signs():
    """common.cuh atomic_{max,min}_float: non-negative patterns go through a signed-int atomic, negative ones through an unsigned atomic
    of the opposite sense; the slot starts at -inf / +inf; NaN is injected as +NaN (max slot) / -NaN (min slot) and must win.  Twin on
    Python ints, any arrival order."""
    def as_int(u): return u - (1 << 32) if u & 0x80000000 else u
    def atomic_max_float(slot, u):          # slot, u: raw uint32 patterns
        if not (u >> 31): return max(as_int(slot), as_int(u)) & 0xFFFFFFFF        # atomicMax(int*)
        return min(slot, u)                                                      # atomicMin(unsigned*)
    def atomic_min_float(slot, u):
        if not (u >> 31): return min(as_int(slot), as_int(u)) & 0xFFFFFFFF        # atomicMin(int*)
        return max(slot, u)                                                      # atomicMax(unsigned*)
    r = np.random.RandomState(3)
    for it in range(300):
        n = int(r.randint(1, 40))
        kind = it % 5
        v = (r.standard_normal(n) * 10.0 ** r.uniform(-3, 3)).astype(np.float32)
        if kind == 1: v = np.abs(v)
        if kind == 2: v = -np.abs(v)
        if kind == 3: v[r.randint(n)] = np.float32(-0.0); v[r.randint(n)] = np.float32(0.0)
        if kind == 4: v[:] = np.float32(r.choice([-0.0, 0.0, np.inf, -np.inf, 1e-45, -1e-45]))
        hi, lo = 0xFF800000, 0x7F800000                                          # minmax_init_kernel: max = -inf, min = +inf
        for u in v.view(np.uint32).tolist():
            hi, lo = atomic_max_float(hi, u), atomic_min_float(lo, u)
        got_hi, got_lo = np.array([hi], np.uint32).view(np.float32)[0], np.array([lo], np.uint32).view(np.float32)[0]
        assert got_hi == v.max() and got_lo == v.min(), (it, v, got_lo, got_hi)   # value equality (either zero may represent 0)
        # NaN poisoning: whatever came before or comes after, the slot ends up NaN
        order = r.permutation(n + 1)
        hi, lo = 0xFF800000, 0x7F800000
        for j in order:
            if j == n: hi, lo = atomic_max_float(hi, 0x7FC00000), atomic_min_float(lo, 0xFFC00000)
            else:
                u = int(v.view(np.uint32)[j]); hi, lo = atomic_max_float(hi, u), atomic_min_float(lo, u)
        assert hi == 0x7FC00000 and lo == 0xFFC00000, (it, hex(hi), hex(lo))


def test_histogram_slot_arithmetic_twin(oracle):
    """collectors.cu SymBin / AsymBin: slot = saturating floor of the fp32 quotient, then ONE unsigned min against `bins` (clip: everything
    out of range, negative wrap-around included, lands in the trash slot) or a clamp to the last bin (no clip) -- against the oracle's
    restatement of the reference's branches (sort.cu:75-89, 113-139)."""
    r = np.random.RandomState(13)
    x = (r.standard_normal(200000) * np.exp(r.uniform(-3, 3, 200000))).astype(np.float32)
    x[:10] = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 3e38, -3e38, 1.0])
    with np.errstate(all='ignore'):
        def floor_sat(t):
            t = np.where(np.isnan(t), 0.0, np.floor(t.astype(np.float64)))
            return np.clip(t, -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)
        for bins in (50, 2048, 4096):
            for hs in (np.float32(0.001), np.float32(0.37), np.float32(x[np.isfinite(x)].max() / bins)):
                for clip in (True, False):
                    b = floor_sat((np.abs(x) / hs).astype(np.float32))
                    slot = np.minimum(b & 0xFFFFFFFF, bins) if clip else np.minimum(b, bins - 1)
                    got = np.bincount(slot[slot < bins], minlength=bins).astype(np.int32)
                    assert np.array_equal(got, oracle.histogram_t(x, hs, bins, clip)), ('sym', bins, float(hs), clip)
            for (vmin, vmax) in ((np.float32(-2.5), np.float32(3.0)), (np.float32(0.0), np.float32(10.0))):
                for clip in (True, False):
                    hs = ((vmax - vmin) / np.float32(bins)).astype(np.float32)                       # fp32, like the kernel
                    b = floor_sat(((x - vmin).astype(np.float32) / hs).astype(np.float32))
                    slot = np.minimum(b & 0xFFFFFFFF, bins) if clip else np.maximum(np.minimum(b, bins - 1), 0)
                    got = np.bincount(slot[slot < bins], minlength=bins).astype(np.int32)
                    assert np.array_equal(got, oracle.histogram_asym_t(x, vmin, vmax, bins, clip)), ('asym', bins, float(vmin), float(vmax), clip)


def test_multi_tensor_span_partitions_cover_every_element_exactly_once():
    """Index twins of the two multi-tensor kernels: (1) multi_histogram_t_kernel / multi_minmax (collectors.cu) give each CTA a contiguous
    span of the concatenated tensors and round the cut points inside a tensor up to a multiple of 4 elements on BOTH sides; (2)
    multi_channel_kernel (fakequant.cu) splits the concatenation of 512-element warp segments.  Every element of every tensor must be
    visited exactly once, whatever the sizes."""
    r = np.random.RandomState(17)
    for it in range(200):
        T = int(r.randint(1, 12))
        ns = [int(r.choice([1, 2, 3, 5, 511, 512, 513, 4096, 70001, int(r.randint(1, 200000))])) for _ in range(T)]
        grid = int(r.choice([1, 2, 7, 148, 1184]))
        # ---- (1) element spans
        prefix = np.concatenate([[0], np.cumsum(ns)])
        total = int(prefix[-1])
        span = -(-total // grid); span = (span + 3) & ~3
        seen = [np.zeros(n, np.int32) for n in ns]
        for cta in range(grid):
            s0 = cta * span; s1 = min(s0 + span, total)
            if s0 >= total: continue
            t = int(np.searchsorted(prefix, s0, side='right') - 1); t = min(t, T - 1)
            while t < T and prefix[t] < s1:
                n = ns[t]
                a = max(s0 - int(prefix[t]), 0); b = min(s1 - int(prefix[t]), n)
                a = min((a + 3) & ~3, n)
                if b < n: b = (b + 3) & ~3
                b = min(b, n)
                if b > a: seen[t][a:b] += 1
                t += 1
        assert all((s == 1).all() for s in seen), (it, ns, grid)
        # ---- (2) segment spans, 8 warps per CTA, 32 lanes x 4 vectors (or groups) of 4 elements per segment
        segs = [(-(-n // 512)) if n > 0 else 0 for n in ns]
        sp = np.concatenate([[0], np.cumsum(segs)]); tot = int(sp[-1])
        span = -(-tot // grid)
        seen = [np.zeros(n, np.int32) for n in ns]
        for cta in range(grid):
            s0 = cta * span; s1 = min(s0 + span, tot)
            if s0 >= tot: continue
            t = int(np.searchsorted(sp, s0, side='right') - 1); t = min(t, T - 1)
            while t < T and sp[t] < s1:
                first, nseg = int(sp[t]), segs[t]
                if nseg:
                    a = max(s0 - first, 0); b = min(s1 - first, nseg)
                    n = ns[t]
                    for warp in range(8):
                        for sg in range(a + warp, b, 8):
                            g = sg * 128 + np.arange(128)                          # the 32 x 4 vector / group indices of this segment
                            e0 = g * 4
                            for k in range(4):
                                idx = e0 + k
                                idx = idx[idx < n]
                                seen[t][idx] += 1
                t += 1
        assert all((s == 1).all() for s in seen), (it, ns, grid)


def test_sampled_thresholds_contain_the_wanted_order_statistics():
    """select.cu, "self-speculation": a cold Quantile_T on >= 8 Mi elements reads one element per stride window (hashed offset), takes the j-th largest
    / smallest of the 16384 samples as thresholds (j = max(12, 3 x need x m / n)) and compacts what lies at or beyond them, counting copies of the
    threshold key itself instead of storing them.  Twin of that rule on the CPU: for bell-shaped, post-ReLU, clipped and heavy-tailed data the
    candidates always contain the `need` wanted elements and the stored ones fit the 256 Ki-key buffer -- i.e. the tensor is read once; for a sample
    that lies (values planted exactly where the sampler looks) the verdict must be "failed", never a wrong selection."""
    m, cap = 16384, 1 << 18
    n = (1 << 23) + 4099
    stride = n // m
    i = np.arange(m, dtype=np.uint64)
    pos = (i * np.uint64(stride) + ((i * np.uint64(0x9E3779B1)) % np.uint64(1 << 32)) % np.uint64(stride)).astype(np.int64)
    assert pos.max() < n and np.all(np.diff(pos) > 0) and np.all(pos // stride == np.arange(m))     # one sample per window, inside the tensor

    def rank_from_end(need): return max(12, -(-3 * need * m // n))
    def rank_ok(j): return j <= m // 4 and 3 * j * (n // m) <= 2 * cap

    def verdicts(x, q):
        r0 = int(min(max(np.rint(np.float32(n) * np.float32(q)), 0), n - 1)); r1 = int(min(max(np.rint(np.float32(n) * (np.float32(1) - np.float32(q))), 0), n - 1))
        need_hi, need_lo = n - r0, r1 + 1
        s = np.sort(x[pos])
        out = []
        for need, side in ((need_hi, 'hi'), (need_lo, 'lo')):
            j = rank_from_end(need)
            if not rank_ok(j): out.append(None); continue
            g = s[m - j] if side == 'hi' else s[j - 1]
            beyond = (x >= g) if side == 'hi' else (x <= g)
            eq = int(np.count_nonzero(x == g)); stored = int(np.count_nonzero(beyond)) - eq
            out.append((stored <= cap and stored + eq >= need, stored, eq, need))
        return out

    rng = np.random.default_rng(5)
    base = rng.standard_normal(n, dtype=np.float32) * 2
    well_behaved = {'randn': base, 'relu': np.maximum(base, 0), 'relu6-like': np.clip(base, 0, 1.5), 'student-t(2)': rng.standard_t(2, n).astype(np.float32)}
    for name, x in well_behaved.items():
        for q in (0.9999, 0.99999, 0.999):
            for v in verdicts(x, q):
                assert v is not None and v[0], (name, q, v)
                assert v[1] <= 8 * max(v[3], 12 * stride), (name, q, v)                       # and not wastefully many: the finish walks them
    # q = 0.99 on 8 Mi elements wants 84 K elements per tail: more than the buffer is allowed to hold on average -> no speculation at all
    assert all(v is None for v in verdicts(base, 0.99))
    lied = base.copy(); lied[pos[:64]] = 1e6; lied[pos[64:128]] = -1e6
    for v in verdicts(lied, 0.9999): assert v is not None and not v[0] and v[1] + v[2] < v[3]   # too few candidates: the regular passes take over
    flat = np.maximum(base, 0); flat[pos] = 3.0
    hi, lo = verdicts(flat, 0.9999)
    assert not hi[0] and hi[1] > cap and not lo[0]                                           # too many: overflow is detected, the buffer handed back
