"""Every kernel family past 2^31 and 2^32 elements, held to sub-range launches and to the C oracle.

Most bindings take any int64 numel (SIZE_CLASS below; tests/test_cpu_large_counts.py checks the table against the CheckSize calls of the
binding sources).  Each case here builds one tensor (or table) across the 2^31 / 2^32 element boundaries and checks every launch twice:
  (a) the whole output or statistic against launches of the same entry point on sub-ranges below 2^31 elements -- sizes the rest of the
      suite already holds to the oracle on every route -- combined exactly (outputs concatenated, min/max folded, histograms summed in int64
      and reduced modulo 2^32 like the int32 bins, order statistics from exact multiplicities);
  (b) the C oracle on host windows of a few thousand elements around every planted index and at 64 seeded random places, bit for bit.

The data is a hash of the 64-bit element index, generated on the device in chunks of 2^26 elements; `host_values` regenerates any window on
the host.  Every case states the bytes it needs and skips when the card has less free memory than that plus 2 GB; the largest needs ~18 GB.
"""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

B31, B32 = 1 << 31, 1 << 32
CHUNK = 1 << 26                                                # device generation step (one int64 index temporary = 512 MB)
SUB = 1 << 28                                                  # sub-range launches
GB = 1 << 30
M32 = 0xFFFFFFFF
K1, K2 = 0x5BD1E995, 0x27D4EB2D                                # both < 2^31: every product stays below 2^63 in int64
WIN = 4096

# Size class of every launching binding: 'refuses' raises "too many element" above 2^31 - 1 elements (CheckSize), 'int64' takes any numel.
REFUSES = {'QuantizeTensor_LT', 'QuantizeTensor_LC', 'QuantizeTensor_toInt', 'QuantizeTensor_LT_Half', 'QuantizeTensor_LC_Half',
           'QuantizeTensor_FT_Half', 'QuantizeTensor_FC_Half', 'QuantizeTensor_LT_B', 'QuantizeTensor_LC_B', 'QuantizeTensor_FT_B',
           'QuantizeTensor_FC_B', 'TensorClip_T', 'TensorClip_C', 'RoundingLoss_LT', 'RoundingLoss_LC', 'RoundingLoss_LT_B', 'RoundingLoss_LC_B'}
INT64 = {'QuantizeTensor_FT', 'QuantizeTensor_FC', 'MinMax_T', 'MinMax_C', 'MinMax_Init', 'Histogram_T', 'Histogram_Asymmetric_T',
         'Histogram_Asymmetric_T_Half', 'Histogram_C', 'Histogram_T_DeviceScale', 'Quantile_T', 'Quantile_T_Guess', 'Quantile_T_Half',
         'Isotone_T', 'Quantile_Guess_Init', 'Multi_MinMax_T', 'Multi_MinMax_T_Half', 'Multi_Histogram_T', 'Multi_Histogram_T_Half',
         'Multi_Quantile_T', 'Multi_Quantile_T_Half', 'Multi_QuantizeTensor_LT', 'Multi_QuantizeTensor_LC', 'Multi_QuantizeTensor_LC_Half',
         'Multi_Paired_Moments', 'MinMax_To_Scale_Offset', 'Hist_Scale_From_MinMax', 'KL_Search', 'MSE_Search'}
SIZE_CLASS = {**{k: 'refuses' for k in REFUSES}, **{k: 'int64' for k in INT64}}


# ---------------------------------------------------------------------------------------------------------------- data
def hash_of(idx):
    """32-bit hash of the int64 element index; the same expression for torch and numpy int64 arrays (no product reaches 2^63)."""
    a = (idx ^ (idx >> 32)) & M32
    a = (a * K1) & M32
    a = a ^ (a >> 15)
    a = (a * K2) & M32
    return a ^ (a >> 13)


# kind -> (code mask, code -> value): 'f32' 65536 values k / 4096 in [-8, 8); 'b16' 512 values k / 16 in [-16, 16) (exact in bf16);
# 'relu' the b16 values clamped at 0 (257 of 512 codes are zero); 'near1' bf16 bit patterns 1.0 +- 1..7 ulps (never 1.0 itself).
KINDS = {'f32': 0xFFFF, 'b16': 0x1FF, 'relu': 0x1FF, 'near1': None}


def code_value(kind, c):
    """Value of code(s) c (numpy or python ints) as float64."""
    c = np.asarray(c, np.int64)
    if kind == 'f32': return (c - 32768) / 4096.0
    if kind == 'b16': return (c - 256) / 16.0
    if kind == 'relu': return np.maximum(c - 256, 0) / 16.0
    j = c % 14
    j = np.where(j < 7, j - 7, j - 6)
    return (np.int32(0x3F80) + j).astype(np.int32).__lshift__(16).view(np.float32).astype(np.float64)


def values_torch(kind, h):
    if kind == 'f32': return ((h & 0xFFFF) - 32768).float() * (1.0 / 4096)
    if kind == 'b16': return ((h & 0x1FF) - 256).float() * (1.0 / 16)
    if kind == 'relu': return ((h & 0x1FF) - 256).clamp_min(0).float() * (1.0 / 16)
    j = h % 14
    j = torch.where(j < 7, j - 7, j - 6)
    return ((j + 0x3F80) << 16).to(torch.int32).view(torch.float32)


def values_np(kind, h):
    if kind == 'near1': return code_value(kind, h).astype(np.float32)
    return code_value(kind, h & KINDS[kind]).astype(np.float32)


def fill(n, kind, dtype, plants=(), device='cuda'):
    x = torch.empty(n, dtype=dtype, device=device)
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        x[a:b] = values_torch(kind, hash_of(torch.arange(a, b, dtype=torch.int64, device=device))).to(dtype)
    for i, v in plants:
        x[i:i + 1].fill_(v)
    return x


def host_values(kind, a, b, plants=(), dtype=torch.float32):
    """The host twin of fill() on [a, b): fp32 values (bf16 kinds are exact in fp32)."""
    x = values_np(kind, hash_of(np.arange(a, b, dtype=np.int64)))
    for i, v in plants:
        if a <= i < b: x[i - a] = np.float32(v)
    return x


def counts_of(kind, n, plants=()):
    """{value: multiplicity} of fill(n, kind, plants), counted on the device in int64 (torch.bincount of the codes)."""
    mask = KINDS[kind] if kind != 'near1' else None
    bins = (mask + 1) if mask is not None else 14
    cnt = torch.zeros(bins, dtype=torch.int64, device='cuda')
    for a in range(0, n, CHUNK):
        h = hash_of(torch.arange(a, min(n, a + CHUNK), dtype=torch.int64, device='cuda'))
        cnt += torch.bincount(h & mask if mask is not None else h % 14, minlength=bins)
    cnt = cnt.cpu().numpy()
    out = {}
    for c in np.nonzero(cnt)[0]:
        v = float(code_value(kind, c))
        out[v] = out.get(v, 0) + int(cnt[c])
    for i, v in plants:
        hv = int(hash_of(np.int64(i)))
        old = float(code_value(kind, hv & mask if mask is not None else hv))
        out[old] -= 1
        out[float(np.float32(v))] = out.get(float(np.float32(v)), 0) + 1
    return out


def order_stat(counts, rank):
    """Element of 0-based ascending rank `rank` of the multiset {value: multiplicity}."""
    run = 0
    for v in sorted(counts):
        run += counts[v]
        if rank < run: return v
    raise AssertionError('rank past the multiset')


def ranks(n, q):
    """_Quantile_T's two ranks, as tests/test_cpu_large_counts.py states them."""
    from test_cpu_large_counts import rank_formula
    return rank_formula(n, q), rank_formula(n, float(np.float32(1) - np.float32(q)))


def boundary_indices(n, row=1):
    """The planted places: 0, 2^31 - 1, 2^31, 2^32 (where n allows), the row boundaries next to them, and n - 1."""
    out = {0, n - 1}
    for b in (B31 - 1, B31, B32):
        for i in (b, b // row * row, b // row * row - 1, (b // row + 1) * row):
            if 0 <= i < n: out.add(i)
    return sorted(out)


def windows(n, seed, row=1, plants=()):
    """[a, b) host windows of ~WIN elements (whole rows) around every boundary / planted index and at 64 seeded random places."""
    r = np.random.RandomState(seed)
    centres = boundary_indices(n, row) + [i for i, _ in plants] + [int(v) for v in r.randint(0, n, 64, dtype=np.int64)]
    w = max(1, WIN // row)
    out = set()
    for c in centres:
        a = max(0, c // row - w // 2) * row
        out.add((a, min(n, a + w * row)))
    return sorted(out)


def bits(a):
    a = a.detach().cpu() if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    if a.dtype in (torch.float32, torch.int32): return a.view(torch.int32).numpy()
    if a.dtype in (torch.bfloat16, torch.float16): return a.view(torch.int16).numpy()
    return a.numpy()


def to_bf16_bits(y32):
    return bits(torch.from_numpy(np.ascontiguousarray(y32, np.float32)).to(torch.bfloat16))


def need(nbytes):
    """Skip unless the card has `nbytes` free plus 2 GB."""
    gc.collect(); torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + 2 * GB:
        pytest.skip(f'needs {nbytes / GB:.1f} GB + 2 GB free, the card has {free / GB:.1f} GB')


@pytest.fixture(autouse=True)
def release():
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize(); torch.cuda.empty_cache()


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


def t1(v):
    return torch.tensor([v], dtype=torch.float32, device='cuda')


def assert_sub_ranges(y, x, launch, rows=None):
    """(a) for element-wise outputs: y equals launch() on every sub-range (whole rows of a [B, ...] tensor when rows is set)."""
    if rows is None:
        for a in range(0, x.numel(), SUB):
            b = min(x.numel(), a + SUB)
            assert np.array_equal(bits(y[a:b]), bits(launch(x[a:b]))), f'sub-range [{a}, {b})'
    else:
        step = max(1, SUB // rows)
        for a in range(0, x.shape[0], step):
            b = min(x.shape[0], a + step)
            assert np.array_equal(bits(y[a:b]), bits(launch(x[a:b]))), f'rows [{a}, {b})'


# ---------------------------------------------------------------------------------------------------------------- element-wise above 2^31
FT_CASES = [(0, 448.0, 'fast'), (1, 448.0, 'fast'), (0, 300.0, 'general'), (4, 300.0, 'general')]   # (rounding, clip, float path)


@pytest.mark.parametrize('mode,clip,path', FT_CASES, ids=[f'mode{m}-{p}' for m, _, p in FT_CASES])
def test_float_quant_t_above_2_31(ext, oracle, mode, clip, path):
    n = B31 + 5
    need(2 * 4 * n + 2 * 4 * SUB)
    plants = [(i, 447.75 - (k % 3) * 0.0625) for k, i in enumerate(boundary_indices(n))]
    x = fill(n, 'f32', torch.float32, plants)
    s, o = t1(0.0078125), t1(0.0)
    launch = lambda v: ext.QuantizeTensor_FT(v, s, o, 4, 3, -clip, clip, mode)
    y = launch(x)
    assert_sub_ranges(y, x, launch)
    for a, b in windows(n, 1, plants=plants):
        xw = host_values('f32', a, b, plants)
        assert np.array_equal(bits(y[a:b]), bits(oracle.float_quant_t(xw, 0.0078125, 0.0, 4, 3, -clip, clip, mode))), (a, b)


# (shape of one row block [C, epc], channel axis) per launch_channel route at n > 2^31: epc % 4 == 0 (vec kernel), epc 9 (generic kernel),
# epc 1 with C % 4 == 0 (channel-last kernel)
FC_ROUTES = {'vec': ((8, 4096), 1), 'generic': ((16, 9), 1), 'channel_last': ((64,), 1)}


def channel_tensor(route, kind='f32', dtype=torch.float32, limit=None, above=B31):
    """Whole row blocks: the most that fit in `limit` elements, or else the fewest that hold more than `above` elements."""
    row, axis = FC_ROUTES[route]
    per = int(np.prod(row))
    B = (limit // per) if limit else above // per + 1
    n = B * per
    C = row[0]
    return n, (B,) + row, axis, C, per


@pytest.mark.parametrize('route', sorted(FC_ROUTES))
def test_float_quant_c_above_2_31(ext, oracle, route):
    n, shape, axis, C, per = channel_tensor(route)
    need(2 * 4 * n + 2 * 4 * SUB)
    plants = [(i, -447.5 + (k % 2) * 0.25) for k, i in enumerate(boundary_indices(n, per))]
    x = fill(n, 'f32', torch.float32, plants).view(shape)
    sc = (torch.arange(C, dtype=torch.float32) % 5 + 1) * 0.0078125
    s, o = sc.cuda(), torch.zeros(C, device='cuda')
    launch = lambda v: ext.QuantizeTensor_FC(v, s, o, 4, 3, -448.0, 448.0, axis, 0)
    y = launch(x)
    assert_sub_ranges(y, x, launch, rows=per)
    yf = y.view(-1)
    for a, b in windows(n, 2, per, plants):
        xw = host_values('f32', a, b, plants).reshape((-1,) + shape[1:])
        assert np.array_equal(bits(yf[a:b]), bits(oracle.float_quant_c(xw, sc.numpy(), np.zeros(C, np.float32), axis)).reshape(-1)), (a, b)


@pytest.fixture(scope='module')
def cabi():
    import ctypes
    import os
    from conftest import ROOT
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    lib = ctypes.CDLL(os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so'))
    V, I, L = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    sig = {'ppq_b200_linear_quant_t': [V, V, L, V, V, I, I, I, V],
           'ppq_b200_linear_quant_c': [V, V, L, L, I, V, V, I, I, I, V],
           'ppq_b200_linear_quant_t_toint': [V, V, I, L, V, V, I, I, I, V],
           'ppq_b200_float_quant_t': [V, V, L, V, V, I, I, ctypes.c_float, ctypes.c_float, I, V]}
    for name, args in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, ctypes.c_int
    return lib


def test_linear_quant_c_abi_above_2_31(ext, cabi, oracle):
    """The C ABI takes int64 n and does not refuse: per-tensor, per-channel and int8 output past 2^31, against the binding on sub-ranges."""
    n = B31 + 5
    need(4 * n + 4 * n + 4 * SUB)
    plants = [(i, 1000.0 if k % 2 else -1000.0) for k, i in enumerate(boundary_indices(n))]
    x = fill(n, 'f32', torch.float32, plants)
    s, o = t1(0.03125), t1(3.0)
    st = torch.cuda.current_stream().cuda_stream
    y = torch.empty_like(x)
    assert cabi.ppq_b200_linear_quant_t(x.data_ptr(), y.data_ptr(), n, s.data_ptr(), o.data_ptr(), -128, 127, 0, st) == 0
    assert_sub_ranges(y, x, lambda v: ext.QuantizeTensor_LT(v, s, o, -128, 127, 0))
    for a, b in windows(n, 3, plants=plants):
        assert np.array_equal(bits(y[a:b]), bits(oracle.linear_quant_t(host_values('f32', a, b, plants), 0.03125, 3.0, -128, 127, 0))), (a, b)
    del y
    q = torch.empty(n, dtype=torch.int8, device='cuda')
    assert cabi.ppq_b200_linear_quant_t_toint(x.data_ptr(), q.data_ptr(), 8, n, s.data_ptr(), o.data_ptr(), -128, 127, 0, st) == 0
    assert_sub_ranges(q, x, lambda v: ext.QuantizeTensor_toInt(v, s, o, -128, 127, -1000, 0, 8))
    for a, b in windows(n, 4, plants=plants):
        _, qi = oracle.linear_quant_t(host_values('f32', a, b, plants), 0.03125, 3.0, -128, 127, 0, return_int=True)
        assert np.array_equal(q[a:b].cpu().numpy(), qi.astype(np.int8)), (a, b)
    del q
    _, shape, axis, C, per = channel_tensor('vec')
    assert shape[0] * per >= n
    B = n // per
    xc = x[:B * per].view((B,) + shape[1:])
    sc = (torch.arange(C, dtype=torch.float32) + 1) * 0.015625
    s2, o2 = sc.cuda(), torch.zeros(C, device='cuda')
    yc = torch.empty_like(xc)
    assert cabi.ppq_b200_linear_quant_c(xc.data_ptr(), yc.data_ptr(), xc.numel(), per // C, C, s2.data_ptr(), o2.data_ptr(), -128, 127, 0, st) == 0
    assert_sub_ranges(yc, xc, lambda v: ext.QuantizeTensor_LC(v, s2, o2, -128, 127, axis, 0), rows=per)
    for a, b in windows(xc.numel(), 5, per):
        xw = host_values('f32', a, b, plants).reshape((-1,) + shape[1:])
        want = oracle.linear_quant_c(xw, sc.numpy(), np.zeros(C, np.float32), axis, -128, 127, 0)
        assert np.array_equal(bits(yc.view(-1)[a:b]), bits(want).reshape(-1)), (a, b)


def test_float_quant_t_abi_in_place_above_2_32(ext, cabi, oracle):
    """2^32 + 5 fp32 elements quantised in place through the C ABI (an element-wise kernel reads each element before it writes it):
    every chunk against the binding on the regenerated chunk, and the oracle on host windows."""
    n = B32 + 5
    need(4 * n + 3 * 4 * CHUNK)
    plants = [(i, 300.0 + k) for k, i in enumerate(boundary_indices(n))]
    x = fill(n, 'f32', torch.float32, plants)
    s, o = t1(0.015625), t1(0.0)
    st = torch.cuda.current_stream().cuda_stream
    assert cabi.ppq_b200_float_quant_t(x.data_ptr(), x.data_ptr(), n, s.data_ptr(), o.data_ptr(), 4, 3, -448.0, 448.0, 0, st) == 0
    for a in range(0, n, CHUNK):
        b = min(n, a + CHUNK)
        src = values_torch('f32', hash_of(torch.arange(a, b, dtype=torch.int64, device='cuda')))
        for i, v in plants:
            if a <= i < b: src[i - a] = v
        assert np.array_equal(bits(x[a:b]), bits(ext.QuantizeTensor_FT(src, s, o, 4, 3, -448.0, 448.0, 0))), (a, b)
    for a, b in windows(n, 10, plants=plants):
        assert np.array_equal(bits(x[a:b]), bits(oracle.float_quant_t(host_values('f32', a, b, plants), 0.015625, 0.0, 4, 3, -448.0, 448.0, 0))), (a, b)


# ---------------------------------------------------------------------------------------------------------------- half at the largest n
def test_half_fake_quant_at_largest_accepted_n(ext, oracle):
    """2^31 - 1 bf16 elements (per-channel: the largest multiple of the row below it): LT / FT / toInt / LC / FC _Half, sub-ranges and oracle."""
    n = B31 - 1
    need(2 * 2 * n + 4 * SUB)
    plants = [(i, 15.9375 if k % 2 else -16.0) for k, i in enumerate(boundary_indices(n))]
    x = fill(n, 'b16', torch.bfloat16, plants)
    s, o = t1(0.0625), t1(0.0)
    cases = [('LT', lambda v: ext.QuantizeTensor_LT_Half(v, s, o, -128, 127, 0),
              lambda xw: to_bf16_bits(oracle.linear_quant_t(xw, 0.0625, 0.0, -128, 127, 0))),
             ('FT', lambda v: ext.QuantizeTensor_FT_Half(v, s, o, 4, 3, -448.0, 448.0, 0),
              lambda xw: to_bf16_bits(oracle.float_quant_t(xw, 0.0625, 0.0, 4, 3, -448.0, 448.0, 0))),
             ('toInt', lambda v: ext.QuantizeTensor_toInt(v, s, o, -100, 100, -1000, 0, 8),
              lambda xw: oracle.linear_quant_t(xw, 0.0625, 0.0, -100, 100, 0, return_int=True)[1].astype(np.int8))]
    for name, launch, want in cases:
        y = launch(x)
        assert_sub_ranges(y, x, launch)
        for a, b in windows(n, 6, plants=plants):
            assert np.array_equal(bits(y[a:b]), want(host_values('b16', a, b, plants))), (name, a, b)
        del y
    _, shape, axis, C, per = channel_tensor('generic', limit=n)
    B = n // per
    xc = x[:B * per].view((B,) + shape[1:])
    sc = (torch.arange(C, dtype=torch.float32) % 3 + 1) * 0.0625
    s2, o2 = sc.cuda(), torch.zeros(C, device='cuda')
    cases = [('LC', lambda v: ext.QuantizeTensor_LC_Half(v, s2, o2, -128, 127, axis, 0),
              lambda xw: to_bf16_bits(oracle.linear_quant_c(xw, sc.numpy(), np.zeros(C, np.float32), axis, -128, 127, 0))),
             ('FC', lambda v: ext.QuantizeTensor_FC_Half(v, s2, o2, 4, 3, -448.0, 448.0, axis, 0),
              lambda xw: to_bf16_bits(oracle.float_quant_c(xw, sc.numpy(), np.zeros(C, np.float32), axis)))]
    for name, launch, want in cases:
        y = launch(xc)
        assert_sub_ranges(y, xc, launch, rows=per)
        for a, b in windows(xc.numel(), 7, per):
            xw = host_values('b16', a, b, plants).reshape((-1,) + shape[1:])
            assert np.array_equal(bits(y.view(-1)[a:b]), want(xw).reshape(-1)), (name, a, b)
        del y


# ---------------------------------------------------------------------------------------------------------------- collectors
def fold_minmax(parts):
    lo = min(p[0] for p in parts); hi = max(p[1] for p in parts)
    return lo, hi


def sub_minmax(ext, x):
    parts = []
    for a in range(0, x.numel(), SUB):
        mm = torch.tensor([float('inf'), float('-inf')], device='cuda')
        ext.MinMax_T(x[a:a + SUB], mm)
        lo, hi = torch.aminmax(x[a:a + SUB].float())
        assert mm.tolist() == [lo.item(), hi.item()], a
        parts.append(mm.tolist())
    return fold_minmax(parts)


def sub_hist(x, launch, bins, rows=None):
    """int64 sum of the sub-range histograms, reduced modulo 2^32 to int32 like the device bins."""
    acc = 0
    step = SUB if rows is None else max(1, SUB // rows)
    for a in range(0, x.shape[0], step):
        h = launch(x[a:a + step]).cpu().numpy().astype(np.int64)
        acc = acc + h
    return ((acc + B31) % B32 - B31).astype(np.int32)


def minmax_c_of(ext, xc, axis, C, step=None):
    """MinMax_C of xc in one launch, or folded by accumulating launches on `step` rows at a time."""
    lo, hi = torch.full((C,), float('inf'), device='cuda'), torch.full((C,), float('-inf'), device='cuda')
    for a in range(0, xc.shape[0], step or xc.shape[0]):
        ext.MinMax_C(xc[a:a + (step or xc.shape[0])], axis, lo, hi)
    return lo, hi


def check_collectors(ext, oracle, x, kind, plants, route, seed, past):
    n = x.numel()
    assert n > past
    mm = torch.tensor([float('inf'), float('-inf')], device='cuda')
    ext.MinMax_T(x, mm)
    assert tuple(mm.tolist()) == sub_minmax(ext, x)
    bins = 2048
    hs = t1(0.01)
    newh = lambda: torch.zeros(bins, dtype=torch.int32, device='cuda')
    launches = {'Histogram_T_DeviceScale': lambda v: (lambda h: (ext.Histogram_T_DeviceScale(v, hs, True, h), h)[1])(newh())}
    if x.dtype == torch.float32:
        launches['Histogram_T'] = lambda v: (lambda h: (ext.Histogram_T(v, 0.01, False, h), h)[1])(newh())
        launches['Histogram_Asymmetric_T'] = lambda v: (lambda h: (ext.Histogram_Asymmetric_T(-6.0, 7.5, v, True, h), h)[1])(newh())
    else:
        launches['Histogram_Asymmetric_T_Half'] = lambda v: (lambda h: (ext.Histogram_Asymmetric_T_Half(-6.0, 7.5, v, True, h), h)[1])(newh())
    for name, launch in launches.items():
        got = launch(x).cpu().numpy()
        assert np.array_equal(got, sub_hist(x, launch, bins)), name
    wins = windows(n, seed, plants=plants)
    for a, b in wins:
        xw = host_values(kind, a, b, plants)
        assert np.array_equal(bits(x[a:b].float()), bits(xw)), (a, b)
        lo, hi = oracle.minmax_t(xw)
        mw = torch.tensor([float('inf'), float('-inf')], device='cuda'); ext.MinMax_T(x[a:b], mw)
        assert mw.tolist() == [float(lo), float(hi)], (a, b)
        hw = torch.zeros(bins, dtype=torch.int32, device='cuda'); ext.Histogram_T_DeviceScale(x[a:b], hs, True, hw)
        assert np.array_equal(hw.cpu().numpy(), oracle.histogram_t(xw, np.float32(0.01), bins, True)), (a, b)
    # per channel, split at row boundaries
    nc, shape, axis, C, per = channel_tensor(route, limit=n)
    assert nc == n, 'the tensor is whole row blocks: every per-channel launch covers all of it'
    xc = x.view(shape)
    step = max(1, SUB // per)
    mins, maxs = minmax_c_of(ext, xc, axis, C)
    wl, wh = minmax_c_of(ext, xc, axis, C, step)                            # accumulating launches fold the sub-ranges
    assert np.array_equal(bits(mins), bits(wl)) and np.array_equal(bits(maxs), bits(wh))
    if x.dtype == torch.float32:
        hc = lambda v: (lambda h: (ext.Histogram_C(v, axis, 0.01, True, h), h)[1])(torch.zeros(C, 512, dtype=torch.int32, device='cuda'))
        assert np.array_equal(hc(xc).cpu().numpy(), sub_hist(xc, hc, 512, rows=per))
        for a, b in windows(xc.numel(), seed + 1, per):
            xw = host_values(kind, a, b, plants).reshape((-1,) + shape[1:])
            lo, hi = oracle.minmax_c(xw, axis)
            ml, mh = torch.full((C,), float('inf'), device='cuda'), torch.full((C,), float('-inf'), device='cuda')
            ext.MinMax_C(xc.view(-1)[a:b].view(xw.shape), axis, ml, mh)
            assert np.array_equal(bits(ml), bits(lo)) and np.array_equal(bits(mh), bits(hi)), (a, b)
    # a NaN at element `past` poisons both slots of the tensor and of its channel (the collectors' NaN rule, as torch.min / max):
    # the whole launch against the folded sub-range launches and torch.aminmax per chunk
    x[past:past + 1].fill_(float('nan'))
    mm = torch.tensor([float('inf'), float('-inf')], device='cuda'); ext.MinMax_T(x, mm)
    folded = torch.tensor([float('inf'), float('-inf')], device='cuda')
    for a in range(0, n, SUB):
        ext.MinMax_T(x[a:a + SUB], folded)
        lo, hi = torch.aminmax(x[a:a + SUB].float())
        assert (lo.isnan() and hi.isnan()) == (a <= past < a + SUB), a
    assert bool(mm.isnan().all()) and bool(folded.isnan().all())
    mins, maxs = minmax_c_of(ext, xc, axis, C)
    wl, wh = minmax_c_of(ext, xc, axis, C, step)
    ch = (past // (per // C)) % C
    for got, want in ((mins, wl), (maxs, wh)):
        nan = got.isnan().cpu().numpy()
        assert nan.tolist() == [c == ch for c in range(C)] and np.array_equal(nan, want.isnan().cpu().numpy())
        assert np.array_equal(bits(got)[~nan], bits(want)[~nan])


def test_collectors_fp32_above_2_31(ext, oracle):
    n = channel_tensor('generic', above=B31)[0]
    need(4 * n + GB)
    plants = [(i, v) for i, v in zip(boundary_indices(n), [9.5, -9.25, 12.0, -0.0, 8.5, -11.0, 10.0, -8.5, 0.0, 7.99])]
    x = fill(n, 'f32', torch.float32, plants)
    check_collectors(ext, oracle, x, 'f32', plants, 'generic', 8, B31)


def test_collectors_bf16_above_2_32(ext, oracle):
    n = channel_tensor('channel_last', above=B32)[0]
    need(2 * n + GB)
    plants = [(i, v) for i, v in zip(boundary_indices(n), [20.0, -24.0, 17.0, -0.0, 18.0, -20.0, 22.0, -17.0, 19.0, -18.0, 16.5, -16.5])]
    x = fill(n, 'b16', torch.bfloat16, plants)
    check_collectors(ext, oracle, x, 'b16', plants, 'channel_last', 9, B32)


def test_histogram_bin_wraps_modulo_2_32(ext):
    """int32 bins wrap like the reference's atomicAdd(int): 2^31 + 3 zeros land in bin 0 as -2^31 + 3."""
    n = B31 + 3
    need(4 * n)
    x = torch.zeros(n, device='cuda')
    h = torch.zeros(16, dtype=torch.int32, device='cuda')
    ext.Histogram_T(x, 0.5, True, h)
    assert h.tolist() == [-B31 + 3] + [0] * 15
    h2 = torch.zeros(16, dtype=torch.int32, device='cuda')
    ext.Histogram_T_DeviceScale(x, t1(0.5), True, h2)
    assert h2.tolist() == h.tolist()


# ---------------------------------------------------------------------------------------------------------------- select
QS = (0.9999, 0.999, 0.5)


def check_quantiles(got, counts, n, q, what):
    r0, r1 = ranks(n, q)
    want = [order_stat(counts, r0), order_stat(counts, r1)]
    assert got == want, f'{what} n={n} q={q}: {got} != {want} (ranks {r0}, {r1})'


@pytest.mark.parametrize('n', [B31 + 1, B31 + 8])
def test_quantile_t_fp32_above_2_31(ext, n):
    need(4 * n + GB)
    plants = [(i, v) for i, v in zip(boundary_indices(n), [100.0, -100.0, 99.5, -99.5, 98.0, -98.0])]
    x = fill(n, 'f32', torch.float32, plants)
    counts = counts_of('f32', n, plants)
    for q in QS:
        check_quantiles(ext.Quantile_T(x, q).tolist(), counts, n, q, 'Quantile_T')
    g = ext.Quantile_Guess_Init(1, x)
    for call in ('cold', 'warm'):
        check_quantiles(ext.Quantile_T_Guess(x, 0.9999, g).tolist(), counts, n, 0.9999, f'Quantile_T_Guess {call}')
    srt = sorted(counts)
    top = [v for v in reversed(srt) for _ in range(min(2, counts[v]))][:2]
    bot = [v for v in srt for _ in range(min(2, counts[v]))][:2]
    assert ext.Isotone_T(x).tolist() == top + bot


def test_quantile_t_half_above_2_32(ext):
    n = B32 + 100
    need(2 * n + GB)
    plants = [(i, v) for i, v in zip(boundary_indices(n), [30.0, -30.0, 29.0, -29.0, 28.0, -28.0, 27.0, -27.0])]
    x = fill(n, 'b16', torch.bfloat16, plants)
    counts = counts_of('b16', n, plants)
    for q in QS:
        check_quantiles(ext.Quantile_T_Half(x, q).tolist(), counts, n, q, 'Quantile_T_Half')
    g = ext.Quantile_Guess_Init(1, x)
    for call in ('cold', 'warm'):
        check_quantiles(ext.Quantile_T_Guess(x, 0.999, g).tolist(), counts, n, 0.999, f'Quantile_T_Guess bf16 {call}')


def test_quantile_post_relu_more_than_2_31_zeros_warm(ext):
    """Speculative path: > 2^31 zeros counted (not stored) as copies of last call's lower key 0."""
    n = B32 + 100
    need(2 * n + GB)
    x = fill(n, 'relu', torch.bfloat16)
    counts = counts_of('relu', n)
    assert counts[0.0] > B31
    g = ext.Quantile_Guess_Init(1, x)
    for call in ('cold', 'warm', 'warm again'):
        got = ext.Quantile_T_Guess(x, 0.9999, g).tolist()
        check_quantiles(got, counts, n, 0.9999, f'post-ReLU {call}')
        assert got[1] == 0.0


def test_quantile_warm_rank_past_more_than_2_31_counted_zeros(ext):
    """Speculative path: last call selected 0, so this call counts its ~2^31 + 429000 zeros without storing them, and the lower rank lands
    past them among 1000 positive subnormals that were stored.  The finish must add the counted copies to its digit counts in 64 bits."""
    n, q, sub = B32 + 100, 0.4999, 1000
    r0, r1 = ranks(n, q)
    zeros = r1 - 100
    assert zeros > B31 and r0 < zeros
    need(2 * n + GB)
    g = ext.Quantile_Guess_Init(1, t1(0.0))
    assert ext.Quantile_T_Guess(torch.zeros(4096, dtype=torch.bfloat16, device='cuda'), q, g).tolist() == [0.0, 0.0]
    x = torch.empty(n, dtype=torch.bfloat16, device='cuda')
    x[:zeros].zero_()
    x[zeros:zeros + sub].view(torch.int16).copy_(torch.arange(sub, device='cuda') % 7 + 1)   # bf16 bit patterns 0x0001-0x0007
    x[zeros + sub:].fill_(1.0)
    counts = {0.0: zeros, 1.0: n - zeros - sub}
    for j in range(1, 8):
        counts[float(np.array([j << 16], np.int32).view(np.float32)[0])] = len(range(j - 1, sub, 7))
    check_quantiles(ext.Quantile_T_Guess(x, q, g).tolist(), counts, n, q, 'counted zeros then subnormals')


def test_quantile_guess_with_every_element_past_threshold(ext):
    """Speculative path: a guess left by a constant tensor of 1.0 puts every element of a 2^32 + 2^20 bf16 tensor (1.0 +- 7 ulps, 900000
    exact 1.0) past both thresholds; the candidate count passes 2^32."""
    n = B32 + (1 << 20)
    ones = 900000
    need(2 * n + GB)
    g = ext.Quantile_Guess_Init(1, t1(0.0))
    prev = torch.ones(4096, dtype=torch.bfloat16, device='cuda')
    assert ext.Quantile_T_Guess(prev, 0.9999, g).tolist() == [1.0, 1.0]
    x = fill(n, 'near1', torch.bfloat16)
    x[:ones].fill_(1.0)
    counts = counts_of('near1', n, [])
    h = hash_of(np.arange(ones, dtype=np.int64))
    for v, c in zip(*np.unique(code_value('near1', h), return_counts=True)):
        counts[float(v)] -= int(c)
    counts[1.0] = counts.get(1.0, 0) + ones
    assert sum(counts.values()) == n
    check_quantiles(ext.Quantile_T_Guess(x, 0.9999, g).tolist(), counts, n, 0.9999, 'guess past every element')
    check_quantiles(ext.Quantile_T_Half(x, 0.9999).tolist(), counts, n, 0.9999, 'Quantile_T_Half')


# ---------------------------------------------------------------------------------------------------------------- tables
def table(tensors, slots=None):
    slots = slots or list(range(len(tensors)))
    return torch.tensor([(t.data_ptr(), t.numel(), s) for t, s in zip(tensors, slots)], dtype=torch.int64).cuda()


def table_sizes(total_past):
    """Sizes whose concatenation puts tensor 1 at offset 2^31 - 3 and lets the last tensor straddle `total_past` (2^31 or 2^32)."""
    if total_past == B31:
        return [B31 - 3, (1 << 20) + 11, 4099]
    return [B31 - 3, B31 - 5, (1 << 20) + 11]


def table_views(base, sizes):
    out, at = [], 0
    for s in sizes:
        out.append(base[at:at + s]); at += s
    return out


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_collector_and_select_tables_past_2_32(ext, dtype):
    sizes = table_sizes(B32)
    total = sum(sizes)
    esz = 4 if dtype == torch.float32 else 2
    need(esz * total + GB)
    kind = 'f32' if dtype == torch.float32 else 'b16'
    base = fill(total, kind, dtype, [(B31, 50.0), (B31 - 3, -50.0), (B32, 49.0), (total - 1, -49.0)])
    ts = table_views(base, sizes)
    half = dtype != torch.float32
    mm = torch.empty(len(ts), 2, device='cuda'); mm[:, 0] = float('inf'); mm[:, 1] = float('-inf')
    if half: ext.Multi_MinMax_T_Half(table(ts), max(sizes), dtype, mm)
    else: ext.Multi_MinMax_T(table(ts), max(sizes), mm)
    for i, t in enumerate(ts):
        w = torch.tensor([float('inf'), float('-inf')], device='cuda'); ext.MinMax_T(t, w)
        assert mm[i].tolist() == w.tolist(), i
    bins = 2048
    hs = torch.tensor([0.01, 0.02, 0.005], device='cuda')
    hist = torch.zeros(len(ts), bins, dtype=torch.int32, device='cuda')
    if half: ext.Multi_Histogram_T_Half(table(ts), max(sizes), dtype, hs, True, hist, bins)
    else: ext.Multi_Histogram_T(table(ts), max(sizes), hs, True, hist, bins)
    for i, t in enumerate(ts):
        w = torch.zeros(bins, dtype=torch.int32, device='cuda'); ext.Histogram_T_DeviceScale(t, hs[i:i + 1], True, w)
        assert torch.equal(hist[i], w), i
    cap = 1 << 18
    ws = torch.empty(ext.Multi_Quantile_Workspace_Bytes(len(ts), cap), dtype=torch.uint8, device='cuda')
    for q in (0.9999, 0.5):
        out = torch.full((len(ts), 2), -7.0, device='cuda')
        if half: ext.Multi_Quantile_T_Half(table(ts), max(sizes), dtype, q, out, 2, ws, cap, None)
        else: ext.Multi_Quantile_T(table(ts), max(sizes), q, out, 2, ws, cap, None)
        for i, t in enumerate(ts):
            w = ext.Quantile_T_Half(t, q) if half else ext.Quantile_T(t, q)
            assert out[i].tolist() == w.tolist(), (q, i)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_quantile_table_with_one_row_past_2_31(ext, dtype):
    n = B31 + 8 if dtype == torch.float32 else B32 + 100
    esz = 4 if dtype == torch.float32 else 2
    need(esz * (n + 5000) + GB)
    kind = 'f32' if dtype == torch.float32 else 'b16'
    plants = [(i, v) for i, v in zip(boundary_indices(n), [40.0, -40.0, 39.0, -39.0, 38.0, -38.0, 37.0, -37.0])]
    big = fill(n, kind, dtype, plants)
    small = fill(5000, kind, dtype)
    counts = counts_of(kind, n, plants)
    cap = 1 << 18
    ws = torch.empty(ext.Multi_Quantile_Workspace_Bytes(2, cap), dtype=torch.uint8, device='cuda')
    guess = ext.Quantile_Guess_Init(2, big)
    for g in (None, guess, guess):                                         # plain, then speculative cold and warm
        out = torch.full((2, 2), -7.0, device='cuda')
        if dtype == torch.float32: ext.Multi_Quantile_T(table([small, big]), n, 0.9999, out, 2, ws, cap, g)
        else: ext.Multi_Quantile_T_Half(table([small, big]), n, dtype, 0.9999, out, 2, ws, cap, g)
        check_quantiles(out[1].tolist(), counts, n, 0.9999, f'Multi_Quantile row past 2^31 guess={g is not None}')
        w = ext.Quantile_T(small, 0.9999) if dtype == torch.float32 else ext.Quantile_T_Half(small, 0.9999)
        assert out[0].tolist() == w.tolist()


# Per-channel tables: tensor 0 holds 2^31 - 3 = 5 x 429496729 elements as [rows, 5, 1] (so tensor 1 starts at concatenated offset 2^31 - 3
# exactly), the others [rows, 4, 9].
LC_GEOMETRY = ((5, 1), (4, 9))
LC_SCALES = {5: ([0.0625, 0.125, 0.03125, 0.25, 0.5], [0.0, 1.0, -1.0, 2.0, -3.0]), 4: ([0.0625, 0.125, 0.03125, 0.25], [0.0, 1.0, -1.0, 2.0])}


def lc_sizes(total_past):
    sizes = table_sizes(total_past)
    C, epc = LC_GEOMETRY[1]
    return [sizes[0]] + [v // (C * epc) * (C * epc) for v in sizes[1:]]


def lc_geometry(t):
    return LC_GEOMETRY[0 if t == 0 else 1]


def same_bits(a, b):
    """Bitwise equality on the device."""
    view = {1: torch.int8, 2: torch.int16, 4: torch.int32}[a.element_size()]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.reshape(-1).view(view), b.reshape(-1).view(view))


def regen(kind, a, b, plants):
    """fill()'s values on [a, b) of the concatenation, regenerated on the device as fp32."""
    v = values_torch(kind, hash_of(torch.arange(a, b, dtype=torch.int64, device='cuda')))
    for i, val in plants:
        if a <= i < b: v[i - a] = val
    return v


@pytest.mark.parametrize('past', [B31, B32], ids=['2_31', '2_32'])
@pytest.mark.parametrize('op', ['LT', 'LC'])
def test_fp32_fake_quant_table_in_place_past(ext, oracle, op, past):
    """Multi_QuantizeTensor_LT / _LC with every output pointer equal to its input (an element-wise kernel reads each element before it
    writes it), so a concatenation past 2^32 fits the memory budget: tensor 1 starts at 2^31 - 3 and one tensor straddles `past`.
    Every tensor against the single-tensor binding on its regenerated input, and the oracle on windows at the tensor boundaries."""
    sizes = table_sizes(past) if op == 'LT' else lc_sizes(past)
    offs = [sum(sizes[:t]) for t in range(len(sizes))]
    total = sum(sizes)
    assert offs[1] == B31 - 3 and any(off < past < off + size for off, size in zip(offs, sizes))
    need(4 * total + 2 * GB)
    plants = [(B31 - 3, 900.0), (B31, -900.0), (min(B32, total - 1), 33.0), (total - 1, 7.0)]
    x = fill(total, 'f32', torch.float32, plants)
    s, o = t1(0.0625), t1(-2.0)
    if op == 'LT':
        views = table_views(x, sizes)
        d = torch.tensor([(v.data_ptr(), v.data_ptr(), s.data_ptr(), o.data_ptr(), v.numel()) for v in views], dtype=torch.int64).cuda()
        ext.Multi_QuantizeTensor_LT(d, max(sizes), -128, 127, 0)
        single = lambda t, v: ext.QuantizeTensor_LT(v, s, o, -128, 127, 0)
        want_host = lambda t, xw: oracle.linear_quant_t(xw, 0.0625, -2.0, -128, 127, 0)
    else:
        sc = {C: (torch.tensor(a, device='cuda'), torch.tensor(b, device='cuda')) for C, (a, b) in LC_SCALES.items()}
        views = [v.view(-1, *lc_geometry(t)) for t, v in enumerate(table_views(x, sizes))]
        d = torch.tensor([(v.data_ptr(), v.data_ptr(), sc[v.shape[1]][0].data_ptr(), sc[v.shape[1]][1].data_ptr(), v.numel(), v.shape[2],
                           v.shape[1]) for v in views], dtype=torch.int64).cuda()
        ext.Multi_QuantizeTensor_LC(d, max(sizes), -128, 127, 0)
        single = lambda t, v: ext.QuantizeTensor_LC(v.view(-1, *lc_geometry(t)), *sc[lc_geometry(t)[0]], -128, 127, 1, 0)
        want_host = lambda t, xw: oracle.linear_quant_c(xw.reshape(-1, *lc_geometry(t)), *map(np.float32, LC_SCALES[lc_geometry(t)[0]]), 1,
                                                        -128, 127, 0)
    flat = x.view(-1)
    for t, (off, size) in enumerate(zip(offs, sizes)):
        row = 1 if op == 'LT' else int(np.prod(lc_geometry(t)))
        step = CHUNK // row * row
        for a in range(0, size, step):
            b = min(size, a + step)
            got, want = flat[off + a:off + b], single(t, regen('f32', off + a, off + b, plants)).reshape(-1)
            assert same_bits(got, want), (op, t, a, b)
        w = WIN // row * row
        for a in sorted({0, max(0, size - w)} | ({(B32 - off) // row * row} if off < B32 < off + size else set())):
            b = min(size, a + w)
            xw = host_values('f32', off + a, off + b, plants)
            assert np.array_equal(bits(flat[off + a:off + b]), bits(want_host(t, xw)).reshape(-1)), (op, t, a, b)


def test_half_lc_table_past_2_32(ext):
    """Multi_QuantizeTensor_LC_Half on a bf16 concatenation past 2^32 (tensor 1 at offset 2^31 - 3), against the single-tensor binding."""
    sizes = lc_sizes(B32)
    total = sum(sizes)
    assert sum(sizes[:1]) == B31 - 3 and sum(sizes[:-1]) < B32 < total
    need(2 * 2 * total + GB)
    x = fill(total, 'b16', torch.bfloat16, [(B32, 15.0), (B31 - 3, -16.0), (B31, 15.5)])
    y = torch.empty_like(x)
    sc = {C: (torch.tensor(a, device='cuda'), torch.tensor(b, device='cuda')) for C, (a, b) in LC_SCALES.items()}
    rows = [v.view(-1, *lc_geometry(t)) for t, v in enumerate(table_views(x, sizes))]
    outs = [v.view(r.shape) for v, r in zip(table_views(y, sizes), rows)]
    d = torch.tensor([(a.data_ptr(), b.data_ptr(), sc[a.shape[1]][0].data_ptr(), sc[a.shape[1]][1].data_ptr(), a.numel(), a.shape[2], a.shape[1])
                      for a, b in zip(rows, outs)], dtype=torch.int64).cuda()
    ext.Multi_QuantizeTensor_LC_Half(d, max(sizes), torch.bfloat16, -128, 127, 0)
    for a, b in zip(rows, outs):
        step = max(1, SUB // (a.shape[1] * a.shape[2]))
        for lo in range(0, a.shape[0], step):
            assert same_bits(b[lo:lo + step], ext.QuantizeTensor_LC_Half(a[lo:lo + step], *sc[a.shape[1]], -128, 127, 1, 0)), lo


# ---------------------------------------------------------------------------------------------------------------- paired moments
def test_paired_moments_one_row_past_2_31(ext):
    """One row of 2^31 + 3 bf16 pairs of small integers: every partial sum is an integer below 2^53, so the four fp64 sums are exact."""
    n = B31 + 3
    need(2 * 2 * n + GB)
    p = torch.empty(n, dtype=torch.bfloat16, device='cuda')
    r = torch.empty_like(p)
    cnt = torch.zeros(64, dtype=torch.int64, device='cuda')
    for a in range(0, n, CHUNK):
        h = hash_of(torch.arange(a, min(n, a + CHUNK), dtype=torch.int64, device='cuda')) & 63
        p[a:a + CHUNK] = ((h & 7) - 4).to(torch.bfloat16)
        r[a:a + CHUNK] = ((h >> 3) - 4).to(torch.bfloat16)
        cnt += torch.bincount(h, minlength=64)
    cnt = cnt.cpu().numpy()
    c = np.arange(64)
    pv, rv = (c & 7) - 4, (c >> 3) - 4
    want = [int((cnt * (pv - rv) ** 2).sum()), int((cnt * rv * rv).sum()), int((cnt * pv * pv).sum()), int((cnt * pv * rv).sum())]
    out = torch.full((1, 4), -1.0, dtype=torch.float64, device='cuda')
    ws = torch.empty(ext.Multi_Paired_Moments_Workspace_Bytes(1, n), dtype=torch.uint8, device='cuda')
    d = torch.tensor([(p.data_ptr(), r.data_ptr(), 1, n, 0)], dtype=torch.int64, device='cuda')
    ext.Multi_Paired_Moments(d, n, torch.bfloat16, out, ws)
    assert out[0].tolist() == [float(v) for v in want]


# ---------------------------------------------------------------------------------------------------------------- refusals
def refusal_calls(ext):
    """One call per 'refuses' binding on zero-stride views of 2^31 elements (no memory behind them)."""
    f = torch.zeros(1, device='cuda').expand(B31)
    fc = torch.zeros(1, 1, device='cuda').expand(2, B31 // 2)
    h = torch.zeros(1, dtype=torch.bfloat16, device='cuda').expand(B31)
    hc = torch.zeros(1, 1, dtype=torch.bfloat16, device='cuda').expand(2, B31 // 2)
    s, o, s2, o2 = t1(0.1), t1(0.0), torch.ones(2, device='cuda'), torch.zeros(2, device='cuda')
    return {
        'QuantizeTensor_LT': lambda: ext.QuantizeTensor_LT(f, s, o, -128, 127, 0),
        'QuantizeTensor_LC': lambda: ext.QuantizeTensor_LC(fc, s2, o2, -128, 127, 0, 0),
        'QuantizeTensor_toInt': lambda: ext.QuantizeTensor_toInt(f, s, o, -128, 127, -1000, 0, 8),
        'QuantizeTensor_LT_Half': lambda: ext.QuantizeTensor_LT_Half(h, s, o, -128, 127, 0),
        'QuantizeTensor_LC_Half': lambda: ext.QuantizeTensor_LC_Half(hc, s2, o2, -128, 127, 0, 0),
        'QuantizeTensor_FT_Half': lambda: ext.QuantizeTensor_FT_Half(h, s, o, 4, 3, -448.0, 448.0, 0),
        'QuantizeTensor_FC_Half': lambda: ext.QuantizeTensor_FC_Half(hc, s2, o2, 4, 3, -448.0, 448.0, 0, 0),
        'QuantizeTensor_LT_B': lambda: ext.QuantizeTensor_LT_B(f, s, o, f, -128, 127, 0),
        'QuantizeTensor_LC_B': lambda: ext.QuantizeTensor_LC_B(fc, s2, o2, fc, -128, 127, 0, 0),
        'QuantizeTensor_FT_B': lambda: ext.QuantizeTensor_FT_B(f, s, o, f, 4, 3, -448.0, 448.0, 0),
        'QuantizeTensor_FC_B': lambda: ext.QuantizeTensor_FC_B(fc, s2, o2, fc, 4, 3, -448.0, 448.0, 0, 0),
        'TensorClip_T': lambda: ext.TensorClip_T(f, f, s),
        'TensorClip_C': lambda: ext.TensorClip_C(fc, fc, s2, 0),
        'RoundingLoss_LT': lambda: ext.RoundingLoss_LT(f, s, o, -128, 127, 0),
        'RoundingLoss_LC': lambda: ext.RoundingLoss_LC(fc, s2, o2, -128, 127, 0, 0),
        'RoundingLoss_LT_B': lambda: ext.RoundingLoss_LT_B(f, f, s, o, -128, 127, 0),
        'RoundingLoss_LC_B': lambda: ext.RoundingLoss_LC_B(fc, fc, s2, o2, -128, 127, 0, 0),
    }


REFUSAL_NAMES = sorted(REFUSES)


@pytest.mark.parametrize('name', REFUSAL_NAMES)
def test_refuses_above_2_31_before_any_allocation(ext, name):
    calls = refusal_calls(ext)
    assert set(calls) == REFUSES
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with pytest.raises(RuntimeError, match='too many element'):
        calls[name]()
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() == before and torch.cuda.memory_allocated() == before
