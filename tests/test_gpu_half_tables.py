"""fp16 / bf16 descriptor tables: the multi-tensor collectors, the multi-tensor select and the weight table on half tensors.

The contract is the one of the single-tensor half kernels, extended to tables: every statistic equals, bit for bit, what the fp32 table
kernel writes for the same table over the upcasts x.float(); the weight table writes what QuantizeTensor_LC_Half returns per weight.
Both are also cross-checked against the single-tensor half collectors.  On top: calibrate_arena(half_inputs=True) renders the scales
and offsets RuntimeCalibrationPass renders for a network cast to half and for an fp32 network under torch.autocast."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HALF = [torch.float16, torch.bfloat16]
EDGE_SIZES = [1, 7, 8, 9, 8191, 8192, 8193]                            # around one 16-byte vector and one 16 KB stage of halves


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


def specials(dtype):
    fi = torch.finfo(dtype)
    sub = torch.tensor(1, dtype=torch.int16).view(dtype).item()        # smallest subnormal
    return [float('nan'), -float('nan'), float('inf'), float('-inf'), 0.0, -0.0, sub, -sub, fi.max, -fi.max]


def neg_nan(dtype):
    return torch.tensor([-1], dtype=torch.int16).view(dtype)           # 0xFFFF: a NaN with the sign bit set


def random_half(n, dtype, seed, relu=False):
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(n, generator=g) * 3
    if relu: x = torch.relu(x)
    return x.to(dtype).cuda()


def slices(base, sizes, offsets):
    """Views of `base` (16-byte aligned) of every size at every element offset from a 16-byte boundary, laid out one after another."""
    out, at = [], 0
    for n in sizes:
        for off in offsets:
            start = (at + 7) // 8 * 8 + off
            out.append(base[start:start + n])
            at = start + n
    assert at <= base.numel()
    return out


def table(tensors, slots):
    return torch.tensor([(t.data_ptr(), t.numel(), s) for t, s in zip(tensors, slots)], dtype=torch.int64).cuda()


def max_n(tensors):
    return max(t.numel() for t in tensors)


def span_of(sizes):
    """The span length multi_stream_kernel forms for a table of these sizes: the total split over the launch's CTAs, rounded up to 8 halves."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = max(1, min(2 * sms, (len(sizes) * max(sizes) + 65535) // 65536))
    return ((sum(sizes) + grid - 1) // grid + 7) // 8 * 8


def bits(t):
    a = t.detach().cpu().numpy()
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_bits(got, want, msg=''):
    assert np.array_equal(bits(got), bits(want)), msg


def minmax_arena(slots):
    mm = torch.empty(slots, 2, device='cuda')
    mm[:, 0] = float('inf'); mm[:, 1] = float('-inf')
    return mm


def both_minmax(ext, tensors, slots, dtype):
    n_slots = max(slots) + 1
    got, want = minmax_arena(n_slots), minmax_arena(n_slots)
    ext.Multi_MinMax_T_Half(table(tensors, slots), max_n(tensors), dtype, got)
    ups = [t.float() for t in tensors]
    ext.Multi_MinMax_T(table(ups, slots), max_n(tensors), want)
    torch.cuda.synchronize()
    return got, want


def both_hist(ext, tensors, slots, dtype, scales, bins, clip):
    n_slots = max(slots) + 1
    got = torch.zeros(n_slots, bins, dtype=torch.int32, device='cuda')
    want = torch.zeros_like(got)
    ext.Multi_Histogram_T_Half(table(tensors, slots), max_n(tensors), dtype, scales, clip, got, bins)
    ups = [t.float() for t in tensors]
    ext.Multi_Histogram_T(table(ups, slots), max_n(tensors), scales, clip, want, bins)
    torch.cuda.synchronize()
    return got, want


def edge_tensors(dtype, seed, relu=False):
    """Every edge size at every element offset 0-7 from a 16-byte boundary, with the special values planted at both ends and the middle."""
    sizes = EDGE_SIZES
    base = random_half(sum(sizes) * 8 + 16 * len(sizes) * 8 + 64, dtype, seed, relu)
    ts = slices(base, sizes, range(8))
    sp = specials(dtype)[2:]                                            # NaN-free: NaN poisoning is checked on its own
    for k, t in enumerate(ts):
        for j, pos in enumerate((0, t.numel() // 2, t.numel() - 1)):
            t[pos] = sp[(k + j) % len(sp)]
    return ts


# ------------------------------------------------------------------------------------------------ min / max and histogram tables
@pytest.mark.parametrize('dtype', HALF)
def test_minmax_table_sizes_offsets_and_specials(ext, dtype):
    ts = edge_tensors(dtype, 1)
    slots = list(range(len(ts)))
    got, want = both_minmax(ext, ts, slots, dtype)
    assert_bits(got, want, 'min/max table vs the fp32 table on the upcasts')
    for k in (0, 9, 17, 30, len(ts) - 1):                              # ... and vs the single-tensor half collector
        one = minmax_arena(1)
        ext.MinMax_T(ts[k], one[0])
        assert_bits(got[k], one[0], f'tensor {k}')
    # finite data only: the extremes are the true ones
    fin = [random_half(n, dtype, 100 + n)[off:] for n, off in ((8200, 1), (77, 3), (9, 7))]
    got, _ = both_minmax(ext, fin, [0, 1, 2], dtype)
    for k, t in enumerate(fin):
        assert got[k, 0].item() == t.float().min().item() and got[k, 1].item() == t.float().max().item()


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('count', [1, 2, 4096])
def test_table_counts_and_repeated_slots(ext, dtype, count):
    base = random_half(count * 24 + 64, dtype, count)
    ts = [base[24 * k + (k % 8):24 * k + (k % 8) + 1 + (k % 16)] for k in range(count)]
    slots = [k % 5 for k in range(count)]                              # several tensors accumulate into one slot
    got, want = both_minmax(ext, ts, slots, dtype)
    assert_bits(got, want, f'{count} tensors, repeated slots')
    scales = torch.full((5,), 0.05, device='cuda')
    got, want = both_hist(ext, ts, slots, dtype, scales, 2048, True)
    assert_bits(got, want, f'{count} tensors, repeated slots, histogram')
    assert int(got.sum().item()) > 0


@pytest.mark.parametrize('dtype', HALF)
def test_one_huge_tensor_among_tiny_ones_and_specials_in_every_stage_of_a_span(ext, dtype):
    tiny = [random_half(40, dtype, k)[k % 8:k % 8 + 1 + k] for k in range(20)]
    huge = random_half(8 * (1 << 20) + 13, dtype, 7)[5:]               # 2-byte aligned base, odd element offset
    ts = tiny[:10] + [huge] + tiny[10:]
    span = span_of([t.numel() for t in ts])
    assert span > 3 * 8192                                              # a span holds several stages
    sp = specials(dtype)[2:]
    first_span_of_huge = (sum(t.numel() for t in tiny[:10]) + span - 1) // span * span - sum(t.numel() for t in tiny[:10])
    for j, pos in enumerate((first_span_of_huge + 3, first_span_of_huge + span // 2, first_span_of_huge + span - 2,
                             first_span_of_huge - 1, first_span_of_huge, huge.numel() - 1)):
        huge[pos] = sp[j % len(sp)]
    slots = list(range(len(ts)))
    got, want = both_minmax(ext, ts, slots, dtype)
    assert_bits(got, want, 'huge among tiny')
    scales = torch.full((len(ts),), 0.01, device='cuda')
    for clip in (True, False):
        got, want = both_hist(ext, ts, slots, dtype, scales, 4096, clip)
        assert_bits(got, want, f'huge among tiny, histogram clip={clip}')
    one = torch.zeros(4096, dtype=torch.int32, device='cuda')
    ext.Histogram_T_DeviceScale(huge, scales[10:11], False, one)
    assert_bits(got[10], one, 'vs the single-tensor half histogram')
    # a tensor of exactly the span length the launch forms, one shorter and one longer, in front of the huge tensor
    s0 = span
    for _ in range(8): s0 = span_of([s0, huge.numel()])
    assert s0 == span_of([s0, huge.numel()])
    for d in (-1, 0, 1):
        first = random_half(s0 + 16, dtype, 50 + d)[3:3 + s0 + d]
        got, want = both_minmax(ext, [first, huge], [0, 1], dtype)
        assert_bits(got, want, f'span length {s0} {d:+d}')
        got, want = both_hist(ext, [first, huge], [0, 1], dtype, scales[:2], 2048, True)
        assert_bits(got, want, f'span length {s0} {d:+d}, histogram')


@pytest.mark.parametrize('dtype', HALF)
def test_nan_of_either_sign_poisons_only_its_slot(ext, dtype):
    for where in ('first', 'middle', 'last'):
        for nan in (torch.tensor([float('nan')]).to(dtype), neg_nan(dtype)):
            ts = [random_half(3 * 8192 + 11, dtype, 3)[1:], random_half(100, dtype, 4), random_half(8192 * 2, dtype, 5)]
            pos = {'first': 2, 'middle': ts[0].numel() // 2, 'last': ts[0].numel() - 1}[where]
            ts[0][pos] = nan.cuda()[0]
            got, want = both_minmax(ext, ts, [0, 1, 2], dtype)
            assert_bits(got, want, f'NaN {where}')
            assert bool(got[0].isnan().all()) and not bool(got[1:].isnan().any())
            got, want = both_hist(ext, ts, [0, 1, 2], dtype, torch.full((3,), 0.02, device='cuda'), 2048, True)
            assert_bits(got, want, f'NaN {where}, histogram')


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('bins', [2048, 4096, 12287])
def test_histogram_table_bins_clip_and_post_relu_data(ext, dtype, bins):
    for relu in (False, True):                                          # post-ReLU: half of the elements pile up in bin 0
        ts = edge_tensors(dtype, 11 + bins, relu)[::3] + [random_half(200000, dtype, bins, relu)[3:]]
        slots = list(range(len(ts)))
        g = torch.Generator().manual_seed(bins)
        scales = (torch.rand(len(ts), generator=g) * 0.01 + 0.0005).cuda()
        for clip in (True, False):
            got, want = both_hist(ext, ts, slots, dtype, scales, bins, clip)
            assert_bits(got, want, f'bins={bins} clip={clip} relu={relu}')
            if not clip:
                assert got.sum(dim=1).tolist() == [t.numel() for t in ts]
        if relu: assert int(got[-1, 0].item()) > 90000


# ------------------------------------------------------------------------------------------------ the select table
def both_quantiles(ext, tensors, slots, dtype, q, cap, guess_h=None, guess_f=None, n_slots=None):
    n_slots = n_slots or max(slots) + 1
    got = torch.full((n_slots, 2), -7.0, device='cuda')
    want = torch.full((n_slots, 2), -7.0, device='cuda')
    ws = torch.empty(ext.Multi_Quantile_Workspace_Bytes(len(tensors), cap), dtype=torch.uint8, device='cuda')
    ext.Multi_Quantile_T_Half(table(tensors, slots), max_n(tensors), dtype, q, got, 2, ws, cap, guess_h)
    ups = [t.float() for t in tensors]
    ext.Multi_Quantile_T(table(ups, slots), max_n(tensors), q, want, 2, ws, cap, guess_f)
    torch.cuda.synchronize()
    return got, want


@pytest.mark.parametrize('dtype', HALF)
def test_quantile_table_cold_sizes_offsets_specials_and_an_empty_row(ext, dtype):
    ts = edge_tensors(dtype, 21) + [random_half(300001, dtype, 22, relu=True)[1:]]
    for k in (3, 20, 41):                                               # NaN of both signs: above +inf and below -inf in the key order
        ts[k][0] = float('nan'); ts[k][-1] = neg_nan(dtype).cuda()[0]
    empty = ts[5][:0]
    ts = ts[:5] + [empty] + ts[5:]
    slots = list(range(len(ts)))
    for q, cap in ((0.9999, 1 << 16), (0.5, 1 << 16), (0.75, 64)):      # 0.5 on odd sizes: half-integer ranks; a small cap forces the refining passes
        got, want = both_quantiles(ext, ts, slots, dtype, q, cap)
        assert_bits(got, want, f'q={q} cap={cap}')
        assert got[5].tolist() == [-7.0, -7.0]                          # the n = 0 row leaves its slot alone
    for k in (0, 13, 30, len(ts) - 1):
        assert_bits(got[k], ext.Quantile_T_Half(ts[k], 0.75), f'tensor {k} vs the single-tensor half select')


@pytest.mark.parametrize('dtype', HALF)
def test_quantile_table_with_a_warm_guess_over_consecutive_batches(ext, dtype):
    shapes = [(1 << 20) + 5, 70001, 8193, 9]
    guess_h, guess_f = ext.Quantile_Guess_Init(len(shapes), torch.zeros(1, device='cuda')), ext.Quantile_Guess_Init(len(shapes), torch.zeros(1, device='cuda'))
    for batch in range(4):                                              # the same activations, batch after batch: the tails move little
        ts = [random_half(n + 8, dtype, 1000 * batch + k, relu=(k == 1))[k:k + n] for k, n in enumerate(shapes)]
        got, want = both_quantiles(ext, ts, [2, 0, 3, 1], dtype, 0.9999, 1 << 16, guess_h, guess_f)
        assert_bits(got, want, f'batch {batch}')
        for k, t in enumerate(ts):
            assert_bits(got[[2, 0, 3, 1][k]], ext.Quantile_T(t.float(), 0.9999), f'batch {batch} tensor {k}')
    assert_bits(guess_h, guess_f, 'the thresholds remembered for the next batch')


# ------------------------------------------------------------------------------------------------ the weight table
def same_half_values(got, want, msg):
    assert got.dtype == want.dtype and got.shape == want.shape, msg
    g, w = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    ok = (g == w) | (got.contiguous().isnan() & want.contiguous().isnan())
    assert bool(ok.all()), f'{msg}: {(~ok).sum().item()} elements differ'


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('rounding', range(8))
def test_weight_table_matches_the_single_tensor_half_kernel(ext, dtype, rounding):
    from ppq_b200.calibration import MultiWeightQuantizer
    g = torch.Generator().manual_seed(rounding)

    def w(*shape):
        x = torch.randn(*shape, generator=g) * 0.2
        x.view(-1)[::7] = torch.round(x.view(-1)[::7] * 16) / 16        # exact ties of x / 0.0625
        return x.to(dtype).cuda()
    conv, dw, lin, big = w(32, 16, 3, 3), w(16, 1, 3, 3), w(10, 24), w(64, 1024)
    cl = w(8, 16, 3, 3).to(memory_format=torch.channels_last)
    buf = w(24 * 40 + 8)
    unaligned = buf[1:1 + 24 * 40].view(24, 40)                        # epc % 8 == 0 but a 2-byte-aligned base: the element-wise route
    sp = w(4, 16)
    sp.view(-1)[:10] = torch.tensor(specials(dtype), dtype=torch.float32).to(dtype).cuda()
    weights = [conv, dw, lin, big, cl, unaligned, sp]
    scales = [(torch.rand(x.shape[0], generator=g) * 0.02 + 0.002).cuda() for x in weights]
    for s in scales: s[0] = 0.0625
    for qmin, qmax, off in ((-128, 127, 0.0), (-8, 7, 0.0), (0, 255, 3.0)):
        offsets = [torch.full((x.shape[0],), off, device='cuda') for x in weights]
        mw = MultiWeightQuantizer(weights, scales, offsets, channel_axis=0, quant_min=qmin, quant_max=qmax, rounding=rounding, half_inputs=True)
        outs = mw()
        torch.cuda.synchronize()
        for k, (x, y, s, o) in enumerate(zip(weights, outs, scales, offsets)):
            assert y.dtype == dtype and y.stride() == mw.weights[k].stride(), k
            same_half_values(y, ext.QuantizeTensor_LC_Half(x, s, o, qmin, qmax, 0, rounding), f'weight {k} {tuple(x.shape)} [{qmin}, {qmax}] mode {rounding}')
            same_half_values(y, ext.QuantizeTensor_LC(x.float(), s, o, qmin, qmax, 0, rounding).to(dtype), f'weight {k} vs fp32(X).to(dtype)')


# ------------------------------------------------------------------------------------------------ calibrate_arena on half and autocast networks
def _net(name, dtype):
    import netspec
    from ppq_b200.executor import TorchExecutor
    spec = netspec.SPECS[name]
    model = netspec.SpecNet(spec, netspec.make_params(spec, 3)).cuda().to(dtype)
    batches = [torch.from_numpy(b).cuda().to(dtype) for b in netspec.make_data(name, 4, 8, 4)]
    ex = TorchExecutor(model, batches[0], fuse_bn=False)
    ex.quantize_parameters()
    return ex, batches


def _hook_reference(name, dtype, method, autocast=False):
    import contextlib
    from ppq_b200.calibration import RuntimeCalibrationPass
    ex, batches = _net(name, dtype)
    cfgs = ex.observed_configs()
    with torch.autocast('cuda', dtype=torch.bfloat16) if autocast else contextlib.nullcontext():
        RuntimeCalibrationPass(method=method).optimize(graph=ex, dataloader=batches, executor=ex, calib_steps=8)
    return [(c.scale.clone(), c.offset.clone()) for c in cfgs]


def _assert_arena_equals(cal, cfgs, want, msg):
    from ppq_b200.core import QuantizationStates as S
    assert len(cfgs) == len(want) > 0
    for k, (c, (ws, wo)) in enumerate(zip(cfgs, want)):
        assert c.state == S.ACTIVATED
        assert_bits(c.scale.reshape(-1), ws.reshape(-1), f'{msg} slot {k} scale')
        assert_bits(c.offset.reshape(-1), wo.reshape(-1), f'{msg} slot {k} offset')
        assert_bits(cal.scale[k].reshape(-1), ws.reshape(-1), f'{msg} slot {k} arena scale')


@pytest.mark.parametrize('dtype', HALF)
@pytest.mark.parametrize('method', ['minmax', 'percentile', 'kl', 'mse'])
def test_calibrate_arena_on_half_networks_equals_the_per_observer_pass(ext, dtype, method):
    from ppq_b200.executor import calibrate_arena
    for name in ('tinyres', 'tinycat'):
        want = _hook_reference(name, dtype, method)
        for deferred in (True, 'auto', False):
            ex, batches = _net(name, dtype)
            cfgs = ex.observed_configs()
            cal = calibrate_arena(ex, batches, method=method, deferred=deferred, half_inputs=True)
            _assert_arena_equals(cal, cfgs, want, f'{name} {method} deferred={deferred}')
            if deferred is True and method == 'minmax':
                assert cal.launches == len(batches) + 1                 # one dtype: one collector launch per forward, plus the search


@pytest.mark.parametrize('method', ['minmax', 'percentile', 'kl', 'mse'])
def test_calibrate_arena_under_autocast_equals_the_per_observer_pass(ext, method):
    """An fp32 network under torch.autocast(bfloat16): fp32 weights stay in the fp32 weight table, the observed activations arrive as fp32
    (the network input) and bf16 (everything a convolution produced), so a deferred forward is observed by two launches."""
    from ppq_b200.executor import calibrate_arena
    for name in ('tinyres', 'tinycat'):
        want = _hook_reference(name, torch.float32, method, autocast=True)
        for deferred in (True, 'auto', False):
            ex, batches = _net(name, torch.float32)
            cfgs = ex.observed_configs()
            seen = set()
            with torch.autocast('cuda', dtype=torch.bfloat16):
                _, tensors = ex.forward(batches[0], collect=True)
                seen = {t.dtype for t in tensors}
                cal = calibrate_arena(ex, batches, method=method, deferred=deferred, half_inputs=True)
            assert seen == {torch.float32, torch.bfloat16}
            _assert_arena_equals(cal, cfgs, want, f'autocast {name} {method} deferred={deferred}')
            if deferred is True and method == 'minmax':
                assert cal.launches == 2 * len(batches) + 1             # a mixed table: two collector launches per forward, plus the search


@pytest.mark.parametrize('dtype', HALF)
def test_calibrate_arena_with_graphs_takes_the_batch_dtype(ext, dtype):
    from ppq_b200.executor import calibrate_arena
    want = _hook_reference('tinyres', dtype, 'kl')
    ex, batches = _net('tinyres', dtype)
    cfgs = ex.observed_configs()
    cal = calibrate_arena(ex, batches, method='kl', graphs=True, half_inputs=True)
    _assert_arena_equals(cal, cfgs, want, 'graphs=True')


@pytest.mark.parametrize('dtype', HALF)
def test_executor_puts_half_weights_in_a_table_of_their_own(ext, dtype):
    from ppq_b200.calibration import MultiWeightQuantizer
    ex, batches = _net('tinyres', dtype)
    ex.forward(batches[0])
    assert list(ex._mw) == [dtype]
    _, mw, ids = ex._mw[dtype]
    assert isinstance(mw, MultiWeightQuantizer) and mw.dtype == dtype and len(ids) >= 4      # every convolution: one launch
    by_id = {id(op.module): op for _, op in ex.quantable_operations() if op.weight_cfg is not None}
    for mid, y in zip(ids, mw()):
        op = by_id[mid]
        want = ext.QuantizeTensor_LC_Half(op.module.weight.data, op.weight_cfg.scale, op.weight_cfg.offset, op.weight_cfg.quant_min,
                                          op.weight_cfg.quant_max, op.weight_cfg.channel_axis, mw.rounding)
        same_half_values(y, want, op.name)


# ------------------------------------------------------------------------------------------------ refusals, all on the host
@pytest.mark.parametrize('dtype', HALF)
def test_refusals_happen_before_a_launch(ext, dtype):
    from ppq_b200.calibration import ArenaCalibrator, MultiWeightQuantizer
    x = random_half(64, dtype, 0)
    t, mm = table([x], [0]), minmax_arena(1)
    hist, hs = torch.zeros(1, 2048, dtype=torch.int32, device='cuda'), torch.ones(1, device='cuda')
    ws = torch.empty(ext.Multi_Quantile_Workspace_Bytes(1, 1 << 16), dtype=torch.uint8, device='cuda')
    out = torch.zeros(1, 2, device='cuda')
    lc = torch.zeros(1, 7, dtype=torch.int64, device='cuda')
    for bad in (torch.float32, torch.float64, torch.int8):             # the _Half names take fp16 / bf16 tables only
        with pytest.raises(RuntimeError, match='Expect to be FP16 or BF16'): ext.Multi_MinMax_T_Half(t, 64, bad, mm)
        with pytest.raises(RuntimeError, match='Expect to be FP16 or BF16'): ext.Multi_Histogram_T_Half(t, 64, bad, hs, True, hist, 2048)
        with pytest.raises(RuntimeError, match='Expect to be FP16 or BF16'): ext.Multi_Quantile_T_Half(t, 64, bad, 0.99, out, 2, ws, 1 << 16, None)
        with pytest.raises(RuntimeError, match='Expect to be FP16 or BF16'): ext.Multi_QuantizeTensor_LC_Half(lc, 64, bad, -128, 127, 0)
    assert mm.tolist() == [[float('inf'), float('-inf')]] and int(hist.sum().item()) == 0
    # without the keyword a half tensor is refused with the texts the fp32-only builders always had
    with pytest.raises(RuntimeError, match='fp32 CUDA tensors'):
        ArenaCalibrator(1, 'cuda', method='minmax').observe([x])
    w = torch.randn(8, 4, device='cuda').to(dtype)
    s, o = [torch.ones(8, device='cuda')] * 2, [torch.zeros(8, device='cuda')] * 2
    with pytest.raises(TypeError, match='fp32 weights, scales and offsets only'):
        MultiWeightQuantizer([w, w], s, o)
    # with it: one dtype per weight table, fp32 scales, no per-tensor half table, dense tensors only
    with pytest.raises(TypeError, match='ONE dtype'):
        MultiWeightQuantizer([w, w.float()], s, o, half_inputs=True)
    with pytest.raises(TypeError, match='ONE dtype'):
        MultiWeightQuantizer([w, w], [s[0].to(dtype)] * 2, o, half_inputs=True)
    with pytest.raises(TypeError, match='ONE dtype'):
        MultiWeightQuantizer([w, w], [torch.ones(1, device='cuda')] * 2, [torch.zeros(1, device='cuda')] * 2, channel_axis=None, half_inputs=True)
    cal = ArenaCalibrator(1, 'cuda', method='minmax', half_inputs=True)
    with pytest.raises(RuntimeError, match='dense'):
        cal.observe([random_half(64, dtype, 1)[::2]])
    with pytest.raises(RuntimeError, match='dense'):
        cal.observe([x.double()])
    assert cal.launches == 0
