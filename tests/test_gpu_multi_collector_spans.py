"""Multi-tensor min/max and histogram (Multi_MinMax_T / Multi_Histogram_T) on tables built to land on the edges of their work partition: each
CTA owns one contiguous span of the concatenated tensors, and the aligned body of each (tensor, span) piece is streamed through a ring of
16 KB stages (4096 floats) while unaligned heads and tails are read directly.  Bit for bit against the oracle and against the per-tensor
collectors (MinMax_T, Histogram_T_DeviceScale)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STAGE = 4096                    # floats per ring stage


@pytest.fixture(scope='module')
def ext():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from ppq_b200.ffi import extension
    return extension()


def span_of(total, count, max_n, ctas_per_sm):
    """The span each CTA owns (multi-tensor launch: at most ctas_per_sm CTAs per SM, >= 64 Ki elements each)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = max(1, min(sms * ctas_per_sm, -(-count * max_n // 65536)))
    return ((-(-total // grid)) + 3) & ~3


class Table:
    """Tensors carved out of one device pool at chosen float offsets (offset % 4 = misalignment of the base), optionally sharing slots."""

    def __init__(self, specs, seed, slots=None, poison=()):
        r = np.random.RandomState(seed)
        starts, pos = [], 0
        for n, off in specs:
            pos = (pos + 3) & ~3
            starts.append(pos + off)
            pos += off + n
        pool = r.standard_normal(pos + 8).astype(np.float32)
        pool[: pos // 2] = np.maximum(pool[: pos // 2], 0)                            # half post-ReLU: a pile-up in bin 0
        for i, k, v in poison: pool[starts[i] + k] = v
        self.np = [pool[s:s + n] for s, (n, _) in zip(starts, specs)]
        self.pool = torch.from_numpy(pool).cuda()
        self.dev = [self.pool[s:s + n] for s, (n, _) in zip(starts, specs)]
        self.slots = list(range(len(specs))) if slots is None else slots
        self.S = max(self.slots) + 1
        self.descs = torch.tensor([[d.data_ptr(), d.numel(), s] for d, s in zip(self.dev, self.slots)], dtype=torch.int64, device='cuda')
        self.max_n = max(n for n, _ in specs)

    def slot_values(self, s):
        return np.concatenate([x for x, t in zip(self.np, self.slots) if t == s])


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check(ext, oracle, tab, bins_list=(2048, 4096, 12287), per_tensor=True):
    mm = torch.empty(tab.S, 2, device='cuda'); mm[:, 0] = float('inf'); mm[:, 1] = float('-inf')
    ext.Multi_MinMax_T(tab.descs, tab.max_n, mm)
    got = mm.cpu().numpy()
    for s in range(tab.S):
        x = tab.slot_values(s)
        if np.isnan(x).any():
            assert np.isnan(got[s]).all(), s
        else:
            lo, hi = oracle.minmax_t(x)
            assert bits(got[s]).tolist() == bits([lo, hi]).tolist(), (s, got[s], lo, hi)
        if per_tensor and tab.slots.count(s) == 1:
            one = torch.empty(2, device='cuda'); ext.MinMax_Init(one[0:1], one[1:2])
            ext.MinMax_T(tab.dev[tab.slots.index(s)], one)
            assert bits(one.cpu().numpy()).tolist() == bits(got[s]).tolist(), s
    for bins in bins_list:
        hs = np.empty(tab.S, np.float32)
        for s in range(tab.S):
            x = tab.slot_values(s)
            f = np.abs(x[np.isfinite(x)])
            hs[s] = np.float32(max(float(f.max()) if f.size else 1.0, 1e-3)) / np.float32(bins)
        hs_dev = torch.from_numpy(hs).cuda()
        for clip in (True, False):
            hist = torch.zeros(tab.S, bins, dtype=torch.int32, device='cuda')
            ext.Multi_Histogram_T(tab.descs, tab.max_n, hs_dev, clip, hist, bins)
            got_h = hist.cpu().numpy()
            for s in range(tab.S):
                want = oracle.histogram_t(tab.slot_values(s), hs[s], bins, clip)
                assert np.array_equal(got_h[s], want), (bins, clip, s)
                if per_tensor and tab.slots.count(s) == 1:
                    one = torch.zeros(bins, dtype=torch.int32, device='cuda')
                    ext.Histogram_T_DeviceScale(tab.dev[tab.slots.index(s)], hs_dev[s:s + 1], clip, one)
                    assert np.array_equal(one.cpu().numpy(), want), (bins, clip, s)


def test_sizes_at_stage_and_span_edges_with_misaligned_bases(ext, oracle):
    sizes = [1, 3, 4, 5, 17, STAGE - 1, STAGE, STAGE + 1, 3 * STAGE + 2]
    specs = [(n, off) for n in sizes for off in (0, 1, 2, 3)]
    total = sum(n for n, _ in specs)
    # a tensor that covers whole spans: its length is a span +- 1 for both launch shapes (2 and 1 CTAs per SM)
    for cps in (2, 1):
        sp = span_of(total + 8 * STAGE, len(specs) + 2, 8 * STAGE, cps)
        specs += [(sp - 1, 1), (sp + 1, 3)]
    check(ext, oracle, Table(specs, seed=1))


@pytest.mark.parametrize('count', [1, 2, 4096])
def test_tensor_counts(ext, oracle, count):
    r = np.random.RandomState(count)
    if count == 1: specs = [(1_000_003, 1)]
    elif count == 2: specs = [(5, 2), (700_001, 3)]
    else: specs = [(int(r.randint(1, 600)), int(r.randint(0, 4))) for _ in range(count)]
    check(ext, oracle, Table(specs, seed=count), bins_list=(4096, 12287) if count > 2 else (2048, 4096, 12287), per_tensor=count <= 2)


def test_one_huge_tensor_among_many_tiny_ones(ext, oracle):
    r = np.random.RandomState(7)
    specs = [(int(r.randint(1, 40)), int(r.randint(0, 4))) for _ in range(300)]
    specs.insert(150, (9_000_001, 1))
    check(ext, oracle, Table(specs, seed=7), bins_list=(4096,), per_tensor=False)


def test_repeated_slots(ext, oracle):
    specs = [(STAGE + 1, 1), (17, 0), (2 * STAGE, 2), (300_001, 3), (5, 1), (4, 0)]
    check(ext, oracle, Table(specs, seed=11, slots=[0, 1, 0, 2, 1, 0]), bins_list=(2048, 4096))


@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_non_finite_in_first_middle_and_last_stage_of_a_span(ext, oracle, value):
    n = 8_000_000
    sp = span_of(n + 64, 3, n, 2)
    k = 5 * sp - 31                                                       # where the sixth CTA's span starts inside the big tensor
    for where in (k + 1, k + sp // 2, k + sp - 2):
        check(ext, oracle, Table([(31, 1), (n, 0), (33, 2)], seed=3, poison=[(1, where, value)]), bins_list=(4096,))
