"""GPU parity against the REFERENCE'S OWN CUDA KERNELS (upstream ppq/csrc compiled unmodified by oracle/build_ref.py; their results
for these seeded inputs are replayed from tests/golden/ref_cuda_calls.json.gz, see tests/refcuda.py).  This is what pins the paths that
have no CPU implementation and no test upstream: FP8 (QuantizeTensor_FT/_FC), Histogram_T / _Asymmetric_T / _C, non-default rounding
modes on the device.  Bit-exact everywhere.
"""
import numpy as np
import pytest
import torch

import refcuda

pytestmark = pytest.mark.gpu


@pytest.fixture
def ref(request):
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return refcuda.reference(request.node.nodeid)


@pytest.fixture(scope='module')
def ext():
    from ppq_b200.ffi import extension
    return extension()


def t1(v):
    return torch.tensor([v], dtype=torch.float32, device='cuda')


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def fp_inputs(n, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(n, device='cuda', generator=g) * 10
    x[::3] = x[::3].half().float()
    x[1::11] = torch.randn(x[1::11].numel(), device='cuda', generator=g) * 2 ** -8
    x[2::13] = torch.randn(x[2::13].numel(), device='cuda', generator=g) * 300
    sp = torch.tensor([0.0, -0.0, float('inf'), float('-inf'), 1e-45, 464.0, 480.0, 448.0, 1.1875, 1.4375, 2.375, 19.0, -1.1875,
                       1.5 * 2 ** -9, 2.5 * 2 ** -9, 2 ** -10, -2 ** -11, 2 ** -6, 3e38, -3e38], device='cuda')
    x[:sp.numel()] = sp
    return x


def test_linear_t_c_vs_reference_kernels(ref, ext):
    g = torch.Generator(device='cuda').manual_seed(1)
    for shape, axis in (([1, 1, 1, 1], 1), ([5, 12, 13, 4], 1), ([50, 120, 130, 4], 1), ([12, 74, 15, 411], 1), ([5011, 7, 7, 1], 0),
                        ([10, 10, 124, 47], 3), ([32, 1, 3, 3], 0), ([2048, 512, 3, 3], 0), ([1, 512, 28, 28], 1)):
        x = torch.rand(shape, device='cuda', generator=g) * 32 - 8
        s, o = torch.rand(1, device='cuda', generator=g) + 1e-3, torch.randint(0, 255, (1,), device='cuda', generator=g).float()
        for mode in range(8):
            for lo, hi in ((0, 255), (-128, 127), (-8, 7)):
                assert same_bits(ext.QuantizeTensor_LT(x, s, o, lo, hi, mode), ref.QuantizeTensor_LT(x, s, o, lo, hi, mode)), (shape, mode, lo)
        C = shape[axis]
        sc, oc = torch.rand(C, device='cuda', generator=g) + 1e-3, torch.randint(0, 255, (C,), device='cuda', generator=g).float()
        for mode in (0, 2, 5):
            assert same_bits(ext.QuantizeTensor_LC(x, sc, oc, 0, 255, axis, mode), ref.QuantizeTensor_LC(x, sc, oc, 0, 255, axis, mode)), (shape, axis, mode)


def test_fp8_vs_reference_kernels(ref, ext):
    """The FP8 pin: ours == the reference's QuantizeTensor_FT/_FC, bit for bit, including exact ties, the subnormal grid,
    saturation, signed zeros and infinities."""
    x = fp_inputs(1 << 20, 7)
    for (E, M, cmin, cmax) in ((4, 3, -448.0, 448.0), (5, 2, -57344.0, 57344.0), (4, 3, -240.0, 240.0), (3, 4, -30.0, 30.0)):
        for s, o in ((1.0, 0.0), (0.125, 0.0), (4.0, 0.0), (0.0078125, 0.0), (0.3, 2.5)):
            for mode in (0, 1, 2, 3, 4, 5, 6, 7):
                a = ext.QuantizeTensor_FT(x, t1(s), t1(o), E, M, cmin, cmax, mode)
                b = ref.QuantizeTensor_FT(x, t1(s), t1(o), E, M, cmin, cmax, mode)
                assert same_bits(a, b), (E, M, s, o, mode)
    xs = x[:64 * 27 * 16].view(64, 27, 16)
    g = torch.Generator(device='cuda').manual_seed(8)
    for axis in (0, 1, 2):
        C = xs.shape[axis]
        sc = 2.0 ** torch.randint(-7, 6, (C,), device='cuda', generator=g).float()
        oc = torch.zeros(C, device='cuda')
        assert same_bits(ext.QuantizeTensor_FC(xs, sc, oc, 4, 3, -448.0, 448.0, axis, 0), ref.QuantizeTensor_FC(xs, sc, oc, 4, 3, -448.0, 448.0, axis, 0)), axis


def test_histograms_vs_reference_kernels(ref, ext):
    g = torch.Generator(device='cuda').manual_seed(3)
    for n, relu in ((31, False), (401408, True), (1 << 21, False)):
        x = torch.randn(n, device='cuda', generator=g) * 2
        if relu: x = torch.relu(x)
        for bins in (4096, 2048, 50):
            hs = float(x.abs().max().item()) / bins
            for clip in (True, False):
                a = torch.zeros(bins, dtype=torch.int32, device='cuda'); b = torch.zeros_like(a)
                ext.Histogram_T(x, hs, clip, a); ref.Histogram_T(x, hs, clip, b)
                assert torch.equal(a, b), (n, bins, clip)
                a.zero_(); b.zero_()
                mn, mx = float(x.min().item()), float(x.max().item())
                ext.Histogram_Asymmetric_T(mn, mx, x, clip, a); ref.Histogram_Asymmetric_T(mn, mx, x, clip, b)
                assert torch.equal(a, b), (n, bins, clip, 'asym')
    x = torch.randn(4, 8, 1000, device='cuda', generator=g)
    for axis in (0, 1):
        C = x.shape[axis]
        a = torch.zeros(C, 128, dtype=torch.int32, device='cuda'); b = torch.zeros_like(a)
        ext.Histogram_C(x, axis, 0.03, True, a); ref.Histogram_C(x, axis, 0.03, True, b)
        assert torch.equal(a, b), axis


def test_compute_mse_loss_vs_reference(ref, ext):
    r = np.random.RandomState(5)
    for _ in range(50):
        h = r.randint(0, 9000, size=2048).tolist()
        step = int(r.randint(1, 9)); start = int(r.randint(0, 512)); end = start + 256 * step
        assert ext.compute_mse_loss(h, start, step, end) == ref.compute_mse_loss(h, start, step, end)
