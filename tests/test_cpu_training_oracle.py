"""CPU pins of the oracle's restatements of the training-pass kernels (LSQ backward, float backward, TensorClip, RoundingLoss and its
backward).  Upstream has no CPU implementation of them, so they are pinned against the torch formulas of the reference's own test
(tests/test_cuda_kernel.py:66-143 upstream), evaluated here on CPU tensors for round-half-even and integer offsets, and against
hand-worked answers for each quirk those formulas cannot see: the two offset roundings, RoundingLoss_LC's unrounded clip test, the
clip boundaries, the widened range of the float backward, NaN, and the normalisers."""
import math

import numpy as np
import pytest
import torch

F32 = np.float32


def lsq_torch(value, dy, scale, offset, qmin, qmax, axis=None):
    """The reference's torch formula (tests/test_cuda_kernel.py:67-79 / 99-114 upstream): grad_x and the per-element grad_s terms."""
    if axis is not None:
        shape = [1 if a != axis else -1 for a in range(value.ndim)]
        scale, offset = scale.view(shape), offset.view(shape)
    qt = torch.round(value / scale) + offset
    cl = qt.clip(qmin, qmax)
    dx = torch.where(cl != qt, torch.zeros_like(dy), dy)
    ds = torch.where(cl == qt, (((qt - offset) * scale) - value) * dy / scale, torch.zeros_like(dy))
    ds = ds + torch.where(qt > qmax, (qmax - offset) * dy, torch.zeros_like(dy))
    ds = ds + torch.where(qt < qmin, (qmin - offset) * dy, torch.zeros_like(dy))
    return dx, ds


def rounding_loss_torch(value, scale, offset, qmin, qmax, dy0, axis=None):
    """train.cu:125-141 / 181-192 upstream as torch ops: (per-element diffs, gradient)."""
    if axis is not None:
        shape = [1 if a != axis % value.ndim else -1 for a in range(value.ndim)]
        scale, offset = scale.view(shape), offset.view(shape)
    q = torch.clamp(torch.round(value / scale) + offset, qmin, qmax)
    deq = (q - offset) * scale
    clipped = (value > scale * (qmax - offset)) | (value < scale * (qmin - offset))
    diff = torch.where(clipped, torch.zeros_like(value), (deq - value).abs())
    grad = torch.where(clipped, torch.zeros_like(value), torch.where(value > deq, 1.0, -1.0) * dy0)
    return diff, grad / torch.sqrt(torch.tensor(float(value.numel())))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize('shape,axis', [([7], None), ([4, 6, 5, 3], None), ([4, 6, 5, 3], 1), ([9, 4], 0), ([2, 3, 11], 2)])
@pytest.mark.parametrize('qmin,qmax', [(0, 255), (-128, 127), (-8, 7), (0, 15)])
def test_lsq_backward_matches_the_torch_formula(oracle, shape, axis, qmin, qmax):
    r = np.random.RandomState(len(shape) * 100 + qmax)
    C = 1 if axis is None else shape[axis]
    s = (r.rand(C) * 0.2 + 0.01).astype(F32)
    o = r.randint(qmin, qmax + 1, C).astype(F32)
    x = ((r.rand(*shape) - 0.5) * (qmax - qmin + 8) * s.max()).astype(F32)
    dy = r.randn(*shape).astype(F32)
    gx, p, f = oracle.linear_quant_backward(x, dy, s, o, qmin, qmax, 0, axis)
    dx, ds = lsq_torch(torch.from_numpy(x), torch.from_numpy(dy), torch.from_numpy(s), torch.from_numpy(o), qmin, qmax, axis)
    assert np.array_equal(bits(gx), bits(dx.numpy()))
    if axis is None:
        assert np.array_equal(bits(p + F32(0)), bits(ds.numpy()))          # same association: (q - v) * dy / s; the formula's adds turn -0 into +0
    else:
        assert np.allclose(p, ds.numpy(), rtol=1e-6, atol=1e-7)            # the LC kernel associates (q - v) / s * dy
    den = x.size * (qmax - qmin if axis is None else qmax)
    assert f == F32(1 / math.sqrt(den))


@pytest.mark.parametrize('axis', [None, 0, 1, -1])
@pytest.mark.parametrize('qmin,qmax', [(-128, 127), (0, 255), (-8, 7)])
def test_rounding_loss_matches_the_torch_formula(oracle, axis, qmin, qmax):
    r = np.random.RandomState(qmax + (axis or 0) + 7)
    shape = [3, 5, 17]
    C = 1 if axis is None else shape[axis]
    s = (r.rand(C) * 0.1 + 0.01).astype(F32)
    o = r.randint(-3, 4, C).astype(F32)
    x = (r.randn(*shape) * 3).astype(F32)
    x.reshape(-1)[:4] = s[0] * (qmax - o[0]), s[0] * (qmin - o[0]), s[0] * (2.5 - o[0]), 0.0      # clip bounds and a tie of channel 0
    dy0 = F32(0.7)
    p, d = oracle.rounding_loss(x, s, o, qmin, qmax, 0, axis)
    g = oracle.rounding_loss_backward(x, [dy0], s, o, qmin, qmax, 0, axis)
    diff, grad = rounding_loss_torch(torch.from_numpy(x), torch.from_numpy(s), torch.from_numpy(o), qmin, qmax, float(dy0), axis)
    assert np.array_equal(bits(p), bits(diff.numpy())) and np.array_equal(bits(g), bits(grad.numpy()))
    assert d == np.sqrt(F32(x.size))


@pytest.mark.parametrize('axis', [None, 1])
def test_tensor_clip_matches_torch(oracle, axis):
    r = np.random.RandomState(3)
    v, ref = r.randn(4, 6, 5).astype(F32), r.randn(4, 6, 5).astype(F32)
    lim = r.rand(1 if axis is None else 6).astype(F32)
    view = [1, -1, 1] if axis is not None else [1, 1, 1]
    tv, tr, tl = torch.from_numpy(v), torch.from_numpy(ref), torch.from_numpy(lim).view(view)
    want = torch.minimum(torch.maximum(tv, tr - tl), tr + tl).numpy()
    assert np.array_equal(bits(oracle.tensor_clip(v, ref, lim, axis)), bits(want))


def test_tensor_clip_known_answers(oracle):
    """CLIP tests `v > hi` before `v < lo` (common.cuh:72-76 upstream)."""
    nan = F32('nan')
    cases = [  # v, reference, limit -> out
        (F32(-0.0), F32(0.0), F32(0.0), F32(-0.0)),     # neither test fires: v itself, sign kept
        (F32(5.0), F32(0.0), F32(-1.0), F32(-1.0)),     # negative limit: lo = 1 > hi = -1, `> hi` wins
        (F32(-5.0), F32(0.0), F32(-1.0), F32(1.0)),
        (F32(0.0), F32(0.0), F32(-1.0), F32(-1.0)),
        (nan, F32(0.0), F32(1.0), nan),
        (F32(3.0), nan, F32(1.0), F32(3.0)),            # NaN bounds: both comparisons false
        (F32(3.0), F32(0.0), nan, F32(3.0)),
        (F32('inf'), F32(0.0), F32('inf'), F32('inf')),
        (F32(2.0), F32('inf'), F32(1.0), F32('inf')),   # lo = hi = inf
    ]
    for v, ref, lim, want in cases:
        got = oracle.tensor_clip([v], [ref], [lim])[0]
        assert bits([got])[0] == bits([want])[0] or (np.isnan(got) and np.isnan(want)), (v, ref, lim, got, want)


def test_offset_roundings_known_answers(oracle):
    """LSQ rounds the offset with roundf (half away from zero), RoundingLoss with nearbyint (half to even)."""
    one, dy = [F32(1.0)], [F32(1.0)]
    # LSQ, x = 0, s = 1: offset 2.5 -> o = 3, qt = 3 > qmax = 2: clipped, partial (2 - 3) * dy   (nearbyint would give o = 2: not clipped)
    gx, p, _ = oracle.linear_quant_backward([0.0], dy, one, [2.5], 0, 2)
    assert gx[0] == 0.0 and p[0] == -1.0
    # offset -0.5 -> o = -1, qt = -1 < qmin = 0: clipped, partial (0 - (-1)) * dy                 (nearbyint: o = -0, qt = 0, partial 0)
    gx, p, _ = oracle.linear_quant_backward([0.0], dy, one, [-0.5], 0, 2)
    assert gx[0] == 0.0 and p[0] == 1.0
    # offset 3.5 -> o = 4 (roundf) and qt = round(0.75) + 4 = 5 = qmax: q = float(5 - 4) * 1, partial (1 - 0.75) * dy
    gx, p, _ = oracle.linear_quant_backward([0.75], dy, one, [3.5], 0, 5)
    assert gx[0] == 1.0 and p[0] == 0.25
    # RoundingLoss_LT, x = 0.8, s = 1, qmax = 3: offset 2.5 -> o = 2 (nearbyint): q = 3, deq = 1, bound 1 * (3 - 2) = 1, not clipped
    p, _ = oracle.rounding_loss([0.8], one, [2.5], -128, 3)
    assert p[0] == F32(1.0) - F32(0.8)                      # with roundf (o = 3): deq = 0, bound 0 -> clipped, 0
    p, _ = oracle.rounding_loss([0.8], one, [3.5], -128, 4)  # 3.5 -> 4: q = 1 + 4 clipped to 4, deq = 0, bound 0 -> clipped
    assert p[0] == 0.0
    p, _ = oracle.rounding_loss([-0.3], one, [-0.5], -1, 3)  # -0.5 -> -0: q = 0, deq = 0, bound -1: |0 - (-0.3)|
    assert p[0] == F32(0.3)


def test_rounding_loss_lc_clips_with_the_unrounded_offset(oracle):
    one = [F32(1.0)]
    # offset 2.5, qmax 3, x = 0.8: q = round(0.8) + 2 = 3, deq = 1.  Per tensor the bound is 1 * (3 - 2) = 1 -> kept;
    # per channel it is 1 * (3 - 2.5) = 0.5 -> 0.8 is "clipped" and contributes nothing, and its gradient is 0.
    pt, _ = oracle.rounding_loss([0.8], one, [2.5], -128, 3)
    pc, _ = oracle.rounding_loss(np.array([0.8], F32), one, [2.5], -128, 3, 0, 0)
    assert pt[0] > 0 and pc[0] == 0.0
    gt = oracle.rounding_loss_backward([0.8], [1.0], one, [2.5], -128, 3)
    gc = oracle.rounding_loss_backward(np.array([0.8], F32), [1.0], one, [2.5], -128, 3, 0, 0)
    assert gt[0] == -1.0 and gc[0] == 0.0                 # 0.8 < deq = 1 -> -1 * dy / sqrt(1)


def test_rounding_loss_clip_boundary_and_neighbours(oracle):
    """v exactly at s * (qmax - o) is not clipped (the test is `>`): deq == v, so the gradient is -dy; one ulp above is clipped."""
    s, o, qmax = F32(0.1), F32(3.0), 127
    b = s * F32(qmax - 3)
    xs = np.array([np.nextafter(b, F32(0)), b, np.nextafter(b, F32(1e9))], F32)
    sq = np.sqrt(F32(1))
    for x, want in zip(xs, [None, -1.0, 0.0]):
        g = oracle.rounding_loss_backward([x], [1.0], [s], [o], -128, qmax)[0]
        if want is not None:
            assert g == F32(want) / sq, (x, g)
    lo = s * F32(-128 - 3)
    assert oracle.rounding_loss_backward([lo], [1.0], [s], [o], -128, qmax)[0] != 0.0
    assert oracle.rounding_loss_backward([np.nextafter(lo, F32(-1e9))], [1.0], [s], [o], -128, qmax)[0] == 0.0


def test_lsq_clip_boundary_known_answers(oracle):
    """LSQ clips on the rounded integer: (qmax - o + 0.5) * s is a tie (half-even decides), one ulp either side is not."""
    s, o, qmax = F32(0.25), F32(1.0), 6
    t = F32(qmax - 1) + F32(0.5)                            # 5.5 -> 6 (even) + 1 = 7 > 6: clipped
    for x, clipped in [(t * s, True), (np.nextafter(t, F32(0)) * s, False), (np.nextafter(t, F32(9)) * s, True),
                       (F32(4.5) * s, False)]:          # 4.5 -> 4 (even) + 1 = 5: kept
        gx, p, _ = oracle.linear_quant_backward([x], [1.0], [s], [o], 0, qmax)
        assert (gx[0] == 0.0) == clipped, (x, gx, p)
        if clipped: assert p[0] == F32(qmax) - o
    # mode HALF_UP sends 4.5 up and HALF_DOWN sends 5.5 down: the mode reaches the backward
    gx, _, _ = oracle.linear_quant_backward([t * s], [1.0], [s], [o], 0, qmax, 2)
    assert gx[0] == 1.0


def test_float_backward_known_answers(oracle):
    """E4M3, s = 1, o = 0.  The backward quantises into [cmin - 1, cmax + 1] (floating.cu:159-160 upstream); an element is saturated
    only when that quantiser returns a widened bound exactly."""
    dy = [F32(0.5)]
    one, zero = [F32(1.0)], [F32(0.0)]

    def fb(u, cmin=-448.0, cmax=448.0, o=zero, mode=0):
        gx, p, d = oracle.float_quant_backward([u], dy, one, o, 4, 3, cmin, cmax, mode)
        return gx[0], p[0], d

    gx, p, _ = fb(449.0)             # exactly cmax + 1: not > 449, its mantissa rounds down to 448 on the grid -> not saturated
    assert gx == 0.5 and p == (F32(448) - F32(449)) * F32(0.5)
    gx, p, _ = fb(448.5)             # inside (cmax, cmax + 1]: rounds to 448, kept
    assert gx == 0.5 and p == F32(-0.25)
    gx, p, _ = fb(449.5)             # beyond cmax + 1: returns 449 -> saturated, partial s * (cmax - o) * dy / s
    assert gx == 0.0 and p == F32(448) * F32(0.5)
    gx, p, _ = fb(-460.0)
    assert gx == 0.0 and p == F32(-448) * F32(0.5)
    gx, p, _ = fb(448.0)             # on the grid at cmax: not saturated (it would be without the widening)
    assert gx == 0.5 and p == 0.0
    # clip 480 = tmax: cmax + 1 = 481 is beyond the format, the quantiser saturates at 480 != 481, so saturated values keep dy
    gx, p, _ = fb(500.0, -480.0, 480.0)
    assert gx == 0.5 and p == (F32(480) - F32(500)) * F32(0.5)
    # off-grid clip 300: widened 301 is returned for u > 301 (saturated) while u = 300.5 rounds to the grid value 288 or 320,
    # and the final CLIP of the quantiser brings 320 back to 301 -- which then counts as saturated
    assert oracle.float_quant_scalar(310.0, 1.0, 4, 3, -301.0, 301.0) == 301.0
    gx, p, _ = fb(310.0, -300.0, 300.0)
    assert gx == 0.0 and p == F32(300) * F32(0.5)
    # NaN: the canonical device NaN goes through the mantissa carry and becomes -0.0 for E4M3; the element keeps dy, its partial is NaN
    assert math.copysign(1.0, oracle.float_quant_scalar(float('nan'), 1.0, 4, 3, -449.0, 449.0)) == -1.0
    gx, p, _ = fb(float('nan'), o=[F32(2.0)])
    assert gx == 0.5 and np.isnan(p)
    # the offset only shifts the dequantised value: u = 10 -> qt = 10, q = (10 - 2) * 1, partial (8 - 10) * dy
    gx, p, _ = fb(10.0, o=[F32(2.0)])
    assert gx == 0.5 and p == F32(-1.0)


def test_normalisers(oracle):
    """LSQ: the host's rsqrtf, i.e. 1 / sqrt in double rounded once; that is not 1.0f / sqrtf(float) -- n = 1, range 127 tells them
    apart.  The float backward divides by sqrtf(n * cmax), RoundingLoss by sqrtf(n)."""
    one = [F32(1.0)]
    _, _, f = oracle.linear_quant_backward([0.3], one, one, [0.0], -127, 0)
    assert f == F32(1 / math.sqrt(127)) and f != F32(1) / np.sqrt(F32(127))
    _, _, f = oracle.linear_quant_backward([0.3], one, one, [0.0], -128, 127, 0, 0)        # per channel: n * qmax
    assert f == F32(1 / math.sqrt(127))
    _, _, f = oracle.linear_quant_backward([0.3], one, one, [0.0], -2 ** 31, 2 ** 31 - 1)   # qmax - qmin wraps to -1: NaN
    assert np.isnan(f)
    _, _, f = oracle.linear_quant_backward(np.zeros((1, 3), F32), np.ones((1, 3), F32), one, [0.0], 0, 2 ** 31 - 1, 0, 0)
    assert f == F32(1 / math.sqrt(float(F32(3.0 * (2 ** 31 - 1)))))
    _, _, d = oracle.float_quant_backward(np.zeros(3, F32), np.ones(3, F32), one, [0.0], 4, 3, -448.0, 448.0)
    assert d == np.sqrt(F32(3) * F32(448))
    _, d = oracle.rounding_loss(np.zeros(5, F32), one, [0.0], -128, 127)
    assert d == np.sqrt(F32(5))


def test_saturating_quotients_and_wrapping_offsets(oracle):
    """Quotients beyond int32 saturate in the conversion; the full int32 range then keeps them (qt == INT_MAX is not > qmax)."""
    one = [F32(1.0)]
    gx, p, _ = oracle.linear_quant_backward([3e38], one, [1e-3], [0.0], -2 ** 31, 2 ** 31 - 1)
    assert gx[0] == 1.0 and p[0] == -np.inf                # q = float(INT_MAX) * s, (q - v) * dy / s overflows
    gx, p, _ = oracle.linear_quant_backward([3e38], one, [1e-3], [0.0], 0, 255)
    assert gx[0] == 0.0 and p[0] == 255.0
    gx, p, _ = oracle.linear_quant_backward([float('nan')], one, one, [0.0], 0, 255)   # NaN -> round2int 0 -> kept, NaN partial
    assert gx[0] == 1.0 and np.isnan(p[0])
    # RoundingLoss: round2int(x / s) + o wraps in int; x = 3e9 * s saturates to INT_MAX, + 5 wraps negative and clips to qmin
    p, _ = oracle.rounding_loss([3e9], one, [5.0], -2 ** 31, 2 ** 31 - 1)
    assert p[0] == 0.0                                     # the clip test bound s * float(qmax - 5) is < 3e9: clipped
    g = oracle.rounding_loss_backward([3e9], [1.0], one, [5.0], -2 ** 31, 2 ** 31 - 1)
    assert g[0] == 0.0
