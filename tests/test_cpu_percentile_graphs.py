"""The static per-batch rows of the percentile arena (ArenaCalibrator(max_batches=S)), driven on host tensors with the select replaced by a
stub that returns known {upper, lower} pairs: what calibrate_arena(method='percentile', graphs=True) replays on the device.

  * every end_batch() files the staging row as row `counter` and advances the counter, so rows land in batch order;
  * the rendered scales are the mean of the list-based calibrator (graphs=False) bit for bit, for S = 1 ... 17 batches;
  * a batch past max_batches raises in begin_batch(), before any select or scatter, and leaves rows and counter as they were;
  * replay_state() names the counter and the guess rows, and reset() starts the counter from zero."""
import types

import numpy as np
import pytest
import torch

T = 5
Q = 0.9999


def pairs(S, seed=7):
    """[S, T, 2] {upper, lower} of batch s, slot t: fp32 values with ragged exponents, so a different summation order would show."""
    r = np.random.RandomState(seed + S)
    up = (r.standard_normal((S, T)) * 10.0 ** r.randint(-3, 4, (S, T))).astype(np.float32)
    lo = -(np.abs(r.standard_normal((S, T))) * 10.0 ** r.randint(-3, 4, (S, T))).astype(np.float32)
    return torch.from_numpy(np.stack([up, lo], axis=-1))


class StubExt:
    """The bindings the percentile arena calls.  A 'tensor' is [batch, slot]; the select returns that batch's known pair."""

    def __init__(self, table):
        self.table, self.calls = table, []

    def _pair(self, x):
        s, t = (int(v) for v in x.tolist())
        return self.table[s, t].clone()

    def Quantile_T(self, x, q):
        assert q == Q
        self.calls.append(('Quantile_T', tuple(x.tolist())))
        return self._pair(x)

    def Quantile_T_Guess(self, x, q, guess):
        assert q == Q and guess.dtype == torch.int32 and guess.numel() == 8
        self.calls.append(('Quantile_T_Guess', tuple(x.tolist()), guess.data_ptr()))
        return self._pair(x)

    def MinMax_To_Scale_Offset(self, maxs, mins, stride, qmin, qmax, sym, p2, min_scale):
        return maxs.clone(), mins.clone()                                  # the averaged pair itself: what the test compares


def calibrator(monkeypatch, table, max_batches=None):
    import ppq_b200.ffi as ffi
    from ppq_b200.calibration import ArenaCalibrator
    stub = StubExt(table)
    monkeypatch.setattr(ffi, 'extension', lambda: stub)
    cal = ArenaCalibrator(T, 'cpu', method='percentile', percentile=Q, max_batches=max_batches)
    if max_batches is not None:
        cal._select_guess = torch.zeros(T, 8, dtype=torch.int32)           # Quantile_Guess_Init's rows on a device
    return cal, stub


def forward(cal, s):
    """One batch: every slot observed as the forward produces it, then the end-of-forward scatter (a no-op without static rows)."""
    cal.begin_batch()
    for t in range(T): cal.observe_one(t, torch.tensor([s, t], dtype=torch.float32))
    cal.end_batch()


def test_rows_land_in_batch_order(monkeypatch):
    S = 6
    table = pairs(S)
    cal, stub = calibrator(monkeypatch, table, max_batches=S)
    assert cal._rows.shape == (S, T, 2) and int(cal._count.item()) == 0
    for s in range(S):
        forward(cal, s)
        assert int(cal._count.item()) == s + 1
        assert torch.equal(cal._rows[s], table[s]), s
        assert torch.equal(cal._rows[s + 1:], torch.zeros(S - s - 1, T, 2)), s
    assert torch.equal(cal.batch_rows(), table.transpose(0, 1)) and cal.batch_rows().is_contiguous()
    guess_rows = [cal._select_guess[t].data_ptr() for t in range(T)]
    assert [c[0] for c in stub.calls] == ['Quantile_T_Guess'] * (S * T)
    assert [c[2] for c in stub.calls] == guess_rows * S                       # slot t always selects through guess row t


@pytest.mark.parametrize('S', list(range(1, 18)))
def test_mean_equals_the_list_based_mean(monkeypatch, S):
    table = pairs(S)
    eager, estub = calibrator(monkeypatch, table)
    for s in range(S): forward(eager, s)
    assert [c[0] for c in estub.calls] == ['Quantile_T'] * (S * T)           # graphs=False keeps its select
    assert eager.end_phase()
    static, _ = calibrator(monkeypatch, table, max_batches=S)
    for s in range(S): forward(static, s)
    assert static.end_phase()
    assert torch.equal(static.batch_rows(), eager.batch_rows())
    # the reference's reduction per tensor (range.py:369): torch.cat(collector, dim=0).float().mean(dim=0)
    want = torch.stack([torch.cat([table[s, t][None] for s in range(S)], dim=0).float().mean(dim=0) for t in range(T)])
    for cal in (eager, static):
        assert torch.equal(cal.scale.view(torch.int32), want[:, 1].contiguous().view(torch.int32)), S
        assert torch.equal(cal.offset.view(torch.int32), want[:, 0].contiguous().view(torch.int32)), S


def test_overrun_raises_before_anything_is_written(monkeypatch):
    S = 3
    table = pairs(S + 1)
    cal, stub = calibrator(monkeypatch, table, max_batches=S)
    for s in range(S): forward(cal, s)
    rows, staging, calls = cal._rows.clone(), cal._staging.clone(), len(stub.calls)
    with pytest.raises(RuntimeError, match='overruns the 3 per-batch rows'):
        forward(cal, S)
    assert torch.equal(cal._rows, rows) and torch.equal(cal._staging, staging)
    assert int(cal._count.item()) == S and len(stub.calls) == calls
    assert cal.end_phase() and torch.equal(cal.batch_rows(), table[:S].transpose(0, 1))


def test_no_batch_raises_the_empty_collector_error(monkeypatch):
    cal, _ = calibrator(monkeypatch, pairs(1), max_batches=0)
    with pytest.raises(ValueError, match='collator is empty'):
        cal.end_phase()


def test_replay_state_and_reset(monkeypatch):
    S = 4
    cal, _ = calibrator(monkeypatch, pairs(S), max_batches=S)
    state = cal.replay_state()
    assert any(t is cal._count for t in state) and any(t is cal._select_guess for t in state)
    for s in range(S): forward(cal, s)
    cal.reset()
    assert int(cal._count.item()) == 0
    for s in range(S): forward(cal, s)                                         # a second pass fits again
    assert int(cal._count.item()) == S
    eager, _ = calibrator(monkeypatch, pairs(S))
    assert not any(t is eager._count or t is eager._select_guess for t in eager.replay_state() if t is not None)
    assert len(eager.replay_state()) == 2                                      # minmax and hist, as for kl / minmax / mse


def test_static_rows_are_percentile_only(monkeypatch):
    import ppq_b200.ffi as ffi
    from ppq_b200.calibration import ArenaCalibrator
    monkeypatch.setattr(ffi, 'extension', lambda: types.SimpleNamespace())
    for method in ('kl', 'minmax', 'mse'):
        with pytest.raises(ValueError, match='max_batches'):
            ArenaCalibrator(T, 'cpu', method=method, max_batches=4)
    with pytest.raises(ValueError, match='max_batches'):
        ArenaCalibrator(T, 'cpu', method='percentile', max_batches=-1)
