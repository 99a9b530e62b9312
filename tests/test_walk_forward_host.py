"""Host side of the walk-forward analysis (ai_crypto_trader_b200/walk_forward.py), without a GPU: window plans on the
market's calendar, the segment tables the driver builds, the seed rule, the reference's gate at every risk level and the
efficiency arithmetic."""
import math

import numpy as np
import pytest

from ai_crypto_trader_b200 import _lib, walk_forward as wf

DAY = 1440
M0 = 19_723 * DAY                   # 2024-01-01T00:00


def _day(minute0, bar_minutes, t):
    return (minute0 + t * bar_minutes) // DAY


def _check_plan(plan, minute0, bar_minutes, N, is_days, oos_days, anchored):
    d0 = minute0 // DAY
    for k, (a, b, c, d) in enumerate(plan):
        assert b == c and a < b < d <= N
        # boundary k: the first bar of day d0 + is_days + k * oos_days
        assert _day(minute0, bar_minutes, b) >= d0 + is_days + k * oos_days
        assert b == 0 or _day(minute0, bar_minutes, b - 1) < d0 + is_days + k * oos_days
        if anchored:
            assert a == 0
        else:
            assert _day(minute0, bar_minutes, a) >= d0 + k * oos_days
            assert a == 0 or _day(minute0, bar_minutes, a - 1) < d0 + k * oos_days
        if k + 1 < len(plan):
            assert d == plan[k + 1][2]
    assert plan[-1][3] == N


@pytest.mark.parametrize("anchored", [False, True])
def test_rolling_and_anchored_plans(anchored):
    N = 60 * DAY
    plan = wf.plan_windows(M0, 1, N, 30, 7, anchored)
    assert len(plan) == 5                                   # boundaries on days 30, 37, 44, 51, 58
    assert plan[0] == (0, 30 * DAY, 30 * DAY, 37 * DAY)
    assert plan[-1] == ((28 if not anchored else 0) * DAY, 58 * DAY, 58 * DAY, N)    # short last window: 2 days
    _check_plan(plan, M0, 1, N, 30, 7, anchored)


def test_minute0_not_at_midnight_and_five_minute_bars():
    m0 = M0 + 13 * 60 + 7                                  # 13:07 on day d0
    N = 40 * DAY // 5
    plan = wf.plan_windows(m0, 5, N, 10, 3, False)
    _check_plan(plan, m0, 5, N, 10, 3, False)
    # the first window starts at bar 0 (day d0's first bar), the first boundary is midnight of day d0 + 10
    assert plan[0][0] == 0
    assert (m0 + plan[0][1] * 5) % DAY < 5 and _day(m0, 5, plan[0][1]) == m0 // DAY + 10
    # day d0 is short (from 13:07): window 0's in-sample bars span 9 days 10:53, rounded up to whole 5-minute bars
    assert plan[0][1] == -(-(10 * DAY - (13 * 60 + 7)) // 5)


def test_plan_refuses_a_market_too_short():
    with pytest.raises(ValueError):
        wf.plan_windows(M0, 1, 30 * DAY, 30, 7)             # ends exactly at the first boundary
    assert len(wf.plan_windows(M0, 1, 30 * DAY + 1, 30, 7)) == 1    # one out-of-sample bar
    with pytest.raises(ValueError):
        wf.plan_windows(M0, 1, 100, 0, 7)


def _valid(seg, begin, j, N, n_indiv):
    rows = seg[begin[j]:begin[j + 1]]
    if len(rows) == 0:
        return False
    prev_end = -1
    for start, end, ind, reserved in rows.tolist():
        if start < 0 or end <= start or end > N or start < prev_end or not 0 <= ind < n_indiv or reserved != 0:
            return False
        prev_end = end
    return True


@pytest.mark.parametrize("anchored", [False, True])
def test_the_driver_builds_valid_schedules(anchored):
    N = 50 * DAY // 15
    plan = wf.plan_windows(M0 + 301, 15, N, 20, 5, anchored)
    pop = 7
    seg, begin = wf.segment_tables(wf.ga_schedules([(a, b) for a, b, _, _ in plan], pop))
    assert seg.dtype == np.dtype(_lib.SEGMENT_DTYPE) and seg.shape == (len(plan) * pop,) and begin.dtype == np.int32
    assert all(_valid(seg, begin, j, N, len(plan) * pop) for j in range(len(plan) * pop))
    assert sorted(seg["individual"].tolist()) == list(range(len(plan) * pop))
    sched = wf.scoring_schedules(plan)
    seg, begin = wf.segment_tables(sched)
    K = len(plan)
    assert len(sched) == 2 * K + 1 and begin[1] == K and begin[-1] == 3 * K
    assert all(_valid(seg, begin, j, N, K) for j in range(2 * K + 1))
    # the stitched schedule covers every out-of-sample bar once, from the first boundary to N
    st = seg[:K]
    assert st["start"][0] == plan[0][2] and st["end"][-1] == N and np.all(st["start"][1:] == st["end"][:-1])


def test_seed_rule():
    assert [wf.window_seed(5, w) for w in range(3)] == [5, 6, 7]
    assert wf.window_seed(None, 4) == 4
    assert wf.window_seed(2 ** 64 - 2, 3) == 1                     # mod 2^64


@pytest.mark.parametrize("level, sharpe, dd, wr", [("LOW", 1.5, 10.0, 0.57), ("MEDIUM", 1.2, 15.0, 0.52),
                                                   ("HIGH", 0.9, 20.0, 0.47)])
def test_gate_at_each_risk_level(level, sharpe, dd, wr):
    t = wf.risk_thresholds()[level]
    assert t["min_sharpe_ratio"] == pytest.approx(sharpe) and t["max_drawdown"] == dd and t["min_win_rate"] == pytest.approx(wr)
    ok = {"sharpe_ratio": sharpe + 0.01, "drawdown": dd, "win_rate": wr + 0.01}
    assert not wf.needs_improvement(ok, t)
    assert wf.needs_improvement(dict(ok, sharpe_ratio=sharpe - 0.01), t)
    assert wf.needs_improvement(dict(ok, drawdown=dd + 0.01), t)
    assert wf.needs_improvement(dict(ok, win_rate=wr - 0.01), t)
    # the reference's defaults: no drawdown key reads as 100 and fires; an empty dict does not
    assert wf.needs_improvement({"sharpe_ratio": 9.0, "win_rate": 0.9}, t)
    assert not wf.needs_improvement({}, t)


def test_risk_thresholds_follow_the_config_block():
    t = wf.risk_thresholds({"min_sharpe_ratio": 2.0, "max_drawdown": 30.0, "min_win_rate": 0.6,
                            "risk_management": {"max_position_size": 0.2}}, leverage_trading=True)
    assert t["LOW"]["min_sharpe_ratio"] == pytest.approx(2.3) and t["HIGH"]["max_drawdown"] == 35.0
    assert t["MEDIUM"]["min_win_rate"] == 0.6
    assert t["MEDIUM"]["position_size_pct"] == pytest.approx(0.1) and t["HIGH"]["position_size_pct"] == pytest.approx(0.15)


def test_gate_performance_reads_percent_drawdown():
    stats = {"sharpe_ratio": np.array([1.0, 2.0]), "win_rate": np.array([0.5, 0.6]), "max_drawdown": np.array([0.1, 0.2])}
    perf = wf.gate_performance(stats)
    assert perf == {"sharpe_ratio": 1.5, "win_rate": pytest.approx(0.55), "drawdown": pytest.approx(15.0)}


def test_efficiency_arithmetic():
    assert wf.efficiency(70.0, 7.0, 300.0, 30.0) == pytest.approx(1.0)
    assert wf.efficiency(-35.0, 7.0, 300.0, 30.0) == pytest.approx(-0.5)
    assert wf.efficiency(10.0, 3.5, 100.0, 10.0) == pytest.approx(10.0 / 3.5 / 10.0)
    assert math.isnan(wf.efficiency(70.0, 7.0, 0.0, 30.0))          # in-sample net profit <= 0
    assert math.isnan(wf.efficiency(70.0, 7.0, -5.0, 30.0))
    assert math.isnan(wf.efficiency(70.0, 7.0, float("nan"), 30.0))
    assert math.isnan(wf.efficiency(70.0, 0.0, 300.0, 30.0))


def test_fitness_of_is_the_reduce_expression():
    assert wf._fitness_of([1.0, 2.0, 4.0]) == (0.0 + 1.0 + 2.0 + 4.0) / 3
    assert math.isnan(wf._fitness_of([1.0, float("nan")]))


def _generation_best_loop(fitness, best):
    """DeviceGeneticAlgorithm.evaluate_population / record_generation, row by row."""
    best = best.copy()
    improved, keep, hi, lo, mean = [], [], [], [], []
    for w, row in enumerate(fitness.tolist()):
        k = None
        for i, f in enumerate(row):
            if f > best[w]:
                best[w], k = f, i
        improved.append(k is not None)
        keep.append(k)
        hi.append(max(row))
        lo.append(min(row))
        mean.append(sum(row) / len(row))
    return improved, keep, best, hi, lo, mean


def test_generation_best_is_the_row_walk():
    rng = np.random.default_rng(3)
    for trial in range(50):
        W, pop = int(rng.integers(1, 6)), int(rng.integers(1, 40))
        fit = rng.normal(size=(W, pop)).round(int(rng.integers(0, 3)))       # ties when rounded
        fit[rng.random((W, pop)) < 0.2] = np.nan
        if trial % 5 == 0:
            fit[:, 0] = np.nan
        if trial % 7 == 0:
            fit[0] = -np.inf
        best = np.where(rng.random(W) < 0.5, -np.inf, rng.normal(size=W))
        improved, keep, new_best, hi, lo, mean = wf.generation_best(fit, best)
        want = _generation_best_loop(fit, best)
        assert improved.tolist() == want[0]
        assert [int(k) for k, i in zip(keep, improved) if i] == [k for k in want[1] if k is not None]
        np.testing.assert_array_equal(new_best, want[2])
        for got, exp in zip((hi, lo, mean), want[3:]):
            np.testing.assert_array_equal(got, np.array(exp))
