"""The book oracle (tests/book_ref.py: C-oracle lanes merged in (bar, symbol, record) order) against the Python
restatement of the reference rules (oracle/simulate_ref.py) and the host StrategyPerformanceMetrics, each given the ONE
concatenated trade list evaluate_strategy hands to calculate_metrics; and the argument checks of b200bt_book_metrics.
CPU only."""
import ctypes as C

import numpy as np
import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE

PERIODS = (5, 9, 14)
SOURCE = [0, 1, 0, 2]            # symbols 0 and 2 are the same series: their records tie on the same bars


def _case(n_bars, bar_minutes):
    from ai_crypto_trader_b200 import synth
    from oracle import indicators_ref
    close = np.ascontiguousarray(synth.synth_ohlcv(3, n_bars)[3][SOURCE])
    bank = np.stack([indicators_ref.rsi_bank(close[s], PERIODS) for s in range(len(SOURCE))])
    bank[3] = np.nan                                       # symbol 3 never trades (no compare with NaN is true)
    pop = synth.random_population(8, seed=4)
    for p in pop:
        p["rsi_period"] = PERIODS[int(p["rsi_period"]) % len(PERIODS)]
    pop += [dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001),
            dict(rsi_period=9, rsi_oversold=0, rsi_overbought=100)]
    return close, bank, pop, synth.EPOCH_2024_MINUTES


@pytest.mark.parametrize("bar_minutes", [1, 1440])
def test_book_oracle_matches_the_reference_rules_on_one_trade_list(bar_minutes):
    import book_ref
    from ai_crypto_trader_b200.strategy_evaluation import StrategyPerformanceMetrics
    from oracle import sim_oracle, simulate_ref
    close, bank, pop, minute0 = _case(1500, bar_minutes)
    goals = {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"]}
    cfg = sim_oracle.config_of(minute0, bar_minutes, goals=goals)
    row = {p: i for i, p in enumerate(PERIODS)}
    crossing = 0
    for p in pop:
        evs, pns, trades = [], [], []
        for s in range(len(SOURCE)):
            rsi = bank[s, row[p["rsi_period"]]]
            _, ev, pn = sim_oracle.lane(close[s], rsi, p, cfg, event_cap=len(close[s]) + 2)
            evs.append(ev)
            pns.append(pn)
            trades += simulate_ref.simulate_trades(p, simulate_ref.market_points(close[s], rsi, f"S{s}", minute0, bar_minutes))
        got = book_ref.book(evs, pns, cfg)
        rec = book_ref.merged(evs, pns)
        crossing += sum(rec[i][1] != rec[i + 1][1] for i in range(0, len(rec) - 1, 2))
        for want in (simulate_ref.calculate_metrics(trades), StrategyPerformanceMetrics.calculate_metrics(trades)):
            assert got["n_records"] == want["total_trades"]
            for mine, theirs in (("total_profit", "total_profit"), ("total_loss", "total_loss"), ("net_profit", "net_profit"),
                                 ("max_drawdown", "max_drawdown"), ("win_rate", "win_rate"),
                                 ("largest_profit", "largest_profit"), ("largest_loss", "largest_loss")):
                assert got[mine] == pytest.approx(want[theirs], rel=1e-12, abs=1e-12), mine
            assert got["sharpe_ratio"] == pytest.approx(want["sharpe_ratio"], rel=1e-9, abs=1e-12)
            assert got["n_records"] < 2 or got["profit_factor"] == pytest.approx(want["profit_factor"], rel=1e-12)
            pairs = int(got["n_records"]) // 2
            assert got["sum_duration_bars"] * bar_minutes == pytest.approx(want["avg_trade_duration"] * pairs, rel=1e-12)
        adv = simulate_ref.calculate_advanced_metrics(simulate_ref.calculate_metrics(trades))
        if got["n_records"] >= 2:
            assert got["sortino_ratio"] == pytest.approx(adv["sortino_ratio"], rel=1e-9)
            assert got["mean_daily_pnl"] == pytest.approx(adv["profit_per_day"], rel=1e-9, abs=1e-12)
        assert got["score"] == pytest.approx(simulate_ref.strategy_score(simulate_ref.calculate_metrics(trades), goals),
                                             rel=1e-9, abs=1e-12, nan_ok=True)
    assert crossing > 0, "no merged pair (2k, 2k + 1) mixes symbols"


def test_single_symbol_book_is_the_oracle_lane():
    import book_ref
    from oracle import sim_oracle
    close, bank, pop, minute0 = _case(4000, 7)
    cfg = sim_oracle.config_of(minute0, 7)
    want, evs, pns = sim_oracle.population(close[1:2], bank[1:2], {p: i for i, p in enumerate(PERIODS)}, pop, cfg,
                                           event_cap=4002)
    got = [book_ref.book(ev, pn, cfg) for ev, pn in zip(evs, pns)]
    sim_oracle.assert_lanes(got, want[:, 0], "one-symbol books", rtol=1e-12, atol=1e-12)


def _book_args(S=10, N=200_000, pop=64, cap=4096, minute0=0, bar_minutes=1, price=DEV):
    """b200bt_book_metrics arguments with non-null dummy device pointers (never dereferenced: every call below is
    rejected before the device is touched)."""
    from ai_crypto_trader_b200 import _lib
    cfg = _lib.SweepConfig(initial_capital=10000.0, minute0=minute0, bar_minutes=bar_minutes, primary=0, secondary_mask=7,
                           variant=0, gap_bar=0, gap_minutes=0)
    return (price, N, S, N, DEV, pop, C.byref(cfg), DEV, DEV, cap, DEV, None, None)


@pytest.mark.parametrize("case, kw, status", [
    ("null price", dict(price=None), EINVAL),
    ("no individuals", dict(pop=0), EINVAL),
    ("negative event cap", dict(cap=-1), EINVAL),
    ("65 symbols", dict(S=65), ELIMIT),
    ("N = 2^30", dict(N=1 << 30), ELIMIT),
    ("S * (N + 1) records beyond 2^32", dict(S=64, N=(1 << 26)), ELIMIT),
    ("zero bar_minutes", dict(bar_minutes=0), EINVAL),
    ("clock beyond 2^32 minutes", dict(minute0=1 << 32), ELIMIT),
])
def test_book_metrics_rejects_bad_arguments(native_lib, case, kw, status):
    from ai_crypto_trader_b200 import _lib
    with pytest.raises(_lib.B200btError) as ei:
        _lib.call("b200bt_book_metrics", *_book_args(**kw))
    assert ei.value.status == status, (case, str(ei.value))


def test_book_metrics_needs_a_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    from ai_crypto_trader_b200 import _lib
    with pytest.raises(_lib.B200btError) as ei:
        _lib.call("b200bt_book_metrics", *_book_args(S=64))
    assert ei.value.status == ENODEVICE
