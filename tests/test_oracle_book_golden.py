"""The book oracle (tests/book_ref.py) and the host StrategyPerformanceMetrics against the reference's own metrics of
multi-symbol trade lists (tests/golden/book_reference.*, written by tests/golden/make_book.py, which executes the
reference's _simulate_trades per symbol, concatenates in symbol order and runs calculate_metrics /
calculate_advanced_metrics / _calculate_strategy_score).  CPU only."""
import json
from pathlib import Path

import numpy as np
import pytest

GOLD = Path(__file__).parent / "golden"
ABS = 1e-12


def _load():
    meta = json.loads((GOLD / "book_reference.json").read_text())
    return meta, np.load(GOLD / "book_reference.npz")


def _f(x):
    return float(x)


def _lanes(meta, arrays, case, params, cfg):
    from oracle import sim_oracle
    close, rsi = arrays[f"close_{case['name']}"], arrays[f"rsi_{case['name']}"]
    row = meta["periods"].index(params.get("rsi_period", 14))
    evs, pns = [], []
    for s in range(close.shape[0]):
        _, ev, pn = sim_oracle.lane(close[s], rsi[s, row], params, cfg, event_cap=close.shape[1] + 2)
        evs.append(ev)
        pns.append(pn)
    return evs, pns


def _cases():
    meta, _ = _load()
    return [(c["name"], i) for c in meta["cases"] for i in range(len(c["books"]))]


@pytest.mark.parametrize("case_name, i", _cases())
def test_book_oracle_matches_the_reference_book(case_name, i):
    import book_ref
    from oracle import sim_oracle
    meta, arrays = _load()
    case = next(c for c in meta["cases"] if c["name"] == case_name)
    ref = case["books"][i]
    bm = case["bar_minutes"]
    cfg = sim_oracle.config_of(meta["minute0"], bm, goals=meta["goals"])
    evs, pns = _lanes(meta, arrays, case, ref["params"], cfg)
    # merged order and record pnl: bit for bit
    rec = book_ref.merged(evs, pns)
    np.testing.assert_array_equal([r[0] for r in rec], arrays[f"bar_{case_name}_{i}"])
    np.testing.assert_array_equal([r[1] for r in rec], arrays[f"sym_{case_name}_{i}"])
    np.testing.assert_array_equal(np.array([r[3] for r in rec], dtype=np.float64), arrays[f"pnl_{case_name}_{i}"])
    got = book_ref.book(evs, pns, cfg)
    m, adv = ref["metrics"], ref["advanced"]
    assert got["n_records"] == m["total_trades"] == ref["n_records"]
    for mine, theirs in (("total_profit", "total_profit"), ("total_loss", "total_loss"), ("net_profit", "net_profit"),
                         ("max_drawdown", "max_drawdown"), ("win_rate", "win_rate"), ("largest_profit", "largest_profit"),
                         ("largest_loss", "largest_loss"), ("profit_factor", "profit_factor")):
        assert got[mine] == pytest.approx(_f(m[theirs]), rel=1e-12, abs=ABS), mine
    assert got["sharpe_ratio"] == pytest.approx(_f(m["sharpe_ratio"]), rel=1e-9, abs=ABS)
    assert got["sum_duration_bars"] * bm == pytest.approx(_f(m["avg_trade_duration"]) * (int(got["n_records"]) // 2),
                                                          rel=1e-12, abs=ABS)
    assert got["n_days"] == len(ref["daily_returns"]) or got["n_records"] < 2
    assert got["sortino_ratio"] == pytest.approx(_f(adv["sortino_ratio"]), rel=1e-9, abs=ABS)
    assert got["mean_daily_pnl"] == pytest.approx(_f(adv["profit_per_day"]), rel=1e-9, abs=ABS)
    assert got["score"] == pytest.approx(_f(ref["score"]), rel=1e-9, abs=ABS, nan_ok=True)
    for g, want in zip(meta["alt_goals"], ref["alt_scores"]):
        c = sim_oracle.config_of(meta["minute0"], bm, goals=g["goals"], advanced=g["advanced"])
        assert book_ref.score(got, c) == pytest.approx(_f(want), rel=1e-9, abs=ABS, nan_ok=True), g
    # symbol dicts: per-symbol net pnl of the lanes
    net = {f"SYN{s:03d}USDT": float(np.sum(pn)) for s, pn in enumerate(pns) if len(pn)}
    assert sorted(k for k, v in net.items() if v > 0) == sorted(ref["profitable_symbols"])
    assert sorted(k for k, v in net.items() if v <= 0) == sorted(ref["unprofitable_symbols"])


@pytest.mark.parametrize("case_name, i", _cases())
def test_host_metrics_match_the_reference_book(case_name, i):
    from ai_crypto_trader_b200.strategy_evaluation import StrategyPerformanceMetrics
    from oracle import simulate_ref
    meta, arrays = _load()
    case = next(c for c in meta["cases"] if c["name"] == case_name)
    ref = case["books"][i]
    close, rsi = arrays[f"close_{case_name}"], arrays[f"rsi_{case_name}"]
    row = meta["periods"].index(ref["params"].get("rsi_period", 14))
    trades = []
    for s in range(close.shape[0]):
        trades += simulate_ref.simulate_trades(ref["params"], simulate_ref.market_points(
            close[s], rsi[s, row], f"SYN{s:03d}USDT", meta["minute0"], case["bar_minutes"]))
    m = StrategyPerformanceMetrics.calculate_metrics(trades)
    for k, v in ref["metrics"].items():
        assert _f(m[k]) == pytest.approx(_f(v), rel=1e-9 if k == "sharpe_ratio" else 1e-12, abs=ABS, nan_ok=True), k
    if case.get("one_record") is not None and i == len(case["books"]) - 1:
        one = StrategyPerformanceMetrics.calculate_metrics(trades[:1])
        for k, v in case["one_record"].items():
            assert _f(one[k]) == pytest.approx(_f(v), rel=1e-12, abs=ABS), k


def test_fixture_holds_the_planted_shapes():
    import book_ref  # noqa: F401
    meta, arrays = _load()
    names = {c["name"]: c for c in meta["cases"]}
    assert {c["bar_minutes"] for c in meta["cases"]} == {1, 1440}
    assert any(b["n_records"] == 0 for c in meta["cases"] for b in c["books"])
    crossing = ties = last = 0
    for c in meta["cases"]:
        for i, b in enumerate(c["books"]):
            bars, syms = arrays[f"bar_{c['name']}_{i}"], arrays[f"sym_{c['name']}_{i}"]
            crossing += int(np.sum(syms[0:len(syms) - 1:2] != syms[1::2]))
            ties += int(np.sum((bars[1:] == bars[:-1]) & (syms[1:] != syms[:-1])))
            last += int(np.sum((bars[1:] == c["n_bars"] - 1) & (bars[:-1] == c["n_bars"] - 1) & (syms[1:] == syms[:-1])))
            assert meta["quiet"] not in set(syms.tolist())
    assert crossing and ties and last, (crossing, ties, last)
    assert names["grid_1m"]["one_record"] is not None
