"""CPU checks of the grid-trading backtest's host side: the restatement (tests/grid_ref.py) against the fixture the
reference's own run() wrote (tests/golden/grid_reference.json), the tick-period conversion, the initial boundaries, gene
decoding and the refusal of volatility_based grids."""
import json
import math
from pathlib import Path

import numpy as np
import pytest

import grid_ref

GOLDEN = Path(__file__).resolve().parent / "golden" / "grid_reference.json"


@pytest.fixture(scope="module")
def fixture():
    return json.loads(GOLDEN.read_text())


def labels_of(fx, case):
    """A case's per-bar regime labels (the fixture stores them as runs [label, length]), or None."""
    if not case["labels"]:
        return None
    return [v for v, n in fx["label_runs"][case["labels"]] for _ in range(n)]


def lane_inputs(fx, case):
    """grid_ref.simulate keyword arguments of a fixture case, with the host's decoding (grid.py)."""
    from ai_crypto_trader_b200 import grid
    closes = fx["series"][case["closes"]]
    labels = labels_of(fx, case)
    bm, start = case["bar_minutes"], case["start_bar"]
    block = dict(case["config"])
    d = grid.decode_individual({}, block, bm)
    hist = grid.daily_closes(np.asarray(closes, dtype=np.float32), case["minute0"], bm, start, d["lookback"]) \
        if d["auto"] else None
    lower, upper = grid.initial_bounds(closes[start], d["lower_pct"], d["upper_pct"], hist)
    table = {r: (t.num_grids, t.lower_pct, t.upper_pct) for r, t in enumerate(grid.regime_table(block)) if t.apply}
    days = [(case["minute0"] + (start + k) * bm) // 1440 for k in range(len(closes) - start)]
    return dict(prices=closes[start:], lower=lower, upper=upper, n=d["num_grids"], kind=d["grid_type"],
                qty=grid.symbol_quantity(block, case["symbol"]), lower_pct=d["lower_pct"], upper_pct=d["upper_pct"],
                rebalance_ticks=d["rebalance_ticks"], adjust_ticks=d["adjust_ticks"],
                adapt=bool(d["flags"] & 1), labels=labels[start:] if labels else None, table=table,
                bar_seconds=60 * bm), days


def test_restatement_equals_the_reference_run(fixture):
    assert len(fixture["cases"]) >= 8
    kinds = set()
    for case in fixture["cases"]:
        kw, days = lane_inputs(fixture, case)
        got = grid_ref.simulate(**kw, days=days)
        kinds.add(kw["kind"])
        gp, perf, fin = case["grid_profits"], case["performance"], case["final"]
        name = case["name"]
        assert got["total_trades"] == gp["total_trades"] == perf["total_trades"], name
        assert got["profitable_trades"] == gp["profitable_trades"], name
        assert math.isclose(got["total_profit"], gp["total_profit"], rel_tol=1e-12, abs_tol=1e-12), name
        assert math.isclose(got["profit_per_day"], perf["profit_per_day"], rel_tol=1e-12, abs_tol=1e-12), name
        assert got["win_rate"] == perf["win_rate"], name
        regs = [(r["tick"], r["lower"], r["upper"], r["n"]) for r in case["regenerations"]]
        assert got["regenerations"] == regs, name
        assert got["levels"] == case["regenerations"][-1]["levels"], name
        assert (got["num_grids"], got["lower"], got["upper"]) == (fin["num_grids"], fin["lower"], fin["upper"]), name
        snaps = [(s["day"], s["tick"], s["total_trades"], s["profitable_trades"]) for s in case["snapshots"]]
        assert [s[:4] for s in got["snapshots"]] == snaps, name
        for s, want in zip(got["snapshots"], case["snapshots"]):
            assert math.isclose(s[4], want["total_profit"], rel_tol=1e-12, abs_tol=1e-12), name
        assert got["near_ties"] == 0 or kw["kind"] == 1
    assert kinds == {0, 1}


def test_fixture_covers_the_rule(fixture):
    cases = {c["name"]: c for c in fixture["cases"]}
    moved = [c["final"]["num_grids"] - c["config"]["num_grids"] for c in fixture["cases"] if not c["labels"]]
    assert max(moved) > 0 and min(moved) < 0                               # both sides of the win-rate rule
    regime = [c for c in fixture["cases"] if c["labels"]]
    seen = set()
    for c in regime:
        lab = labels_of(fixture, c)
        seen |= set(lab[c["start_bar"]:])
    assert seen == {0, 1, 2, 3, 4}
    exact = cases["arithmetic exact levels"]
    assert exact["regenerations"][0]["levels"] == [768.0 + 64 * i for i in range(9)]
    closes = fixture["series"][exact["closes"]]
    assert len(set(closes) & set(exact["regenerations"][0]["levels"])) >= 5       # prices exactly on levels
    assert any(len(c["regenerations"]) > 50 for c in fixture["cases"])


NAN = math.nan
FLAT = dict(rebalance_ticks=10 ** 6, adjust_ticks=10 ** 6, lower_pct=5.0, upper_pct=5.0, qty=1.0)
# lanes the fixture does not hold: repeated levels (an arithmetic step under an ulp, a geometric ratio of 1.0) and NaN
# closes (on the first tick, mid-series, on a rebalance tick that would regenerate, and on the last tick)
EDGE_LANES = {
    "repeated arithmetic levels": dict(FLAT, prices=[99, 101, 99, 101], lower=100.0, upper=100 * (1 + 6e-16), n=8, kind=0),
    "geometric ratio 1.0": dict(FLAT, prices=[99, 101, 100, 99, 100, 101], lower=100.0, upper=100.0, n=5, kind=1),
    "NaN mid-series": dict(FLAT, prices=[100.5, NAN, 100.5, 99], lower=95.0, upper=105.0, n=10, kind=0),
    "NaN runs": dict(FLAT, prices=[NAN, 101, 97, NAN, NAN, 103, 96, 104, NAN], lower=95.0, upper=105.0, n=10, kind=0),
    "NaN on a rebalance tick": dict(FLAT, prices=[100, 104, NAN, 90, 100, 110, 90], lower=95.0, upper=105.0, n=4, kind=0,
                                    rebalance_ticks=2),
}


def test_fast_restatement_matches(fixture):
    cases = [(c["name"], lane_inputs(fixture, c)[0]) for c in fixture["cases"]] + list(EDGE_LANES.items())
    for name, kw in cases:
        a, b = grid_ref.simulate(**kw), grid_ref.simulate_fast(**kw)
        for f in grid_ref.FIELDS:
            if f == "near_ties":
                continue
            assert math.isclose(a[f], b[f], rel_tol=1e-9, abs_tol=1e-9) or (math.isnan(a[f]) and math.isnan(b[f])), \
                (name, f, a[f], b[f])
        # profits are sums of non-negative steps: no absolute floor, which would hide a step of 1e-14
        assert a["profitable_trades"] == b["profitable_trades"], name
        assert math.isclose(a["total_profit"], b["total_profit"], rel_tol=1e-9, abs_tol=0.0), name


def test_edge_lanes_follow_the_reference_rule():
    """levels.index prices every copy of a repeated level by the step under its first copy; a NaN close is no move."""
    rep = grid_ref.simulate(**EDGE_LANES["repeated arithmetic levels"])
    lv = grid_ref.levels(100.0, 100 * (1 + 6e-16), 8, 0)
    assert len(set(lv)) < len(lv)
    assert (rep["up_crossings"], rep["profitable_trades"]) == (18, 16)
    assert rep["total_profit"] == 2 * sum(x - lv[lv.index(x) - 1] for x in lv if lv.index(x) > 0)
    geo = grid_ref.simulate(**EDGE_LANES["geometric ratio 1.0"])
    assert (geo["up_crossings"], geo["profitable_trades"], geo["total_profit"]) == (18, 0, 0.0)
    nan = grid_ref.simulate(**EDGE_LANES["NaN mid-series"])
    assert (nan["down_crossings"], nan["up_crossings"], nan["near_ties"]) == (2, 0, 0)
    reb = grid_ref.simulate(**EDGE_LANES["NaN on a rebalance tick"])
    assert reb["regenerations"][1][0] == 4 and reb["n_rebalance_checks"] == 3
    last = EDGE_LANES["NaN runs"]
    assert math.isnan(grid_ref.simulate(**last)["mark_to_market"])
    assert math.isnan(grid_ref.simulate_fast(**last)["mark_to_market"])


def test_period_ticks():
    from ai_crypto_trader_b200.grid import period_ticks
    assert period_ticks(3600, 1) == 61
    assert period_ticks(86400, 1) == 1441
    assert period_ticks(3600, 5) == 13
    assert period_ticks(3599, 5) == 12
    assert period_ticks(1800.5, 1) == 31
    assert period_ticks(0, 1) == 1
    assert period_ticks(59.999, 1) == 1
    assert period_ticks(60, 1) == 2
    assert period_ticks(1e18, 1) == 2 ** 31 - 1
    for sec in (0, 1, 59, 60, 61, 119.5, 3600, 7200.25):
        for bm in (1, 5, 15):
            k = period_ticks(sec, bm)
            assert k * 60 * bm > sec and (k == 1 or (k - 1) * 60 * bm <= sec)
    with pytest.raises(ValueError):
        period_ticks(-1, 1)


def test_initial_bounds_against_numpy():
    from ai_crypto_trader_b200 import grid
    rng = np.random.default_rng(3)
    close = (100 * np.exp(np.cumsum(0.01 * rng.standard_normal(20 * 288)))).astype(np.float32)
    m0 = 28_401_120
    start = 15 * 288 + 17
    hist = grid.daily_closes(close, m0, 5, start, 14)
    t0 = m0 + start * 5
    want = []
    for d in range(t0 // 1440 - 14, t0 // 1440 + 1):
        if d * 1440 < t0 - 14 * 1440:
            continue
        bars = [b for b in range(start + 1) if d * 1440 <= m0 + 5 * b <= min(t0, d * 1440 + 1439)]
        want.append(float(close[bars[-1]]))
    assert hist == want and len(hist) == 14          # t0 is not midnight: 13 whole days and the current one
    p0 = float(close[start])
    lo, up = grid.initial_bounds(p0, 5.0, 5.0, hist)
    vol = np.std(hist) / np.mean(hist) * 100
    assert (lo, up) == (p0 * (1 - vol / 100), p0 * (1 + vol / 100))
    assert grid.initial_bounds(1024.0, 25, 25) == (768.0, 1280.0)
    with pytest.raises(ValueError):
        grid.daily_closes(close, m0, 5, 10, 14)                  # no room for the lookback


def test_gene_decoding_and_refusals():
    from ai_crypto_trader_b200 import grid
    ranges = grid.grid_param_ranges()
    assert set(ranges) == {"num_grids", "grid_type", "lower_boundary_pct", "upper_boundary_pct", "auto_boundaries",
                           "volatility_lookback", "rebalance_frequency", "auto_adjust_period", "adapt_to_market_regime"}
    assert ranges["grid_type"] == (0, 1)
    d = grid.decode_individual({"num_grids": 12, "grid_type": 1, "auto_boundaries": 0, "adapt_to_market_regime": 1,
                                "rebalance_frequency": 3600, "auto_adjust_period": 86400}, {}, 1)
    assert (d["num_grids"], d["grid_type"], d["rebalance_ticks"], d["adjust_ticks"], d["flags"], d["auto"]) == \
        (12, 1, 61, 1441, 1, False)
    d = grid.decode_individual({}, {}, 1)                        # the reference's defaults
    assert (d["num_grids"], d["grid_type"], d["flags"], d["lookback"], d["lower_pct"]) == (10, 0, 3, 14, 5.0)
    assert grid.decode_individual({"grid_type": "geometric"}, {}, 1)["grid_type"] == 1
    for bad in ({"grid_type": "volatility_based"}, {"grid_type": 2}, {"grid_type": "custom"}, {"num_grids": 0},
                {"num_grids": 128}, {"lower_boundary_pct": 100.0}, {"upper_boundary_pct": 0.0}):
        with pytest.raises(ValueError):
            grid.decode_individual(bad, {}, 1)
    with pytest.raises(ValueError, match="volatility_based"):
        grid.decode_individual({"grid_type": "volatility_based"}, {}, 1)


def test_config_tables():
    from ai_crypto_trader_b200 import grid
    block = {"ranging_num_grids": 14, "volatile_lower_boundary_pct": 7.5, "quantity_per_grid": 0.02,
             "symbol_settings": [{"symbol": "BTCUSDC", "quantity_per_grid": 0.001, "lower_boundary_pct": 4.0}]}
    t = grid.regime_table(block)
    assert [r.apply for r in t] == [0, 0, 1, 1, 0]
    assert (t[2].num_grids, t[2].lower_pct, t[3].num_grids, t[3].lower_pct, t[3].upper_pct) == (14, 3.0, 12, 7.5, 6.0)
    assert grid.symbol_quantity(block, "BTCUSDC") == 0.001
    assert grid.symbol_quantity(block, "ETHUSDC") == 0.02
    assert grid.grid_block({"grid_trading": block}) is block
