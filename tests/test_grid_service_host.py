"""The coupled restatement (tests/grid_service_ref.py) against the reference's own multi-symbol run()
(tests/golden/grid_service_reference.json, written by make_grid_service.py) and against the per-lane restatement where
the coupling cannot act."""
import json
import math
from pathlib import Path

import numpy as np
import pytest

import grid_ref
import grid_service_ref

GOLDEN = Path(__file__).resolve().parent / "golden" / "grid_service_reference.json"
REGIMES = {"ranging": 2, "volatile": 3}


def _walks(seed, S, T, lattice=False):
    rng = np.random.default_rng(seed)
    if lattice:
        return [list(1024 + np.cumsum(rng.integers(-2, 3, T)) * 16.0) for _ in range(S)]
    return [list(np.round(100 * np.exp(np.cumsum(0.002 * rng.standard_normal(T))) * 16) / 16) for _ in range(S)]


@pytest.mark.parametrize("kind", [0, 1])
def test_one_symbol_is_the_lane_restatement(kind):
    p = _walks(1, 1, 3000)
    labels = list(np.repeat(np.random.default_rng(2).integers(0, 5, 100), 30)[:3000])
    table = {2: (15, 3.0, 3.0), 3: (12, 6.0, 6.0)}
    kw = dict(n=9, kind=kind, lower_pct=1.0, upper_pct=1.5, rebalance_ticks=37, adjust_ticks=101, adapt=True,
              labels=labels, table=table)
    svc = grid_service_ref.simulate_service(p, [(p[0][0] * 0.99, p[0][0] * 1.01)], qty=[0.5], **kw)
    lane = grid_ref.simulate(p[0], p[0][0] * 0.99, p[0][0] * 1.01, qty=0.5, **kw)
    for f in grid_ref.FIELDS:
        if f != "num_grids":                   # the lane's grid here, the service's value in grid_ref
            assert svc["lanes"][0][f] == lane[f], f
    assert svc["lanes"][0]["regenerations"] == lane["regenerations"]
    assert svc["service"]["num_grids"] == lane["num_grids"]


def test_long_adjust_period_is_independent_lanes():
    S, T = 4, 2500
    p = _walks(3, S, T, lattice=True)
    bounds = [(x[0] * 0.98, x[0] * 1.02) for x in p]
    svc = grid_service_ref.simulate_service(p, bounds, 7, 0, [0.1, 0.2, 0.3, 0.4], 1.0, 1.0, 50, T)
    for s in range(S):
        lane = grid_ref.simulate(p[s], *bounds[s], 7, 0, [0.1, 0.2, 0.3, 0.4][s], 1.0, 1.0, 50, T)
        for f in grid_ref.FIELDS:
            assert svc["lanes"][s][f] == lane[f], (s, f)


def test_coupled_win_rate_steps_add_up():
    """Without a regime source each symbol's +-2 step moves the shared num_grids: with S rising symbols one adjust tick
    moves it by 2 S (up to the clamp at 20)."""
    T = 400
    p = [[100.0 + 0.25 * k for k in range(T)] for _ in range(3)]
    svc = grid_service_ref.simulate_service(p, [(99.0, 101.0)] * 3, 6, 0, [1.0] * 3, 1.0, 1.0, 5, 60)
    traj = [a[1] for a in svc["adjustments"]]
    assert traj[0] == 12 and traj[1] == 18 and max(traj) == 20
    assert svc["service"]["max_num_grids"] == 20 and svc["service"]["n_num_grids_changes"] == 3


def _fixture():
    return json.loads(GOLDEN.read_text())


def _case_inputs(fx, case):
    from ai_crypto_trader_b200 import grid
    closes, labels = grid_service_ref.fixture_series(fx, case)
    block = grid.grid_block(case["config"])
    defaults = {k: block.get(k, v) for k, v in grid.DEFAULTS.items()}
    d = grid.decode_individual({}, defaults, case["bar_minutes"])
    bounds = []
    for s, row in enumerate(closes):
        hist = grid.daily_closes(np.asarray(row, dtype=np.float32), case["minute0"], case["bar_minutes"],
                                 case["start_bar"], d["lookback"]) if d["auto"] else None
        bounds.append(grid.initial_bounds(row[case["start_bar"]], d["lower_pct"], d["upper_pct"], hist))
    table = {r: (t.num_grids, t.lower_pct, t.upper_pct) for r, t in enumerate(grid.regime_table(block)) if t.apply}
    qty = [grid.symbol_quantity(block, sym) for sym in case["symbols"]]
    st = case["start_bar"]
    got = grid_service_ref.simulate_service(
        [row[st:] for row in closes], bounds, d["num_grids"], d["grid_type"], qty, d["lower_pct"], d["upper_pct"],
        d["rebalance_ticks"], d["adjust_ticks"], bool(d["flags"] & 1), labels[st:] if labels else None, table,
        60 * case["bar_minutes"])
    got["initial"] = (d["num_grids"], d["lower_pct"], d["upper_pct"])
    got["labels"] = labels[st:] if labels else None
    return got


def _service_at_writes(got, case):
    """The service's (num_grids, lower_pct, upper_pct) at the grid_config writes, listed where they change."""
    writes = sorted({t for regs in case["regenerations"].values() for t, _ in regs})
    out, vals, j, adj = [], got["initial"], 0, got["adjustments"]
    for t in writes:
        while j < len(adj) and adj[j][0] < t:              # the adjustment follows the rebalances of its tick
            vals = adj[j][1:]
            j += 1
        if not out or out[-1][1:] != list(vals):
            out.append([t] + list(vals))
    return out


def test_restatement_matches_the_reference_run():
    fx = _fixture()
    for case in fx["cases"]:
        got = _case_inputs(fx, case)
        name = case["name"]
        for s, sym in enumerate(case["symbols"]):
            lane, gp = got["lanes"][s], case["grid_profits"][sym]
            assert lane["total_trades"] == gp["total_trades"], (name, sym)
            assert lane["profitable_trades"] == gp["profitable_trades"], (name, sym)
            assert math.isclose(lane["total_profit"], gp["total_profit"], rel_tol=1e-12, abs_tol=1e-12), (name, sym)
            assert [[k, n] for k, _, _, n in lane["regenerations"]] == case["regenerations"][sym], (name, sym)
            assert [lane["lower"], lane["upper"]] == case["final_grid"][sym], (name, sym)
        assert _service_at_writes(got, case) == case["service"], name                # the num_grids trajectory
        f = case["final"]
        sv = got["service"]
        assert (sv["num_grids"], sv["lower_pct"], sv["upper_pct"]) == \
            (f["num_grids"], f["lower_boundary_pct"], f["upper_boundary_pct"]), name
        perf = case["performance"]
        assert (sv["total_trades"], sv["profitable_trades"]) == (perf["total_trades"], perf["profitable_trades"]), name
        assert math.isclose(sv["total_profit"], perf["total_profit"], rel_tol=1e-12, abs_tol=1e-12), name
        assert math.isclose(sv["win_rate"], perf["win_rate"], rel_tol=1e-15), name


def test_fixture_covers_every_branch():
    fx = _fixture()
    cases = fx["cases"]
    assert {len(c["symbols"]) for c in cases} >= {2, 3, 5}
    assert any(c["symbols"] == ["BTCUSDC", "ETHUSDC", "BNBUSDC"] and c["name"].startswith("config.json") for c in cases)
    assert {c["bar_minutes"] for c in cases} >= {1, 5, 60}
    assert any(c["config"].get("grid_type") == "geometric" for c in cases)
    assert any(c["config"].get("auto_boundaries", True) for c in cases)
    assert any(c["config"].get("auto_adjust_period", 86400) < c["config"].get("rebalance_frequency", 3600)
               for c in cases)
    assert any(min(c["grid_profits"][s]["total_trades"] for s in c["symbols"]) <= 10 for c in cases)
    clamp20 = clamp5 = regime_last = False
    for c in cases:
        got = _case_inputs(fx, c)
        sv = got["service"]
        if c["labels"] is None:
            clamp20 |= sv["max_num_grids"] == 20
            clamp5 |= sv["min_num_grids"] == 5
        elif c["config"].get("adapt_to_market_regime", True):
            # an adjust tick whose label fires the rule (ranging 15, volatile 12) ends on the last symbol's step
            rule = {2: 15, 3: 12}
            regime_last |= any(got["labels"][k] in rule and n != rule[got["labels"][k]]
                               for k, n, _, _ in got["adjustments"])
    assert clamp20 and clamp5 and regime_last
