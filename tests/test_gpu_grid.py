"""b200bt_grid_sweep on the H100 against the restatement (tests/grid_ref.py, itself pinned to the reference's run()):
the fixture's cases, random populations on several clocks with exact level hits, flat stretches and gaps, determinism,
the objective matrix, per-day profit rows, the GA loops over GridSweep and a configs[1]-sized run."""
import json
import math
import random
from pathlib import Path

import numpy as np
import pytest

import grid_ref

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "grid_reference.json"
M0 = 28_401_120
EXACT = ("total_trades", "profitable_trades", "up_crossings", "down_crossings", "n_regenerations", "num_grids", "lower",
         "upper", "position", "max_position", "min_position", "n_rebalance_checks", "n_adjustments", "n_ticks")


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def market_of(torch, closes, bar_minutes=1, minute0=M0):
    from ai_crypto_trader_b200.sweep import MarketData
    c = np.asarray(closes, dtype=np.float32)
    c = c[None] if c.ndim == 1 else c
    ohlcv = np.zeros((5,) + c.shape, dtype=np.float32)
    ohlcv[3] = c
    return MarketData(ohlcv, minute0=minute0, bar_minutes=bar_minutes)


def ref_lane(sweep, params, s, fast=True):
    """grid_ref on lane (params, symbol s) of a GridSweep, with the host's decoding."""
    from ai_crypto_trader_b200 import grid
    m = sweep.market
    d = grid.decode_individual(params, sweep.defaults, m.bar_minutes)
    _, bounds = sweep.decode([params])
    close = sweep.market.close[s].cpu().numpy().astype(np.float64)
    labels = None
    if sweep.labels is not None:
        labels = sweep.labels[0 if sweep.ld_labels == 0 else s].cpu().numpy()[sweep.start_bar:]
    table = {r: (t.num_grids, t.lower_pct, t.upper_pct) for r, t in enumerate(sweep.table) if t.apply}
    kw = dict(prices=close[sweep.start_bar:], lower=float(bounds[0, s, 0]), upper=float(bounds[0, s, 1]),
              n=d["num_grids"], kind=d["grid_type"], qty=float(sweep.quantity[s]), lower_pct=d["lower_pct"],
              upper_pct=d["upper_pct"], rebalance_ticks=d["rebalance_ticks"], adjust_ticks=d["adjust_ticks"],
              adapt=bool(d["flags"] & 1), labels=labels, table=table, bar_seconds=60 * m.bar_minutes)
    if fast:
        return grid_ref.simulate_fast(**kw)
    days = [(m.minute0 + (sweep.start_bar + k) * m.bar_minutes) // 1440 for k in range(m.N - sweep.start_bar)]
    return grid_ref.simulate(**kw, days=days)


def check_lanes(sweep, population, stats, lanes=None, profit_tol=1e-9):
    """Exact counts / regenerations / final grid on every lane without near ties; on lanes with near ties the counts
    may move by at most the levels those ticks could cross.  Returns the number of lanes with near ties."""
    tied = 0
    S = sweep.market.S
    for i, s in (lanes or [(i, s) for i in range(len(population)) for s in range(S)]):
        want = ref_lane(sweep, population[i], s)
        got = {f: float(stats[f][i, s]) for f in stats}
        if got["near_ties"] > 0:
            tied += 1
            assert abs(got["total_trades"] - want["total_trades"]) <= 2 * got["near_ties"] * 128, (i, s)
            continue
        for f in EXACT:
            assert got[f] == want[f], (i, s, f, got[f], want[f])
        for f in ("total_profit", "cash", "profit_per_day", "mark_to_market", "win_rate"):
            assert math.isclose(got[f], want[f], rel_tol=profit_tol, abs_tol=profit_tol * max(1.0, abs(want["cash"]))), \
                (i, s, f, got[f], want[f])
    return tied


def random_population(n, seed, ranges=None):
    from ai_crypto_trader_b200.grid import grid_param_ranges
    rng = random.Random(seed)
    ranges = ranges or grid_param_ranges()
    return [{k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi)) for k, (lo, hi) in ranges.items()}
            for _ in range(n)]


def test_fixture_cases_on_the_gpu(torch):
    from ai_crypto_trader_b200.grid import GridSweep
    fx = json.loads(GOLDEN.read_text())
    for case in fx["cases"]:
        closes = fx["series"][case["closes"]]
        m = market_of(torch, closes, case["bar_minutes"], case["minute0"])
        labels = None
        if case["labels"]:
            runs = fx["label_runs"][case["labels"]]
            labels = torch.tensor([v for v, n in runs for _ in range(n)], dtype=torch.uint8, device="cuda")[None]
        cfg = dict(case["config"], symbol_settings=[])
        sweep = GridSweep(m, start_bar=case["start_bar"], regime=labels, config=cfg)
        st = sweep.grid_stats([{}])
        got = {f: float(v[0, 0]) for f, v in st.items()}
        name = case["name"]
        if got["near_ties"] > 0:              # prices on geometric levels: only the near-tie bound holds
            assert "geometric" in case["config"]["grid_type"], name
            check_lanes(sweep, [{}], st)
            continue
        assert got["total_trades"] == case["grid_profits"]["total_trades"], name
        assert got["profitable_trades"] == case["grid_profits"]["profitable_trades"], name
        assert got["n_regenerations"] == len(case["regenerations"]) - 1, name
        assert (got["num_grids"], got["lower"], got["upper"]) == \
            (case["final"]["num_grids"], case["final"]["lower"], case["final"]["upper"]), name
        assert math.isclose(got["total_profit"], case["grid_profits"]["total_profit"], rel_tol=1e-12, abs_tol=1e-12), name
        assert math.isclose(got["profit_per_day"], case["performance"]["profit_per_day"], rel_tol=1e-12, abs_tol=1e-12)
        assert got["win_rate"] == case["performance"]["win_rate"], name
        check_lanes(sweep, [{}], st, profit_tol=1e-12)


@pytest.mark.parametrize("bar_minutes", [1, 5])
def test_random_population_against_the_restatement(torch, bar_minutes):
    from ai_crypto_trader_b200.grid import GridSweep
    rng = np.random.default_rng(11 + bar_minutes)
    S, N = 3, 40 * 1440 // bar_minutes
    close = np.empty((S, N), dtype=np.float32)
    close[0] = 30000 * np.exp(np.cumsum(0.0015 * rng.standard_normal(N)))
    close[1] = 2000 * np.exp(np.cumsum(0.004 * rng.standard_normal(N)))
    # exact level hits, flat stretches and gaps of many levels: a walk on a 1/64 lattice around 1024 with long pauses
    steps = np.where(rng.random(N) < 0.4, 0, np.where(rng.random(N) < 0.01, rng.integers(-40, 41, N),
                                                      rng.integers(-2, 3, N))) * (1024 / 64)
    close[2] = 1024 + np.clip(np.cumsum(steps) / 8, -400, 800)
    close[2, N // 2: N // 2 + 2000] = close[2, N // 2]
    m = market_of(torch, close, bar_minutes)
    labels = torch.tensor(np.repeat(rng.integers(0, 5, N // 60 + 1), 60)[:N], dtype=torch.uint8, device="cuda")[None]
    sweep = GridSweep(m, quantity=[0.01, 0.1, 0.5], regime=labels, start_bar=31 * 1440 // bar_minutes + 7)
    pop = random_population(48, 5) + [{"num_grids": 8, "grid_type": 0, "auto_boundaries": 0, "lower_boundary_pct": 25.0,
                                       "upper_boundary_pct": 25.0, "adapt_to_market_regime": 0}]
    st = sweep.grid_stats(pop)
    tied = check_lanes(sweep, pop, st)
    geo = sum(1 for p in pop if p.get("grid_type", 0) == 1) * S
    assert tied <= max(2, geo // 4)
    assert np.all(st["near_ties"][[i for i, p in enumerate(pop) if p.get("grid_type", 0) == 0]] == 0)
    assert np.all(st["n_ticks"] == N - sweep.start_bar)


def test_deterministic_and_duplicates(torch):
    from ai_crypto_trader_b200.grid import GridSweep
    from ai_crypto_trader_b200 import synth
    m = market_of(torch, synth.synth_ohlcv(2, 60 * 1440)[3])
    sweep = GridSweep(m, quantity=0.01)
    pop = random_population(40, 9)
    sweep.grid_stats(pop)
    a = sweep.stats_device().clone()
    sweep.grid_stats(pop)
    b = sweep.stats_device().clone()
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    dup = pop[:5] + pop[:5] + pop[5:10]
    st = sweep.grid_stats(dup)
    assert sweep._inverse is not None
    assert np.array_equal(st["total_trades"][:5], st["total_trades"][5:10])
    assert np.array_equal(st["total_profit"][10:], a[5:10, :, 0].cpu().numpy())


def test_objective_matrix_and_fitness(torch):
    from ai_crypto_trader_b200.grid import GridSweep, OBJECTIVE_FIELDS
    from ai_crypto_trader_b200 import synth
    m = market_of(torch, synth.synth_ohlcv(3, 50 * 1440)[3])
    sweep = GridSweep(m, quantity=0.01)
    pop = random_population(33, 4)
    objs = [(f, True) for f in ("total_profit", "mark_to_market", "win_rate", "n_regenerations", "min_position")]
    got = sweep.evaluate_objectives(pop, objs)
    st = sweep.grid_stats()
    for j, (f, _) in enumerate(objs):
        want = np.array([sum(st[f][i, s] for s in range(m.S)) / m.S for i in range(len(pop))])
        assert np.array_equal(got[:, j], want), f
    fit = sweep.evaluate(pop)
    assert np.array_equal(fit, got[:, 0])
    assert sweep.fitness_function.batch(pop) == [float(x) for x in fit]
    with pytest.raises(ValueError):
        sweep.evaluate_objectives(pop, [("near_ties", True)])
    assert "near_ties" not in OBJECTIVE_FIELDS


def test_day_profit_rows(torch):
    from ai_crypto_trader_b200.grid import GridSweep
    rng = np.random.default_rng(5)
    S, N = 2, 45 * 288
    close = (1000 * np.exp(np.cumsum(0.003 * rng.standard_normal((S, N)), axis=1))).astype(np.float32)
    m = market_of(torch, close, 5, M0 + 777)
    sweep = GridSweep(m, quantity=[0.1, 0.2], start_bar=31 * 288)
    pop = random_population(20, 2) + random_population(3, 2)
    rows, first_day = sweep.day_profit(pop)
    st = sweep.grid_stats()
    rows = rows.cpu().numpy()
    assert rows.shape == (len(pop), (M0 + 777 + (N - 1) * 5) // 1440 - (M0 + 777) // 1440 + 1)
    assert first_day == (M0 + 777) // 1440
    tot = st["total_profit"].sum(axis=1)
    assert np.allclose(rows.sum(axis=1), tot, rtol=1e-12, atol=1e-9)
    stats_only = GridSweep(m, quantity=[0.1, 0.2], start_bar=31 * 288).grid_stats(pop)
    for f in st:
        assert np.array_equal(st[f], stats_only[f]), f                          # the day path changes no stat
    for i in (0, 7, 21):
        want = np.zeros(rows.shape[1])
        for s in range(S):
            for d, v in ref_lane(sweep, pop[i], s, fast=False)["day_profit"].items():
                want[d - first_day] += v
        assert np.allclose(rows[i], want, rtol=1e-12, atol=1e-9), i
    assert np.all(rows[:, : (31 * 288 * 5 + 777) // 1440 - 1] == 0.0)           # before the start bar


def test_genetic_algorithms_over_grid_sweep(torch):
    from ai_crypto_trader_b200.genetic_algorithm import (DeviceGeneticAlgorithm, GeneticAlgorithm,
                                                         ParetoGeneticAlgorithm)
    from ai_crypto_trader_b200.grid import GridSweep, grid_param_ranges
    from ai_crypto_trader_b200 import synth
    m = market_of(torch, synth.synth_ohlcv(2, 45 * 1440)[3])
    sweep = GridSweep(m, quantity=0.01)
    seed = {"num_grids": 10, "grid_type": 0, "lower_boundary_pct": 5.0, "upper_boundary_pct": 5.0, "auto_boundaries": 1,
            "volatility_lookback": 14, "rebalance_frequency": 3600, "auto_adjust_period": 86400,
            "adapt_to_market_regime": 1}
    seed_fit = sweep.evaluate([seed])[0]
    ga = GeneticAlgorithm(grid_param_ranges(), sweep.fitness_function, population_size=24, generations=3, random_seed=1)
    ga.run([seed])
    assert ga.best_fitness > seed_fit
    dga = DeviceGeneticAlgorithm(grid_param_ranges(), sweep.fitness_function, population_size=24, generations=3,
                                 random_seed=2)
    dga.run([seed])
    assert dga.best_fitness > seed_fit
    objs = [("total_profit", True), ("mark_to_market", True)]
    pga = ParetoGeneticAlgorithm(grid_param_ranges(), lambda p: sweep.evaluate_objectives_device(p, objs), objs,
                                 population_size=24, generations=3, random_seed=3)
    front = pga.run([seed])
    assert front and max(f["objectives"]["total_profit"] for f in front) > seed_fit


def test_configs1_sized_run(torch):
    """BASELINE configs[1]'s shape: 1024 individuals x 10 symbols x 1M 1-minute bars; 64 lanes against the restatement."""
    from ai_crypto_trader_b200.grid import GridSweep
    from ai_crypto_trader_b200 import synth
    m = market_of(torch, synth.synth_ohlcv(10, 1_000_000)[3])
    sweep = GridSweep(m, quantity=0.01)
    pop = random_population(1024, 77)
    st = sweep.grid_stats(pop)
    assert np.all(np.isfinite(st["total_profit"])) and np.all(st["n_ticks"] == m.N - sweep.start_bar)
    rng = np.random.default_rng(1)
    lanes = [(int(i), int(s)) for i, s in zip(rng.integers(0, 1024, 64), rng.integers(0, 10, 64))]
    tied = check_lanes(sweep, pop, st, lanes)
    assert tied <= 16
