"""b200bt_grid_service_sweep on the H100 against the coupled restatement (tests/grid_service_ref.py): random populations
on 1 .. 40 symbols (17 and 40 run several symbols per warp) and several clocks, the bit-equality with b200bt_grid_sweep
where the coupling cannot act, determinism, NaN stats, day rows, the objective matrix and a GA loop."""
import json
import math
import random
from pathlib import Path

import numpy as np
import pytest

import grid_service_ref

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "grid_service_reference.json"
M0 = 28_401_120
EXACT = ("total_trades", "profitable_trades", "up_crossings", "down_crossings", "n_regenerations", "num_grids", "lower",
         "upper", "position", "max_position", "min_position", "n_rebalance_checks", "n_adjustments", "n_ticks")
SERVICE_EXACT = ("total_trades", "profitable_trades", "win_rate", "num_grids", "lower_pct", "upper_pct", "n_adjustments",
                 "n_num_grids_changes", "min_num_grids", "max_num_grids")
# short periods so that a few days of bars hold many rebalances and adjustments
RANGES = {"num_grids": (3, 30), "grid_type": (0, 1), "lower_boundary_pct": (0.3, 4.0), "upper_boundary_pct": (0.3, 4.0),
          "auto_boundaries": (0, 1), "volatility_lookback": (1, 3), "rebalance_frequency": (60, 7200),
          "auto_adjust_period": (300, 14400), "adapt_to_market_regime": (0, 1)}


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def market_of(torch, closes, bar_minutes=1, minute0=M0, symbols=None):
    from ai_crypto_trader_b200.sweep import MarketData
    c = np.asarray(closes, dtype=np.float32)
    c = c[None] if c.ndim == 1 else c
    ohlcv = np.zeros((5,) + c.shape, dtype=np.float32)
    ohlcv[3] = c
    return MarketData(ohlcv, minute0=minute0, bar_minutes=bar_minutes, symbols=symbols)


def random_population(n, seed, ranges=RANGES):
    rng = random.Random(seed)
    return [{k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi)) for k, (lo, hi) in ranges.items()}
            for _ in range(n)]


def lattice_market(rng, S, N):
    """S symbols: log-normal walks and walks on a coarse lattice with flat stretches (exact level hits)."""
    close = np.empty((S, N), dtype=np.float32)
    for s in range(S):
        if s % 3 == 2:
            steps = np.where(rng.random(N) < 0.4, 0, rng.integers(-3, 4, N)) * (1024 / 64)
            close[s] = 1024 + np.clip(np.cumsum(steps) / 8, -400, 800)
        else:
            close[s] = np.round((100 + 50 * s) * np.exp(np.cumsum(0.002 * rng.standard_normal(N))) * 16) / 16
    return close


def ref_service(sweep, params, days=False):
    from ai_crypto_trader_b200 import grid
    m = sweep.market
    d = grid.decode_individual(params, sweep.defaults, m.bar_minutes)
    _, bounds = sweep.decode([params])
    close = m.close.cpu().numpy().astype(np.float64)[:, sweep.start_bar:]
    labels = sweep.labels[0].cpu().numpy()[sweep.start_bar:] if sweep.labels is not None else None
    table = {r: (t.num_grids, t.lower_pct, t.upper_pct) for r, t in enumerate(sweep.table) if t.apply}
    day_idx = None
    if days:
        day_idx = [(m.minute0 + (sweep.start_bar + k) * m.bar_minutes) // 1440 for k in range(m.N - sweep.start_bar)]
    return grid_service_ref.simulate_service(
        close, [tuple(bounds[0, s]) for s in range(m.S)], d["num_grids"], d["grid_type"], list(sweep.quantity),
        d["lower_pct"], d["upper_pct"], d["rebalance_ticks"], d["adjust_ticks"], bool(d["flags"] & 1), labels, table,
        60 * m.bar_minutes, day_idx)


def check_population(sweep, population, tol=1e-9):
    """Every individual whose lanes have no geometric near tie: lane counts, grids and the service record exact, sums
    within tol.  Returns the number of individuals skipped for near ties."""
    st = sweep.grid_stats(population)
    sv = sweep.service_stats()
    skipped = 0
    for i, params in enumerate(population):
        if np.any(st["near_ties"][i] > 0):
            skipped += 1
            continue
        want = ref_service(sweep, params)
        for s, lane in enumerate(want["lanes"]):
            for f in EXACT:
                assert st[f][i, s] == lane[f], (i, s, f, st[f][i, s], lane[f])
            for f in ("total_profit", "cash", "profit_per_day", "mark_to_market", "win_rate"):
                assert math.isclose(st[f][i, s], lane[f], rel_tol=tol, abs_tol=tol * max(1.0, abs(lane["cash"]))), \
                    (i, s, f)
        for f in SERVICE_EXACT:
            assert sv[f][i] == want["service"][f], (i, f, sv[f][i], want["service"][f])
        for f in ("total_profit", "profit_per_day"):
            assert math.isclose(sv[f][i], want["service"][f], rel_tol=tol, abs_tol=tol), (i, f)
    return skipped


@pytest.mark.parametrize("S,bar_minutes", [(1, 1), (2, 5), (3, 1), (3, 60), (16, 1), (17, 5), (40, 1)])
def test_random_population_against_the_restatement(torch, S, bar_minutes):
    from ai_crypto_trader_b200.grid import GridSweep
    rng = np.random.default_rng(100 * S + bar_minutes)
    lookback = 3 * 1440 // bar_minutes
    N = lookback + (3000 if S <= 3 else 1200) * (1 if bar_minutes == 1 else 2)
    m = market_of(torch, lattice_market(rng, S, N), bar_minutes)
    labels = torch.tensor(np.repeat(rng.integers(0, 6, N // 30 + 1), 30)[:N], dtype=torch.uint8, device="cuda")[None]
    sweep = GridSweep(m, quantity=[0.01 * (s + 1) for s in range(S)], regime=labels, start_bar=lookback + 3,
                      service=True)
    pop = random_population(10 if S <= 3 else 4, S + bar_minutes)
    pop.append({"num_grids": 10, "grid_type": 0, "auto_boundaries": 0, "lower_boundary_pct": 1.0,
                "upper_boundary_pct": 1.0, "adapt_to_market_regime": 1, "rebalance_frequency": 600,
                "auto_adjust_period": 1200 * bar_minutes})
    skipped = check_population(sweep, pop)
    assert skipped <= len(pop) // 2
    sv = sweep.service_stats()
    assert sv["n_adjustments"][-1] > 0


def test_coupling_acts(torch):
    """Without a regime source the win-rate steps of several symbols add up: the service's num_grids trajectory is not
    the one of any single lane of the per-lane sweep."""
    from ai_crypto_trader_b200.grid import GridSweep
    up = [[100.0 + 0.25 * k for k in range(400)] for _ in range(3)]       # every crossing is profitable
    m = market_of(torch, up)
    p = {"num_grids": 6, "grid_type": 0, "auto_boundaries": 0, "lower_boundary_pct": 1.0, "upper_boundary_pct": 1.0,
         "adapt_to_market_regime": 0, "rebalance_frequency": 240, "auto_adjust_period": 3540}
    svc = GridSweep(m, quantity=0.1, start_bar=0, service=True)
    lane = GridSweep(m, quantity=0.1, start_bar=0)
    a, b = svc.grid_stats([p]), lane.grid_stats([p])
    sv = svc.service_stats()
    assert sv["max_num_grids"][0] == 20 and sv["n_num_grids_changes"][0] == 3       # 6 -> 12 -> 18 -> 20
    assert not np.array_equal(a["total_trades"], b["total_trades"])
    assert check_population(svc, [p]) == 0


def test_bit_equal_to_the_lane_sweep_where_nothing_couples(torch):
    """An adjust period longer than the series (one symbol or three): the lanes are b200bt_grid_sweep's, bit for bit
    (stats and day rows)."""
    from ai_crypto_trader_b200.grid import GridSweep
    rng = np.random.default_rng(8)
    N = 4 * 1440 + 4000
    close = lattice_market(rng, 3, N)
    for S in (1, 3):
        m = market_of(torch, close[:S], 1, M0 + 333)
        pop = [dict(p, auto_adjust_period=10 ** 7) for p in random_population(24, 40 + S)]
        kw = dict(quantity=0.05, start_bar=3 * 1440 + 1)
        svc, lane = GridSweep(m, service=True, **kw), GridSweep(m, **kw)
        a, b = svc.grid_stats(pop), lane.grid_stats(pop)
        for f in a:
            assert np.array_equal(a[f], b[f], equal_nan=True), (S, f)
        ra, _ = svc.day_profit(pop)
        rb, _ = lane.day_profit(pop)
        assert torch.equal(ra.view(torch.int64), rb.view(torch.int64)), S
        for f in a:                                    # the day path changes no stat
            assert np.array_equal(svc.grid_stats()[f], a[f]), f


def test_deterministic_duplicates_and_day_rows(torch):
    from ai_crypto_trader_b200.grid import GridSweep
    rng = np.random.default_rng(21)
    S, N = 17, 3 * 1440 + 2500
    m = market_of(torch, lattice_market(rng, S, N), 1, M0 + 777)
    sweep = GridSweep(m, quantity=0.02, start_bar=3 * 1440 + 5, service=True)
    pop = random_population(12, 9)
    sweep.grid_stats(pop)
    a, sa = sweep.stats_device().clone(), sweep._service.clone()
    sweep.grid_stats(pop)
    assert torch.equal(a.view(torch.int64), sweep.stats_device().view(torch.int64))
    assert torch.equal(sa.view(torch.int64), sweep._service.view(torch.int64))
    dup = pop[:3] + pop[:3] + pop[3:6]
    st = sweep.grid_stats(dup)
    assert sweep._inverse is not None
    assert np.array_equal(st["total_profit"][:3], st["total_profit"][3:6])
    assert np.array_equal(sweep.service_stats()["num_grids"][6:], sa[3:6, 5].cpu().numpy())
    rows, first_day = sweep.day_profit(pop)
    rows = rows.cpu().numpy()
    st = sweep.grid_stats()
    sv = sweep.service_stats()
    assert np.allclose(rows.sum(axis=1), sv["total_profit"], rtol=1e-12, atol=1e-9)
    for i in (0, 5):
        if np.any(st["near_ties"][i] > 0):
            continue
        want = ref_service(sweep, pop[i], days=True)["day_profit"]
        ref = np.zeros(rows.shape[1])
        for d, v in want.items():
            ref[d - first_day] += v
        assert np.allclose(rows[i], ref, rtol=1e-12, atol=1e-9), i


def test_nan_stats_for_out_of_limit_individuals(torch):
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.grid import GridSweep
    rng = np.random.default_rng(2)
    m = market_of(torch, lattice_market(rng, 3, 3000))
    sweep = GridSweep(m, quantity=0.1, start_bar=10, service=True)
    good = {"num_grids": 8, "auto_boundaries": 0}
    packed, bounds = sweep.decode([good, good, good])
    rows = (_lib.GridIndividual * 3).from_buffer_copy(packed.tobytes())
    rows[1].num_grids = 0
    rows[2].adjust_ticks = 0
    indiv = torch.from_numpy(np.frombuffer(bytes(rows), dtype=np.uint8).copy()).cuda()
    bnd = torch.from_numpy(bounds).cuda()
    stats = torch.zeros((3, 3, 20), dtype=torch.float64, device="cuda")
    service = torch.zeros((3, 12), dtype=torch.float64, device="cuda")
    _lib.call("b200bt_grid_service_sweep", m.close.data_ptr(), _lib.ld(m.close), 3, m.N, 10, 1, m.minute0,
              indiv.data_ptr(), 3, sweep._qty.data_ptr(), bnd.data_ptr(), None, 0, None, stats.data_ptr(),
              service.data_ptr(), None, 0, _lib.current_stream())
    st, sv = stats.cpu().numpy(), service.cpu().numpy()
    assert np.all(np.isfinite(st[0])) and np.all(np.isfinite(sv[0]))
    assert np.all(np.isnan(st[1:])) and np.all(np.isnan(sv[1:]))
    ref = GridSweep(m, quantity=0.1, start_bar=10, service=True)
    want = ref.grid_stats([good])
    for k, f in enumerate(_lib.GRID_STATS_FIELDS):
        assert np.array_equal(st[0, :, k], want[f][0]), f
    assert np.array_equal(sv[0], [ref.service_stats()[f][0] for f in _lib.GRID_SERVICE_FIELDS])


def test_regime_true_needs_the_primary_symbol(torch, monkeypatch):
    from ai_crypto_trader_b200.grid import GridSweep
    from ai_crypto_trader_b200 import synth
    m = market_of(torch, synth.synth_ohlcv(2, 5 * 1440)[3], symbols=["ETHUSDC", "BNBUSDC"])
    monkeypatch.delenv("PRIMARY_TRADING_SYMBOL", raising=False)
    with pytest.raises(ValueError):
        GridSweep(m, regime=True, service=True)
    monkeypatch.setenv("PRIMARY_TRADING_SYMBOL", "BNBUSDC")
    sweep = GridSweep(m, regime=True, service=True, start_bar=2 * 1440)
    assert sweep.labels.shape == (1, m.N) and sweep.ld_labels == 0
    labels = torch.zeros((2, m.N), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        GridSweep(m, regime=labels, service=True)


def test_objective_matrix_ga_and_backtest_service(torch):
    from ai_crypto_trader_b200.genetic_algorithm import GeneticAlgorithm
    from ai_crypto_trader_b200.grid import GridSweep, GridTradingStrategy, grid_param_ranges
    from ai_crypto_trader_b200 import synth
    m = market_of(torch, synth.synth_ohlcv(3, 45 * 1440)[3], symbols=["BTCUSDC", "ETHUSDC", "BNBUSDC"])
    sweep = GridSweep(m, quantity=0.01, service=True)
    pop = random_population(20, 4, grid_param_ranges())
    objs = [(f, True) for f in ("total_profit", "mark_to_market", "win_rate", "num_grids")]
    got = sweep.evaluate_objectives(pop, objs)
    st = sweep.grid_stats()
    for j, (f, _) in enumerate(objs):
        want = np.array([sum(st[f][i, s] for s in range(m.S)) / m.S for i in range(len(pop))])
        assert np.array_equal(got[:, j], want), f
    assert np.array_equal(sweep.evaluate(pop), got[:, 0])
    seed = {"num_grids": 10, "grid_type": 0, "lower_boundary_pct": 5.0, "upper_boundary_pct": 5.0, "auto_boundaries": 1,
            "volatility_lookback": 14, "rebalance_frequency": 3600, "auto_adjust_period": 86400,
            "adapt_to_market_regime": 1}
    seed_fit = sweep.evaluate([seed])[0]
    ga = GeneticAlgorithm(grid_param_ranges(), sweep.fitness_function, population_size=16, generations=2, random_seed=1)
    ga.run([seed])
    assert ga.best_fitness >= seed_fit
    res = GridTradingStrategy({"grid_trading": {"quantity_per_grid": 0.01}}).backtest_service(m, seed)
    assert res is not None and set(res["grid_profits"]) == {"BTCUSDC", "ETHUSDC", "BNBUSDC"}
    st = sweep.grid_stats([seed])
    assert res["performance"]["total_trades"] == int(st["total_trades"][0].sum())
    assert res["performance"]["symbol_profits"]["ETHUSDC"] == st["total_profit"][0, 1]


def test_fixture_cases_on_the_gpu(torch):
    from ai_crypto_trader_b200.grid import GridSweep
    fx = json.loads(GOLDEN.read_text())
    for case in fx["cases"]:
        bm = case["bar_minutes"]
        closes, lab = grid_service_ref.fixture_series(fx, case)
        m = market_of(torch, closes, bm, case["minute0"], symbols=case["symbols"])
        labels = torch.tensor(lab, dtype=torch.uint8, device="cuda")[None] if lab else None
        sweep = GridSweep(m, start_bar=case["start_bar"], regime=labels, config=case["config"], service=True)
        st = sweep.grid_stats([{}])
        sv = {f: float(v[0]) for f, v in sweep.service_stats().items()}
        name = case["name"]
        if np.any(st["near_ties"][0] > 0):
            assert case["config"].get("grid_type") == "geometric", name
            continue
        for s, sym in enumerate(case["symbols"]):
            gp = case["grid_profits"][sym]
            assert st["total_trades"][0, s] == gp["total_trades"], (name, sym)
            assert st["profitable_trades"][0, s] == gp["profitable_trades"], (name, sym)
            assert math.isclose(st["total_profit"][0, s], gp["total_profit"], rel_tol=1e-12, abs_tol=1e-12), (name, sym)
            regens = case["regenerations"][sym]
            assert st["n_regenerations"][0, s] == len(regens) - 1, (name, sym)
            assert [st["num_grids"][0, s], st["lower"][0, s], st["upper"][0, s]] == \
                [regens[-1][1]] + case["final_grid"][sym], (name, sym)
        f = case["final"]
        assert (sv["num_grids"], sv["lower_pct"], sv["upper_pct"]) == \
            (f["num_grids"], f["lower_boundary_pct"], f["upper_boundary_pct"]), name
        perf = case["performance"]
        assert (sv["total_trades"], sv["profitable_trades"]) == (perf["total_trades"], perf["profitable_trades"]), name
        assert math.isclose(sv["total_profit"], perf["total_profit"], rel_tol=1e-12, abs_tol=1e-12), name
