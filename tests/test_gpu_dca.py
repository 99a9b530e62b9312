"""b200bt_dca_dip_pct and b200bt_dca_sweep on the H100 against the restatements (tests/dca_ref.py, themselves pinned to the
reference's run()): every stats field, service total and day row compared with ==.  The fixture's cases, random
populations on 1-, 5- and 1440-minute clocks with and without labels and rebalancing, S = 1, 3, 10 and 32 (33 with and
without rebalancing), duplicates and determinism, the objective matrix, the GA loops and a configs[1]-sized run."""
import json
import random
from pathlib import Path

import numpy as np
import pytest

import dca_ref

pytestmark = pytest.mark.gpu
M0 = 28_401_120


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def market_of(torch, closes, highs, bar_minutes=1, minute0=M0, symbols=None):
    from ai_crypto_trader_b200.sweep import MarketData
    c = np.atleast_2d(np.asarray(closes, dtype=np.float32))
    ohlcv = np.zeros((5,) + c.shape, dtype=np.float32)
    ohlcv[3] = c
    ohlcv[1] = np.atleast_2d(np.asarray(highs, dtype=np.float32))
    return MarketData(ohlcv, minute0=minute0, bar_minutes=bar_minutes, symbols=symbols)


def random_market(torch, S, N, bar_minutes, seed, minute0=M0):
    rng = np.random.default_rng(seed)
    vol = 0.002 * np.sqrt(bar_minutes)
    base = 100.0 * 10.0 ** (np.arange(S) % 4)
    close = base[:, None] * np.exp(np.cumsum(vol * rng.standard_normal((S, N)), axis=1))
    close = (np.round(close * 16) / 16).clip(1 / 16).astype(np.float32)
    high = (close * (1 + np.abs(rng.normal(0, vol, (S, N))))).astype(np.float32)
    return market_of(torch, close, np.maximum(high, close), bar_minutes, minute0)


def random_population(n, seed, **fixed):
    from ai_crypto_trader_b200.dca import dca_param_ranges
    rng = random.Random(seed)
    return [dict({k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi))
                  for k, (lo, hi) in dca_param_ranges().items()}, **fixed) for _ in range(n)]


def ref_individual(sweep, params):
    from ai_crypto_trader_b200 import dca
    m = sweep.market
    dec = dca.decode_individual(params, sweep.block, m.symbols, m.bar_minutes)
    labels = None if sweep.labels is None else sweep.labels.cpu().numpy()
    return dca_ref.simulate(m.close.cpu().numpy().astype(np.float64), sweep.dip.cpu().numpy(), m.minute0, m.bar_minutes,
                            sweep.start_bar, dec, labels=labels, precision=sweep.precision,
                            usdc_balance=sweep.usdc_balance)


def check(sweep, population, individuals=None, rows=None):
    from ai_crypto_trader_b200.dca import FIELDS
    st = sweep.dca_stats()
    sv = sweep.service_stats()
    first_day, D = sweep.calendar_days()
    for i in (range(len(population)) if individuals is None else individuals):
        want = ref_individual(sweep, population[i])
        for s in range(sweep.market.S):
            for f in FIELDS:
                assert st[f][i, s] == want["stats"][s][f], (i, s, f, st[f][i, s], want["stats"][s][f])
        for f, v in want["service"].items():
            assert sv[f][i] == v, (i, f)
        if rows is not None:
            full = np.zeros(D)
            for d, v in want["day"].items():
                full[d - first_day] = v
            assert np.array_equal(rows[i], full), i
    return st


def test_dip_series_against_the_restatement(torch):
    from ai_crypto_trader_b200.dca import dip_pct
    for bm, m0, N in ((1, M0 + 3, 20 * 1440), (5, M0 + 1437, 9 * 288), (1440, M0, 40), (60, M0 + 30, 24 * 15)):
        m = random_market(torch, 3, N, bm, bm, m0)
        got = dip_pct(m).cpu().numpy()
        high, close = m.high.cpu().numpy(), m.close.cpu().numpy()
        for s in range(3):
            want = dca_ref.dip_series(high[s].astype(np.float64), close[s].astype(np.float64), m0, bm)
            assert np.array_equal(got[s], want, equal_nan=True), (bm, s)


def test_fixture_cases_on_the_gpu(torch):
    from test_dca_host import CASES, precision_of, POSITION_FIELDS
    from ai_crypto_trader_b200.dca import DCASweep
    for case in CASES:
        m = market_of(torch, case["closes"], case["highs"], case["bar_minutes"], case["minute0"], case["symbols"])
        labels = None if case["labels"] is None else torch.from_numpy(case["labels"]).cuda()
        sweep = DCASweep(m, config=case["config"], regime=labels, start_bar=case["start_bar"], usdc_balance=case["usdc"],
                         quantity_precision=precision_of(case))
        st = sweep.dca_stats([{}])
        for s, sym in enumerate(case["symbols"]):
            want = case["positions"][sym]
            for f in POSITION_FIELDS:
                assert st[f][0, s] == want[f], (case["name"], sym, f)
            kinds = [p[1] for p in want["purchases"]]
            assert (st["n_scheduled"][0, s], st["n_dip"][0, s], st["n_rebalance"][0, s]) == \
                (kinds.count("scheduled"), kinds.count("dip"), kinds.count("rebalance"))
            assert st["next_scheduled_us"][0, s] == case["next_scheduled_us"][sym]
            assert st["last_dip_tick"][0, s] == case["last_dip_tick"][sym]
        sv = sweep.service_stats()
        assert {k: v[0] for k, v in sv.items()} == case["service"], case["name"]
        check(sweep, [{}])


@pytest.mark.parametrize("bar_minutes", [1, 5, 1440])
@pytest.mark.parametrize("labelled", [False, True])
def test_random_populations_against_the_restatement(torch, bar_minutes, labelled):
    from ai_crypto_trader_b200.dca import DCASweep
    S = 3
    N = {1: 25 * 1440, 5: 40 * 288, 1440: 400}[bar_minutes]
    m = random_market(torch, S, N, bar_minutes, 100 + bar_minutes)
    labels = None
    if labelled:
        rng = np.random.default_rng(bar_minutes)
        labels = torch.tensor(rng.integers(0, 7, (S, N)), dtype=torch.uint8, device="cuda")
    cfg = {"symbol_settings": [{"symbol": m.symbols[-1], "allocation": 0.5, "interval_hours": 13,
                                "base_order_size_usdc": 70}],
           "scheduling_strategies": {"weighted_scheduling": {"enabled": True}}}
    sweep = DCASweep(m, config=cfg, regime=labels, start_bar=N // 10, usdc_balance=1500.0,
                     quantity_precision=[6, 3, 0])
    pop = random_population(24, bar_minutes) + random_population(8, 7, periodic_rebalancing=0)
    pop += random_population(4, 8, rebalance_interval_days=0, max_dip_frequency_days=0, dip_threshold_pct=0.5)
    sweep.dca_stats(pop)
    rows, first_day = sweep.day_pnl(pop)
    st = check(sweep, pop, rows=rows.cpu().numpy())
    assert st["n_rebalance"].sum() > 0 and st["n_dip"].sum() > 0 and st["n_zero_quantity"].sum() > 0
    assert np.all(rows.cpu().numpy()[:, : (M0 + N // 10 * bar_minutes) // 1440 - M0 // 1440] == 0.0)


@pytest.mark.parametrize("S", [1, 10, 32, 33])
def test_symbol_counts(torch, S):
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.dca import DCASweep
    m = random_market(torch, S, 12 * 288, 5, S)
    pop = random_population(6, S, periodic_rebalancing=0)
    sweep = DCASweep(m, start_bar=288)
    if S > 32:
        with pytest.raises(_lib.B200btError):
            sweep.dca_stats(random_population(2, 1, periodic_rebalancing=1))
    else:
        pop += random_population(6, S + 1, periodic_rebalancing=1, rebalance_interval_days=1)
    sweep.dca_stats(pop)
    check(sweep, pop, individuals=range(0, len(pop), 2))


def test_deterministic_and_duplicates(torch):
    from ai_crypto_trader_b200.dca import DCASweep
    m = random_market(torch, 4, 30 * 1440, 1, 5)
    sweep = DCASweep(m, start_bar=1440)
    pop = random_population(30, 9)
    sweep.dca_stats(pop)
    a = sweep.stats_device().clone()
    sweep.dca_stats(pop)
    b = sweep.stats_device().clone()
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    dup = pop[:5] + pop[:5] + pop[5:10]
    st = sweep.dca_stats(dup)
    assert sweep._inverse is not None
    assert np.array_equal(st["purchase_hash"][:5], st["purchase_hash"][5:10])
    assert np.array_equal(st["total_invested"][10:], a[5:10, :, 0].cpu().numpy())


def test_objective_matrix_and_fitness(torch):
    from ai_crypto_trader_b200.dca import DCASweep, OBJECTIVE_FIELDS
    m = random_market(torch, 3, 20 * 1440, 1, 6)
    sweep = DCASweep(m, start_bar=1440)
    pop = random_population(33, 4)
    objs = [(f, True) for f in ("profit_loss_pct", "total_profit_pct", "n_dip", "min_day_profit_loss", "total_value")]
    got = sweep.evaluate_objectives(pop, objs)
    st, sv = sweep.dca_stats(), sweep.service_stats()
    for j, (f, _) in enumerate(objs):
        want = sv[f] if f in sv else np.array([sum(st[f][i, s] for s in range(m.S)) / m.S for i in range(len(pop))])
        assert np.array_equal(got[:, j], want), f
    fit = sweep.evaluate(pop)
    assert np.array_equal(fit, got[:, 1])
    assert sweep.fitness_function.batch(pop) == [float(x) for x in fit]
    with pytest.raises(ValueError):
        sweep.evaluate_objectives(pop, [("purchase_hash", True)])
    assert "purchase_hash" not in OBJECTIVE_FIELDS


def test_genetic_algorithms_over_dca_sweep(torch):
    from ai_crypto_trader_b200.genetic_algorithm import DeviceGeneticAlgorithm, ParetoGeneticAlgorithm
    from ai_crypto_trader_b200.dca import DCASweep, dca_param_ranges
    m = random_market(torch, 3, 60 * 1440, 1, 8)
    sweep = DCASweep(m, start_bar=1440, usdc_balance=1000.0)
    seed = random_population(1, 1)[0]
    seed_fit = sweep.evaluate([seed])[0]
    dga = DeviceGeneticAlgorithm(dca_param_ranges(), sweep.fitness_function, population_size=24, generations=3,
                                 random_seed=2)
    dga.run([seed])
    assert dga.best_fitness >= seed_fit
    objs = [("total_profit_pct", True), ("min_day_profit_loss", True)]
    pga = ParetoGeneticAlgorithm(dca_param_ranges(), lambda p: sweep.evaluate_objectives_device(p, objs), objs,
                                 population_size=24, generations=3, random_seed=3)
    front = pga.run([seed])
    assert front and max(f["objectives"]["total_profit_pct"] for f in front) >= seed_fit


def test_backtest_result_shape(torch):
    from ai_crypto_trader_b200.dca import DCAStrategy
    m = random_market(torch, 2, 10 * 1440, 1, 9)
    out = DCAStrategy({"dca_strategy": {"interval_hours": 12}}).backtest(m, {"dip_threshold_pct": 2.0}, start_bar=1440)
    assert set(out) == {"dca_positions", "dca_performance", "stats"}
    assert set(out["dca_positions"]) == set(m.symbols)
    assert out["dca_performance"]["total_purchases"] > 0
    assert DCAStrategy().backtest(m, {}, start_bar=10 ** 9) is None


def test_configs1_sized_run(torch):
    """BASELINE configs[1]'s shape: 1024 individuals x 10 symbols x 1M 1-minute bars; 7 individuals (70 lanes) against
    the restatement."""
    from ai_crypto_trader_b200.dca import DCASweep
    from ai_crypto_trader_b200 import synth
    ohlcv = synth.synth_ohlcv(10, 1_000_000)
    m = market_of(torch, ohlcv[3], np.maximum(ohlcv[1], ohlcv[3]))
    sweep = DCASweep(m, start_bar=7 * 1440, usdc_balance=5000.0)
    pop = random_population(1024, 77)
    st = sweep.dca_stats(pop)
    assert np.all(np.isfinite(st["total_invested"])) and np.all(st["n_ticks"] == m.N - sweep.start_bar)
    check(sweep, pop, individuals=[int(i) for i in np.random.default_rng(1).integers(0, 1024, 7)])
