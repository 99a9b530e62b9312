"""Book metrics on the GPU at scale and through the service layer:

* the reference's own multi-symbol books (tests/golden/book_reference.*) through PopulationSweep(aggregation="book");
* 64 symbols (K = 512 / 64 = 8 staged records per symbol and window: windows bounded by the staged records, not by bars);
* configs[1] at full size (1024 individuals x 10 symbols x 1M bars): EVERY book of a random population and of the
  generation-3 population of a GA run (dense records) against the oracle;
* the event-buffer budget when a learnt cap is too small;
* a short GA run under aggregation="book", StrategyEvaluationSystem.evaluate_book / evaluate_population and the
  aggregation option of StrategyEvolutionService.
Oracle: tests/book_ref.py on oracle/sim_oracle.c's lanes.  Exact: counts, trade hash, days, merged-pair durations;
float statistics, score and fitness rel 1e-9."""
import json
import os
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pytest

from gpu_fixtures import torch_cuda

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"
DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)


def _books(close, bank, period_row, population, cfg):
    """Oracle books of `population` (list of dicts).  Lanes and books run in threads (ctypes and NumPy release the GIL),
    128 individuals at a time: their event lists are held at once."""
    import book_ref
    from oracle import sim_oracle
    workers = min(32, os.cpu_count() or 1)
    books = []
    with ThreadPoolExecutor(max_workers=workers) as ex:
        for k in range(0, len(population), 128):
            _, evs, pns = sim_oracle.population(close, bank, period_row, population[k:k + 128], cfg,
                                                event_cap=close.shape[1] + 2, workers=workers)
            books += ex.map(lambda ev, pn: book_ref.book(ev, pn, cfg), evs, pns)
    return books


def test_reference_books(torch_cuda):
    """The reference's own calculate_metrics / calculate_advanced_metrics / _calculate_strategy_score of multi-symbol
    lists (tests/golden/make_book.py) against the GPU book pass."""
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    meta = json.loads((GOLD / "book_reference.json").read_text())
    arrays = np.load(GOLD / "book_reference.npz")
    for case in meta["cases"]:
        close, rsi = arrays[f"close_{case['name']}"], arrays[f"rsi_{case['name']}"]
        market = MarketData.from_close(torch_cuda.from_numpy(close).cuda(), minute0=meta["minute0"],
                                       bar_minutes=case["bar_minutes"])
        bank = torch_cuda.from_numpy(np.ascontiguousarray(rsi)).cuda()
        pop = [b["params"] for b in case["books"]]
        for k, g in enumerate([{"goals": meta["goals"], "advanced": False}] + meta["alt_goals"]):
            sweep = PopulationSweep.from_bank(market, bank, meta["periods"], optimization_goals=g["goals"],
                                              score_on_advanced=g["advanced"], aggregation="book")
            fit = sweep.evaluate(pop)
            want = [b["score"] if k == 0 else b["alt_scores"][k - 1] for b in case["books"]]
            np.testing.assert_allclose(fit, [float(w) for w in want], rtol=1e-9, atol=1e-12, equal_nan=True,
                                       err_msg=f"{case['name']}: {g}")
        st = sweep.book_stats()
        for i, b in enumerate(case["books"]):
            m = b["metrics"]
            assert st["n_records"][i] == m["total_trades"]
            for mine, theirs, rel in (("net_profit", "net_profit", 1e-9), ("max_drawdown", "max_drawdown", 1e-9),
                                      ("sharpe_ratio", "sharpe_ratio", 1e-9), ("win_rate", "win_rate", 1e-12),
                                      ("return_pct", "return_pct", 1e-9),
                                      ("avg_trade_duration", "avg_trade_duration", 1e-12)):
                assert st[mine][i] == pytest.approx(float(m[theirs]), rel=rel, abs=1e-11), (case["name"], i, mine)
            assert st["n_days"][i] == len(b["daily_returns"]) or m["total_trades"] < 2
            prof = {f"SYN{s:03d}USDT" for s in np.nonzero(st["profitable_symbols"][i])[0]}
            assert prof == set(b["profitable_symbols"]), (case["name"], i)


def test_sixty_four_symbols(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    S, N = 64, 12_000
    close = np.ascontiguousarray(synth.synth_ohlcv(5, N)[3][[s % 5 for s in range(S)]])
    market = MarketData.from_close(torch_cuda.from_numpy(close).cuda())
    periods = (5, 14)
    bank = PopulationSweep(market, rsi_periods=periods, mode="fused").bank.clone()
    pop = synth.random_population(6, seed=2)
    for p in pop:
        p["rsi_period"] = periods[int(p["rsi_period"]) % 2]
    pop += [dict(DENSE), dict(DENSE, rsi_overbought=55, take_profit=0.5)]
    sweep = PopulationSweep.from_bank(market, bank, periods, aggregation="book")
    fit = sweep.evaluate(pop)
    want = _books(close, bank.cpu().numpy(), {5: 0, 14: 1}, pop, sim_oracle.config_of(market.minute0, 1))
    sim_oracle.assert_lanes(sweep.book_stats(), want, "S = 64")
    np.testing.assert_allclose(fit, [w["score"] for w in want], rtol=1e-9, atol=1e-11, equal_nan=True)
    assert want[len(pop) - 2]["n_records"] > S * N // 4          # the dense books fill windows of 8 records per symbol


def test_full_size_every_book(torch_cuda):
    """configs[1]: every book of a random population and of generation 3 of a GA run against the oracle."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import GeneticAlgorithm
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import sim_oracle
    S, N, POP = 10, 1_000_000, 1024
    ohlcv = synth.synth_ohlcv(S, N)
    market = MarketData(ohlcv)
    random_pop = synth.random_population(POP, seed=42)
    ga = GeneticAlgorithm(synth.param_ranges(), PopulationSweep(market).fitness_function, population_size=POP,
                          generations=3, random_seed=42)
    ga.run(seeded_individuals=random_pop)
    cfg = sim_oracle.config_of(market.minute0, 1)
    records = {}
    for label, pop in (("random", random_pop), ("generation 3", list(ga.population))):
        sweep = PopulationSweep(market, aggregation="book")
        fit = sweep.evaluate(pop)
        want = _books(ohlcv[3], sweep.bank.cpu().numpy(), sweep.period_row, pop, cfg)
        sim_oracle.assert_lanes(sweep.book_stats(), want, label)
        np.testing.assert_allclose(fit, [w["score"] for w in want], rtol=1e-9, atol=1e-11, equal_nan=True)
        records[label] = sum(w["n_records"] for w in want)
    assert records["generation 3"] > 3 * records["random"], records


def test_resweep_keeps_within_the_event_budget(torch_cuda):
    """A learnt cap far too small AND a budget of a few individuals: the lost slices are swept again in pieces whose
    event buffers stay within max_event_bytes, with the same results as one exact sweep."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    S, N = 4, 30_000
    market = MarketData(synth.synth_ohlcv(S, N))
    pop = synth.random_population(20, seed=9) + [dict(DENSE)]
    exact = PopulationSweep(market, aggregation="book", mode="fused")
    fit = exact.evaluate(pop)
    ref = exact.book_stats()
    busiest = int(exact.lane_stats()["n_records"].max())
    budget = 3 * S * 4 * busiest
    tight = PopulationSweep(market, aggregation="book", mode="fused", max_event_bytes=budget)
    tight._book_cap = 16
    np.testing.assert_array_equal(tight.evaluate(pop), fit)
    assert tight.book_resweeps > 0 and 0 < tight.last_event_bytes <= budget, (tight.last_event_bytes, budget)
    got = tight.book_stats()
    for f in ref:
        np.testing.assert_array_equal(got[f], ref[f], err_msg=f)


def _small_market(torch):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    ohlcv = synth.synth_ohlcv(4, 20_000)
    return MarketData(ohlcv), ohlcv


def test_ga_run_reports_the_oracle_book_score(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import GeneticAlgorithm
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import sim_oracle
    market, ohlcv = _small_market(torch_cuda)
    sweep = PopulationSweep(market, aggregation="book")
    ga = GeneticAlgorithm(synth.param_ranges(), sweep.fitness_function, population_size=32, generations=3, random_seed=7)
    best = ga.run()
    top = ga.get_generation_history()[-1]
    want = _books(ohlcv[3], sweep.bank.cpu().numpy(), sweep.period_row, [top["best_individual"]],
                         sim_oracle.config_of(market.minute0, 1))[0]
    assert top["best_fitness"] == pytest.approx(want["score"], rel=1e-9, abs=1e-11)
    assert best == top["best_individual"] or ga.best_fitness >= top["best_fitness"]


def test_evaluate_book_and_the_service_options(torch_cuda):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.evolution import StrategyEvolutionService
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from oracle import simulate_ref
    market, ohlcv = _small_market(torch_cuda)
    ses = StrategyEvaluationSystem(config={})
    params = {"rsi_period": 9, "rsi_overbought": 68, "rsi_oversold": 32, "take_profit": 1.5, "stop_loss": 1.0}
    out = ses.evaluate_book("s1", params, market)
    sweep = PopulationSweep(market, aggregation="book", score_on_advanced=True)
    fit = sweep.evaluate([params])
    st = sweep.book_stats()
    assert out["total_trades"] == st["n_records"][0] > 0
    for mine, key in (("net_profit", "net_profit"), ("max_drawdown", "max_drawdown"), ("sharpe_ratio", "sharpe_ratio"),
                      ("win_rate", "win_rate"), ("profit_factor", "profit_factor"), ("sortino_ratio", "sortino_ratio"),
                      ("return_pct", "return_pct"), ("avg_trade_duration", "avg_trade_duration")):
        assert out[key] == pytest.approx(float(st[mine][0]), rel=1e-9, abs=1e-11), key
    assert out["score"] == fit[0]
    assert {"daily_returns", "monthly_returns", "equity_curve", "profitable_symbols", "unprofitable_symbols"} <= set(out)
    assert len(out["equity_curve"]) == out["total_trades"] + 1 and len(out["daily_returns"]) == st["n_days"][0]
    # the records it formats are those of the reference rule on the concatenated symbols
    trades = []
    bank = sweep.bank.cpu().numpy()
    for s in range(market.S):
        trades += simulate_ref.simulate_trades(params, simulate_ref.market_points(
            ohlcv[3, s], bank[s, sweep.period_row[9]], market.symbols[s], market.minute0))
    ref = simulate_ref.calculate_metrics(trades)
    for key in ("total_trades", "net_profit", "max_drawdown", "sharpe_ratio", "avg_trade_duration"):
        assert out[key] == pytest.approx(ref[key], rel=1e-9, abs=1e-11), key
    assert ses.evaluate_book("bad", dict(params, rsi_period=99), market) == {}
    # evaluate_population and the evolution service
    pop = synth.random_population(12, seed=1)
    book_fit = ses.evaluate_population(pop, market, aggregation="book")
    np.testing.assert_array_equal(book_fit, PopulationSweep(market, aggregation="book").evaluate(pop))
    assert StrategyEvolutionService(market, config={"evolution": {"fitness_aggregation": "book"}}).sweep.aggregation == "book"
    assert StrategyEvolutionService(market, config={}).sweep.aggregation == "mean"
    assert StrategyEvolutionService(market, config={}, aggregation="book").sweep.aggregation == "book"
