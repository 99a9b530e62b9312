"""Generate the committed golden fixtures by EXECUTING the reference's own code.

Run where a copy of the reference tree exists (a checkout named `reference` beside this repository, or
B200BT_REFERENCE_ROOT=<reference tree>):

    python tests/golden/make_golden.py

Writes (all small, committed):
    tests/golden/sim_cases.json   parameter sets + reference metrics / score
    tests/golden/sim_cases.npz    fp32 inputs + reference trade records
    tests/golden/ga_run.json      seeded GeneticAlgorithm trajectory
    tests/golden/mc_reference.*   MonteCarloService results + its own paths (NumPy seed fixed)
    tests/golden/bt_reference.*   StrategyTester.backtest_strategy runs (LLM stubbed, `ta` shimmed)
    tests/golden/pf_reference.json PortfolioRiskService VaR / CVaR / correlation / portfolio VaR
    tests/golden/cv_reference.json StrategyEvaluationSystem.cross_validate_strategy on flat data points
    tests/golden/ra_reference.json ResultAnalyzer load / filter / generate_summary_report on a set of result files
Inputs are the fp32 synthetic series of ai_crypto_trader_b200.synth; the RSI
bank is oracle.indicators_ref.rsi_bank (float64 pandas, rounded to fp32).
The reference functions executed are
    StrategyEvaluationSystem._simulate_trades      services/strategy_evaluation.py:746
    StrategyPerformanceMetrics.calculate_metrics   :32
    StrategyEvaluationSystem._calculate_strategy_score :579
    GeneticAlgorithm                               services/genetic_algorithm.py:27
"""
from __future__ import annotations

import json
import math
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
OUT = Path(__file__).resolve().parent

from ai_crypto_trader_b200 import synth  # noqa: E402
from oracle import indicators_ref, ref_runner, simulate_ref  # noqa: E402

N_BARS = 6000          # 4.2 days of 1-minute bars
PERIODS = list(range(5, 31))

CASES = [
    # name, params
    ("default", {}),
    ("ga_typical", {"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30, "take_profit": 3, "stop_loss": 2}),
    ("fast_rsi_tight", {"rsi_period": 5, "rsi_overbought": 65, "rsi_oversold": 35, "take_profit": 1, "stop_loss": 1}),
    ("slow_rsi_wide", {"rsi_period": 30, "rsi_overbought": 85, "rsi_oversold": 15, "take_profit": 10, "stop_loss": 5}),
    ("leverage_floats", {"rsi_period": 9, "rsi_overbought": 71, "rsi_oversold": 33, "take_profit": 2.7312, "stop_loss": 0.5519}),
    ("tiny_tp_sl", {"rsi_period": 7, "rsi_overbought": 66, "rsi_oversold": 34, "take_profit": 0.05, "stop_loss": 0.05}),
    ("no_trades", {"rsi_period": 20, "rsi_overbought": 99.99, "rsi_oversold": 0.01, "take_profit": 3, "stop_loss": 2}),
    ("big_position", {"rsi_period": 11, "rsi_overbought": 68, "rsi_oversold": 32, "take_profit": 2, "stop_loss": 1, "max_position_size": 50}),
    ("short_bias", {"rsi_period": 6, "rsi_overbought": 65, "rsi_oversold": 15, "take_profit": 1, "stop_loss": 3}),
    ("inverted_thresholds", {"rsi_period": 10, "rsi_overbought": 40, "rsi_oversold": 60, "take_profit": 2, "stop_loss": 2}),
]

SCALARS = ["total_trades", "win_rate", "profit_factor", "sharpe_ratio", "max_drawdown", "average_profit",
           "average_loss", "largest_profit", "largest_loss", "total_profit", "total_loss", "net_profit",
           "return_pct", "avg_trade_duration", "risk_reward_ratio"]


# other optimisation goals (config.json evolution.optimization_goals) x the dict the score is taken on
# (False: calculate_metrics' dict, the composition of cross_validate_strategy; True: calculate_advanced_metrics' dict,
# the composition of evaluate_strategy :545-557)
ALT_GOALS = [
    ({"primary": "return_pct", "secondary": ["win_rate", "expectancy"]}, True),
    ({"primary": "return_pct", "secondary": ["win_rate", "expectancy"]}, False),       # expectancy absent: factor 1
    ({"primary": "sortino_ratio", "secondary": ["max_drawdown"]}, True),
    ({"primary": "sortino_ratio", "secondary": ["max_drawdown"]}, False),              # unknown key: 0
    ({"primary": "expectancy", "secondary": ["profit_factor", "no_such_metric"]}, True),
    ({"primary": "total_trades", "secondary": []}, False),
    ({"primary": "average_loss", "secondary": ["max_drawdown", "win_rate"]}, False),
    ({"primary": "calmar_ratio", "secondary": ["expectancy"]}, True),
    ({"primary": "profit_per_day", "secondary": ["win_rate"], "constraints": {"min_trades_per_day": 20}}, True),
    ({"primary": "largest_profit", "secondary": ["max_drawdown"]}, False),
    ({"primary": "recovery_factor", "secondary": []}, True),
    ({"primary": "not_a_metric", "secondary": ["win_rate"]}, True),
]


def jsonable(x):
    x = float(x)
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    if math.isnan(x):
        return "nan"
    return x


def make_sim():
    ses, metrics_cls = ref_runner.strategy_evaluation()
    goals = ref_runner.optimization_goals()
    arrays = {}
    cases = []
    for sym in (0, 3):
        d = synth.synth_symbol(sym, N_BARS)
        bank = indicators_ref.rsi_bank(d["close"], PERIODS)
        arrays[f"close_{sym}"] = d["close"]
        for period in sorted({c[1].get("rsi_period", 14) for c in CASES}):
            arrays[f"rsi_{sym}_{period}"] = bank[PERIODS.index(period)]
        for name, params in CASES:
            period = params.get("rsi_period", 14)
            rsi_row = bank[PERIODS.index(period)]
            points = simulate_ref.market_points(d["close"], rsi_row, f"SYN{sym:03d}USDT", synth.EPOCH_2024_MINUTES)
            ts_to_bar = {p["timestamp"]: i for i, p in enumerate(points)}
            trades = ses._simulate_trades(name, dict(params), points)            # REFERENCE
            m = metrics_cls.calculate_metrics(trades)                            # REFERENCE
            score = ses._calculate_strategy_score(m)                             # REFERENCE
            adv = metrics_cls.calculate_advanced_metrics(m)                      # REFERENCE (:231-319)
            alt = []
            for g, on_advanced in ALT_GOALS:                                     # REFERENCE (:579-633), other goal sets
                ses.optimization_goals = g
                alt.append(jsonable(ses._calculate_strategy_score(adv if on_advanced else m)))
            ses.optimization_goals = goals
            key = f"{name}_{sym}"
            arrays[f"bar_{key}"] = np.array([ts_to_bar[t["timestamp"]] for t in trades], dtype=np.int64)
            arrays[f"sell_{key}"] = np.array([t["side"] == "sell" for t in trades], dtype=np.bool_)
            arrays[f"price_{key}"] = np.array([t["price"] for t in trades], dtype=np.float64)
            arrays[f"qty_{key}"] = np.array([t["quantity"] for t in trades], dtype=np.float64)
            arrays[f"pnl_{key}"] = np.array([t["pnl"] for t in trades], dtype=np.float64)
            arrays[f"equity_{key}"] = np.array(m.get("equity_curve", [10000.0]), dtype=np.float64)
            daily = m.get("daily_returns", {})
            arrays[f"daily_{key}"] = np.array([daily[k] for k in sorted(daily)], dtype=np.float64)
            cases.append({"key": key, "name": name, "symbol": sym, "params": params,
                          "metrics": {k: jsonable(m[k]) for k in SCALARS}, "score": jsonable(score),
                          "advanced": {k: jsonable(adv[k]) for k in simulate_ref.ADVANCED_KEYS}, "alt_scores": alt,
                          "n_records": len(trades)})
            print(f"{key:28s} records={len(trades):5d} score={float(score):.6g}")
    np.savez_compressed(OUT / "sim_cases.npz", **arrays)
    (OUT / "sim_cases.json").write_text(json.dumps(
        {"n_bars": N_BARS, "periods": PERIODS, "minute0": synth.EPOCH_2024_MINUTES, "goals": goals,
         "alt_goals": [{"goals": g, "advanced": a} for g, a in ALT_GOALS],
         "cases": cases}, indent=1))


def make_ga():
    GA = ref_runner.genetic_algorithm_class()
    ranges = synth.param_ranges()

    def fitness(ind):
        # deterministic toy fitness: smooth, non-degenerate, no data involved
        s = 0.0
        for i, (k, (lo, hi)) in enumerate(ranges.items()):
            x = (ind[k] - lo) / (hi - lo)
            s += math.sin(3.0 * x + 0.37 * i) * (1.0 + 0.1 * i)
        return s

    runs = []
    for pop, gens, seed, seeded in ((20, 10, 42, True), (64, 5, 7, False)):
        ga = GA(param_ranges=ranges, fitness_function=fitness, population_size=pop, generations=gens,
                mutation_rate=0.2, crossover_rate=0.8, elitism_pct=0.1, random_seed=seed)
        seed_ind = {k: (lo + hi) // 2 if isinstance(lo, int) and isinstance(hi, int) else 0.5 * (lo + hi)
                    for k, (lo, hi) in ranges.items()}
        seed_ind["take_profit"] = 300      # out of range: initialize_population clamps (:96-103)
        seed_ind["rsi_period"] = 1
        seeds = [seed_ind] if seeded else None
        best = ga.run(seeded_individuals=seeds)
        hist = ga.get_generation_history()
        runs.append({
            "pop": pop, "generations": gens, "seed": seed, "seeded": seeds,
            "best": best, "best_fitness": ga.best_fitness,
            "final_population": ga.population, "final_fitness": ga.fitness_scores,
            "history": [{k: h[k] for k in ("generation", "best_fitness", "avg_fitness", "min_fitness",
                                           "best_individual", "diversity")} for h in hist],
            "diversity": ga.get_population_diversity(),
        })
        print(f"GA pop={pop} gens={gens} seed={seed}: best_fitness={ga.best_fitness:.6f}")
    (OUT / "ga_run.json").write_text(json.dumps({"runs": runs}, indent=1))




def make_mc():
    """Reference MonteCarloService.run_monte_carlo_simulation, NumPy global seed fixed,
    `store_all_paths` on so the fixture holds the reference's own paths."""
    import pandas as pd
    out = {}
    meta = []
    rng = np.random.default_rng(7)
    returns = rng.normal(5e-4, 0.02, 60)
    for method, n, days, scenario in (("geometric_brownian_motion", 400, 30, "base"),
                                      ("geometric_brownian_motion", 250, 12, "volatile"),
                                      ("historical", 120, 20, "bear")):
        params = {
            "num_simulations": n, "time_horizon_days": days, "confidence_level": 0.95, "lookback_days": 60,
            "return_method": "log", "simulation_method": method, "plot_chart": False, "store_all_paths": True,
            "scenarios": {"base": {}, "bull": {"drift_factor": 1.5, "volatility_factor": 0.8},
                          "bear": {"drift_factor": 0.5, "volatility_factor": 1.2},
                          "volatile": {"drift_factor": 1.0, "volatility_factor": 2.0},
                          "crab": {"drift_factor": 0.2, "volatility_factor": 0.5}}}
        svc = ref_runner.monte_carlo_service(params)
        svc.historical_data["SYNUSDC"] = pd.DataFrame({"returns": returns})
        np.random.seed(20240921)
        res = svc.run_monte_carlo_simulation("SYNUSDC", 100.0, scenario=scenario)      # REFERENCE
        assert res, "reference simulation failed"
        key = f"{method}_{scenario}"
        out[f"paths_{key}"] = np.array(res["paths"], dtype=np.float64)
        res = dict(res); res.pop("paths"); res.pop("timestamp")
        meta.append({"key": key, "method": method, "scenario": scenario, "n": n, "days": days, "result": res})
        print(f"MC {key}: VaR={res['risk_metrics']['var']:.4f} mdd_mean={res['risk_metrics']['max_drawdown']['mean']:.4f}")
    out["returns"] = returns
    # portfolio statistics (:577-659) on reference simulations
    svc = ref_runner.monte_carlo_service(params)
    svc.historical_data["AAAUSDC"] = pd.DataFrame({"returns": returns})
    svc.historical_data["BBBUSDC"] = pd.DataFrame({"returns": returns * 1.5})
    holdings = {"total_value": 15000.0, "assets": {"AAA": {"value_usdc": 6000.0, "current_price": 10.0},
                                                    "BBB": {"value_usdc": 4000.0, "current_price": 2.5},
                                                    "USDC": {"value_usdc": 5000.0, "current_price": 1.0}}}
    np.random.seed(99)
    sims = {}
    for a in ("AAA", "BBB"):
        for sc in params["scenarios"]:
            r = svc.run_monte_carlo_simulation(f"{a}USDC", holdings["assets"][a]["current_price"], scenario=sc)
            r = dict(r); r.pop("paths"); r.pop("timestamp")
            sims[f"{a}USDC_{sc}"] = r
    pstats = svc._calculate_portfolio_stats(holdings, sims)                             # REFERENCE
    np.savez_compressed(OUT / "mc_reference.npz", **out)
    (OUT / "mc_reference.json").write_text(json.dumps(
        {"cases": meta, "portfolio": {"holdings": holdings, "simulations": sims, "stats": pstats}}, indent=1))


def bt_frame(n, crash, vol_scale, sym=0):
    """OHLCV DataFrame for the configs[0] fixtures: the synthetic series, optionally ending in a
    10 % sell-off over the last 60 bars (drives the constant technical signal to BUY/strength>=70)."""
    import pandas as pd
    d = synth.synth_symbol(sym, n)
    cols = {k: d[k].astype(np.float64).copy() for k in synth.FIELDS}
    if crash:
        f = np.ones(n)
        f[-60:] = np.linspace(1.0, 0.90, 60)
        for k in ("open", "high", "low", "close"):
            cols[k] *= f
    cols["volume"] *= vol_scale
    idx = pd.date_range("2024-01-01", periods=n, freq="min")
    return pd.DataFrame({k: v.astype(np.float32).astype(np.float64) for k, v in cols.items()}, index=idx)  # fp32 market data, widened (CSV-loaded frames are float64)


BT_CASES = [("crash_trading", 3000, True, 1000.0, 0), ("quiet_no_entry", 2500, False, 1.0, 1),
            ("crash_lowvolume", 1200, True, 1.0, 2)]


def make_bt():
    """Reference StrategyTester.backtest_strategy (LLM stubbed, `ta` shimmed; oracle/ref_runner.py)."""
    arrays, meta = {}, []
    for name, n, crash, vs, sym in BT_CASES:
        df = bt_frame(n, crash, vs, sym)
        stats, tester, bms = ref_runner.run_reference_backtest(df)                    # REFERENCE
        bar = {t.isoformat(): i for i, t in enumerate(df.index)}
        tr = stats["trades"]
        arrays[f"entry_bar_{name}"] = np.array([bar[t["entry_time"]] for t in tr], dtype=np.int64)
        arrays[f"exit_bar_{name}"] = np.array([bar[t["exit_time"]] for t in tr], dtype=np.int64)
        arrays[f"reason_{name}"] = np.array([{"Stop Loss": 1, "Take Profit": 2, "End of Test": 3}[t["exit_reason"]] for t in tr], dtype=np.int64)
        for k in ("entry_price", "quantity", "position_size", "pnl", "pnl_pct"):
            arrays[f"{k}_{name}"] = np.array([t[k] for t in tr], dtype=np.float64)
        arrays[f"eq_bar_{name}"] = np.array([bar[p["timestamp"]] for p in stats["equity_curve"]], dtype=np.int64)
        arrays[f"eq_{name}"] = np.array([p["equity"] for p in stats["equity_curve"]], dtype=np.float64)
        arrays[f"dd_{name}"] = np.array([[p["drawdown"], p["drawdown_pct"]] for p in stats["drawdown_curve"]], dtype=np.float64).reshape(-1, 2)
        # the per-bar constants the reference feeds its signal (one market update is enough: they are frame constants)
        upd = tester.prepare_market_data(df.iloc[:], "SYNUSDC")[-1]
        sig = bms.TradingSignal(symbol="SYNUSDC", price=upd["current_price"], rsi=upd["rsi"], stoch_k=upd["stoch_k"],
                                macd=upd["macd"], volume=upd["avg_volume"], volatility=upd["volatility"],
                                williams_r=upd["williams_r"], trend=upd["trend"], trend_strength=upd["trend_strength"],
                                bb_position=upd["bb_position"])
        consts = {k: upd[k] for k in ("rsi", "stoch_k", "macd", "williams_r", "bb_position", "trend", "trend_strength",
                                      "volatility", "avg_volume", "price_change_1m", "price_change_3m",
                                      "price_change_5m", "price_change_15m")}
        scal = {k: jsonable(v) if not isinstance(v, str) else v for k, v in stats.items() if not isinstance(v, list)}
        meta.append({"name": name, "n": n, "crash": crash, "vol_scale": vs, "symbol": sym, "stats": scal,
                     "constants": {k: (v if isinstance(v, str) else jsonable(v)) for k, v in consts.items()},
                     "signal": sig.signal, "strength": jsonable(sig.strength), "n_trades": len(tr)})
        print(f"BT {name}: trades={len(tr)} final={stats['final_balance']:.4f} signal={sig.signal} strength={sig.strength:.2f}")
    np.savez_compressed(OUT / "bt_reference.npz", **arrays)
    (OUT / "bt_reference.json").write_text(json.dumps({"cases": meta}, indent=1))


def make_pf():
    """Reference PortfolioRiskService.calculate_var / calculate_conditional_var / calculate_asset_correlation /
    calculate_portfolio_var (services/portfolio_risk_service.py:217-396) on the synthetic closes (fp32 values
    held in float64 frames, as the other fixtures)."""
    import pandas as pd
    svc = ref_runner.portfolio_risk_service()
    S, N = 6, 5000
    ohlcv = synth.synth_ohlcv(S, N)
    close = ohlcv[3].astype(np.float64)
    # make the series co-move a little (the synthetic symbols are independent) and punch holes into one of them
    close[1] = close[1] * (close[0] / close[0][0]) ** 0.5
    close[2] = close[2] * (close[0][0] / close[0]) ** 0.25
    close = close.astype(np.float32).astype(np.float64)
    symbols = [f"S{i}USDC" for i in range(S)]
    frames = {}
    for i, sym in enumerate(symbols):
        df = pd.DataFrame({"close": close[i]})
        df["returns"] = df["close"].pct_change()
        frames[sym] = df
    holes = [100, 101, 2500, 4999]
    frames[symbols[3]].loc[holes, "returns"] = np.nan
    svc.historical_data = frames
    out = {"S": S, "N": N, "symbols": symbols, "holes": holes, "var": {}, "cvar": {}}
    for conf in (0.95, 0.99, 0.9):
        out["var"][str(conf)] = [svc.calculate_var(frames[s]["returns"], conf, 1000.0) for s in symbols]
        out["cvar"][str(conf)] = [svc.calculate_conditional_var(frames[s]["returns"], conf, 1000.0) for s in symbols]
    corr = svc.calculate_asset_correlation(symbols)
    out["correlation"] = [[float(corr[a][b]) for b in symbols] for a in symbols]
    svc.asset_correlations = corr
    values = [1200.0, 800.0, 50.0, 3000.0, 10.0, 440.0]
    holdings = {"assets": {s.replace("USDC", ""): {"value_usdc": v} for s, v in zip(symbols, values)}, "total_value": 6000.0}
    holdings["assets"]["USDC"] = {"value_usdc": 500.0}
    svc.asset_correlations = {a.replace("USDC", ""): {b.replace("USDC", ""): corr[a][b] for b in symbols} for a in symbols}
    var_est = {s.replace("USDC", ""): v / 1000.0 for s, v in zip(symbols, out["var"]["0.95"])}
    out["holdings_values"] = values
    out["portfolio_var"] = float(svc.calculate_portfolio_var(holdings, var_est))
    out["close_transform"] = "close[1] *= (close[0]/close[0][0])**0.5; close[2] *= (close[0][0]/close[0])**0.25; rounded to fp32"
    (OUT / "pf_reference.json").write_text(json.dumps(out, indent=1))
    print("PF: var95", out["var"]["0.95"][:3], "corr01", out["correlation"][0][1], "pvar", out["portfolio_var"])


CV_BARS, CV_SYMBOL, CV_FOLDS = 30000, 2, 5
CV_CASES = [
    ("cv_typical", {"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30, "take_profit": 3, "stop_loss": 2}),
    ("cv_fast", {"rsi_period": 6, "rsi_overbought": 66, "rsi_oversold": 34, "take_profit": 1, "stop_loss": 1}),
    ("cv_holder", {"rsi_period": 21, "rsi_overbought": 80, "rsi_oversold": 20, "take_profit": 10, "stop_loss": 5}),
]


def make_cv():
    """Reference StrategyEvaluationSystem.cross_validate_strategy (services/strategy_evaluation.py:635-744) on a
    FLAT list of market-data points (what its type hint says; with its own caller's list of periods it raises).
    The plotting hook (:739) is switched off on the instance; nothing else is touched."""
    ses, _ = ref_runner.strategy_evaluation()
    ses._visualize_cv_results = lambda results: None
    d = synth.synth_symbol(CV_SYMBOL, CV_BARS)
    out = {"n_bars": CV_BARS, "symbol": CV_SYMBOL, "k_folds": CV_FOLDS, "minute0": synth.EPOCH_2024_MINUTES, "cases": []}
    for name, params in CV_CASES:
        rsi = indicators_ref.rsi_bank(d["close"], [params["rsi_period"]])[0]
        pts = simulate_ref.market_points(d["close"], rsi, f"SYN{CV_SYMBOL:03d}USDT", synth.EPOCH_2024_MINUTES)
        for p, v in zip(pts, d["volume"]):
            p["volume"] = float(v)
        res = ses.cross_validate_strategy(name, dict(params), pts, k_folds=CV_FOLDS)          # REFERENCE
        folds = [{k: (v if k == "market_conditions" else
                      ({m: jsonable(x) for m, x in v.items()} if isinstance(v, dict) else jsonable(v)))
                  for k, v in f.items()} for f in res["fold_results"]]
        out["cases"].append({"name": name, "params": params, "fold_results": folds,
                             "cv_summary": {k: jsonable(v) for k, v in res["cv_summary"].items()}})
        print(f"CV {name}: mean_test_score={res['cv_summary']['mean_test_score']:.6g} "
              f"mean_train_score={res['cv_summary']['mean_train_score']:.6g}")
    (OUT / "cv_reference.json").write_text(json.dumps(out, indent=1))


def ra_results():
    """A small set of backtest result documents in the shape StrategyTester.save_results writes
    (backtesting/strategy_tester.py:432-458): ties, a loss-maker, missing keys, a zero initial balance."""
    def doc(strategy, symbol, interval, ib, fb, trades, wr, pf, sh, dd):
        return {"strategy": strategy, "symbol": symbol, "interval": interval, "start_date": "2024-01-01T00:00:00",
                "end_date": "2024-02-01T00:00:00",
                "stats": {"initial_balance": ib, "final_balance": fb, "total_trades": trades, "win_rate": wr,
                          "profit_factor": pf, "sharpe_ratio": sh, "max_drawdown_pct": dd}}
    docs = [doc("AI_Social_Strategy", "BTCUSDC", "1h", 10000.0, 11234.5, 42, 57.14, 1.62, 1.1, 6.3),
            doc("AI_Social_Strategy", "ETHUSDC", "1h", 10000.0, 9321.25, 18, 38.9, 0.71, -0.8, 11.2),
            doc("AI_Social_Strategy", "BTCUSDC", "5m", 10000.0, 11234.5, 310, 51.0, 1.08, 0.4, 9.9),     # return tie with #0
            doc("Baseline", "SOLUSDC", "1m", 5000.0, 5000.0, 0, 0, 0, 0, 0),
            doc("Baseline", "BTCUSDC", "1h", 0, 120.0, 3, 66.7, 2.5, 0.2, 1.0),                          # zero initial balance
            doc("AI_Social_Strategy", "ETHUSDC", "15m", 20000.0, 26000.0, 77, 61.0, 2.2, 1.9, 4.4)]
    docs.append({"symbol": "XRPUSDC", "stats": {"final_balance": 50.0}})                                  # missing keys
    docs.append({"strategy": "NoStats", "symbol": "ADAUSDC", "interval": "1d"})                           # no stats at all
    return docs


def make_ra():
    """Reference ResultAnalyzer (backtesting/result_analyzer.py:23-72, :226-328): the documents above written as
    result files, then load_results / get_available_results / filter_results / generate_summary_report executed."""
    import tempfile
    ref_runner.strategy_tester()          # imports the reference's `backtesting` package behind the ta / plotting stubs
    from backtesting.result_analyzer import ResultAnalyzer
    d = Path(tempfile.mkdtemp(prefix="b200bt_ra_"))
    docs = ra_results()
    for i, doc in enumerate(docs):
        (d / f"result_{i:02d}.json").write_text(json.dumps(doc))
    (d / "broken.json").write_text("{not json")
    ra = ResultAnalyzer(str(d))
    avail = sorted(ra.get_available_results(), key=lambda r: r["file_path"])
    strip = lambda rs: [dict(r, file_path=Path(r["file_path"]).name) for r in rs]
    by_name = lambda rs: sorted(Path(r["file_path"]).name for r in rs)
    filters = [dict(symbol="BTCUSDC"), dict(strategy="Baseline"), dict(interval="1h", min_trades=10),
               dict(symbol="ETHUSDC", interval="15m"), dict(min_trades=1), dict(strategy="nope")]
    summary = ra.generate_summary_report(avail)
    for k in ("strategies", "symbols", "intervals"):
        summary[k] = sorted(summary[k])
    summary["best_result"] = strip([summary["best_result"]])[0]
    summary["worst_result"] = strip([summary["worst_result"]])[0]
    for r in summary["results"]:
        r["file_path"] = Path(r["file_path"]).name
    out = {"documents": docs, "available": strip(avail),
           "filters": [{"criteria": f, "files": by_name(ra.filter_results(**f))} for f in filters],
           "summary": summary, "summary_empty": ra.generate_summary_report([]),
           "load_missing": ra.load_results(str(d / "does_not_exist.json")),
           "load_first": ra.load_results(str(d / "result_00.json"))}
    (OUT / "ra_reference.json").write_text(json.dumps(out, indent=1))
    print("RA:", len(avail), "results; best", summary["best_result"]["file_path"], "worst", summary["worst_result"]["file_path"])


if __name__ == "__main__":
    which = sys.argv[1:] or ["sim", "ga", "mc", "bt", "pf", "cv", "ra"]
    if "sim" in which:
        make_sim()
    if "ga" in which:
        make_ga()
    if "mc" in which:
        make_mc()
    if "bt" in which:
        make_bt()
    if "pf" in which:
        make_pf()
    if "cv" in which:
        make_cv()
    if "ra" in which:
        make_ra()
