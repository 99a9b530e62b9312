"""k-fold cross-validation (SURVEY 8-f3) against the reference's own cross_validate_strategy outputs."""
import json
from pathlib import Path

import numpy as np
import pytest

from conftest import unjson
from gpu_fixtures import torch_cuda

GOLD = Path(__file__).parent / "golden"
pytestmark = pytest.mark.gpu
CV_CLOSE = ("sharpe_ratio", "max_drawdown", "win_rate", "profit_factor", "score")    # the lane fields a fold reports


def _points(ref, params):
    from ai_crypto_trader_b200 import synth
    from oracle import indicators_ref, simulate_ref
    d = synth.synth_symbol(ref["symbol"], ref["n_bars"])
    rsi = indicators_ref.rsi_bank(d["close"], [params["rsi_period"]])[0]
    pts = simulate_ref.market_points(d["close"], rsi, f"SYN{ref['symbol']:03d}USDT", ref["minute0"])
    for p, v in zip(pts, d["volume"]):
        p["volume"] = float(v)
    return pts, d, rsi


def test_cross_validate_strategy_matches_reference(torch_cuda):
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    ref = json.loads((GOLD / "cv_reference.json").read_text())
    ses = StrategyEvaluationSystem(config={})
    for case in ref["cases"]:
        pts, _, _ = _points(ref, case["params"])
        got = ses.cross_validate_strategy(case["name"], dict(case["params"]), pts, k_folds=ref["k_folds"])
        assert got["k_folds"] == ref["k_folds"] and len(got["fold_results"]) == len(case["fold_results"])
        for g, w in zip(got["fold_results"], case["fold_results"]):
            assert g["fold"] == w["fold"]
            for side in ("train_metrics", "test_metrics"):
                for k, v in w[side].items():
                    assert g[side][k] == pytest.approx(unjson(v), rel=1e-9, abs=1e-12), (case["name"], g["fold"], side, k)
            assert g["train_score"] == pytest.approx(unjson(w["train_score"]), rel=1e-9, abs=1e-12)
            assert g["test_score"] == pytest.approx(unjson(w["test_score"]), rel=1e-9, abs=1e-12)
            mc_g, mc_w = g["market_conditions"], w["market_conditions"]
            assert mc_g["trend"] == mc_w["trend"] and mc_g["period_start"] == mc_w["period_start"]
            assert mc_g["period_end"] == mc_w["period_end"]
            assert mc_g["volatility"] == pytest.approx(mc_w["volatility"], rel=1e-12)
            assert mc_g["volume"] == pytest.approx(mc_w["volume"], rel=1e-12)
        for k, v in case["cv_summary"].items():
            assert got["cv_summary"][k] == pytest.approx(unjson(v), rel=1e-8, abs=1e-10), (case["name"], k)


def test_cross_validate_population_vs_oracle_with_gap(torch_cuda):
    """Batched form on two symbols and a bank of periods: every (fold, individual, symbol) lane equals the C oracle run
    on the glued series with the same calendar gap."""
    import torch
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.strategy_evaluation import StrategyEvaluationSystem
    from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
    from oracle import indicators_ref, sim_oracle
    S, N, K = 2, 20_000, 4
    ohlcv = synth.synth_ohlcv(S, N, first_symbol=4)
    market = MarketData(ohlcv)
    sweep = PopulationSweep(market, mode="fused")
    population = synth.random_population(12, seed=9)
    population[0].update(rsi_oversold=35, rsi_overbought=65, rsi_period=5, take_profit=1, stop_loss=1)
    ses = StrategyEvaluationSystem(config={})
    cv = ses.cross_validate_population(population, market.close, sweep.bank, sweep.periods, market.minute0, 1, K)
    bank = np.stack([indicators_ref.rsi_bank(ohlcv[3, s], sweep.periods) for s in range(S)])
    fold = N // K
    for f in range(K):
        a, b = f * fold, (f + 1) * fold if f < K - 1 else N
        gap = (a, b - a) if 0 < a and b < N else (0, 0)
        m0 = market.minute0 + (b if a == 0 else 0)
        train = [np.concatenate([x[..., :a], x[..., b:]], axis=-1) for x in (ohlcv[3], bank)]
        want_tr, _, _ = sim_oracle.population(*train, sweep.period_row, population,
                                              sim_oracle.config_of(m0, 1, gap_bar=gap[0], gap_minutes=gap[1]))
        want_te, _, _ = sim_oracle.population(ohlcv[3, :, a:b], bank[..., a:b], sweep.period_row, population,
                                              sim_oracle.config_of(market.minute0 + a, 1))
        for side, want in (("train", want_tr), ("test", want_te)):
            sim_oracle.assert_lanes({k: cv[f"{side}_{k}"][f] for k in ("n_records",) + CV_CLOSE}, want,
                                    f"fold {f} {side}", exact=("n_records",), close=CV_CLOSE)
