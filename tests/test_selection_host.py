"""Host side of the strategy selection replay (ai_crypto_trader_b200/strategy_selection.py), no GPU: the scalar scoring and
switch methods against the reference service's own output (tests/golden/selection_reference.json, made by
tests/golden/make_selection.py), environment parsing and weight normalisation, the check clock and per-candidate refresh
plan, the switch scan and its records, and the stitched schedule."""
import json
from pathlib import Path

import numpy as np
import pytest

from selection_ref import drive, host_service

GOLDEN = json.loads((Path(__file__).parent / "golden" / "selection_reference.json").read_text())


def _svc(profile, hour):
    cases, params = GOLDEN["cases"], GOLDEN["params"]
    svc = host_service({"current_risk_profile": profile, "current_hour": hour})
    svc.strategy_metrics = {str(i): m for i, m in enumerate(cases)}
    svc.worker_parameters = {str(i): params[i % len(params)] for i in range(len(cases)) if params[i % len(params)] is not None}
    return svc


@pytest.mark.parametrize("entry", GOLDEN["results"], ids=lambda e: f"{e['profile']}-{e['hour']:02d}h")
def test_scalar_methods_match_the_reference(entry):
    svc = _svc(entry["profile"], entry["hour"])
    strategies = [{"worker_id": str(i)} for i in range(len(GOLDEN["cases"]))]
    assert drive(svc.calculate_risk_scores(strategies)) == entry["risk"]
    assert drive(svc.calculate_historical_performance_scores(strategies)) == entry["historical"]
    assert drive(svc.calculate_social_sentiment_scores(strategies)) == entry["social"]
    assert drive(svc.calculate_volatility_scores(strategies)) == entry["volatility"]
    base = {str(i): 0.05 * i + 0.3 for i in range(len(GOLDEN["cases"]))}
    assert drive(svc.apply_time_based_adjustments(base)) == entry["time"]
    assert drive(svc.calculate_feature_importance_scores(strategies)) == {s["worker_id"]: 0.5 for s in strategies}


def test_should_switch_matches_the_reference():
    svc = host_service()
    svc.strategy_selection = {"a": {"selection_score": 0.6}}
    for case in GOLDEN["switch"]:
        new = {"worker_id": case["new"], "selection_score": case["score"], "selection_confidence": case["score"]}
        assert drive(svc.should_switch_strategy(case["current"], new)) == case["switch"], case


def test_update_risk_profile():
    svc = host_service()
    assert drive(svc.update_risk_profile("aggressive")) and svc.current_risk_profile == "aggressive"
    assert not drive(svc.update_risk_profile("reckless")) and svc.current_risk_profile == "aggressive"


def test_weights_from_the_environment(monkeypatch):
    from ai_crypto_trader_b200.strategy_selection import WEIGHT_ENV, selection_weights_from_env
    for _, env, _ in WEIGHT_ENV:
        monkeypatch.delenv(env, raising=False)
    total = 0.30 + 0.25 + 0.15 + 0.15 + 0.10 + 0.05          # :81, summed in the dict's order
    assert selection_weights_from_env() == {
        "market_regime": 0.30 / total, "historical_performance": 0.25 / total, "risk_profile": 0.15 / total,
        "social_sentiment": 0.15 / total, "market_volatility": 0.10 / total, "feature_importance": 0.05 / total}
    monkeypatch.setenv("WEIGHT_MARKET_REGIME", "1.0")
    monkeypatch.setenv("WEIGHT_FEATURE_IMPORTANCE", "0.3")
    w = selection_weights_from_env()
    total = 1.0 + 0.25 + 0.15 + 0.15 + 0.10 + 0.3
    assert w["market_regime"] == 1.0 / total and w["feature_importance"] == 0.3 / total
    assert w["historical_performance"] == 0.25 / total


def test_check_clock():
    from ai_crypto_trader_b200.strategy_selection import check_bars, n_checks
    assert check_bars(300, 1) == 5 and check_bars(300, 5) == 1 and check_bars(60, 1) == 1
    for bad in ((300, 7), (30, 1), (0, 1), (-300, 1)):
        with pytest.raises(ValueError):
            check_bars(*bad)
    assert n_checks(10, 0, 5) == 2 and n_checks(10, 9, 5) == 1 and n_checks(11, 0, 5) == 3
    for start in (-1, 10):
        with pytest.raises(ValueError):
            n_checks(10, start, 5)


def test_refresh_plan_per_candidate():
    """The oracle's refresh plan (the GPU replay is held to the oracle built on it)."""
    from selection_ref import refresh_checks
    bars = list(range(0, 200, 5))
    minute = lambda t: 1000 + t
    # no record before bar 22: the empty fetches are not cached, the first snapshot is at the first check after it
    assert refresh_checks(bars, 22, minute, 3600)[0] == 5
    # then every 60 minutes of the clock: 12 checks of 5 bars
    assert refresh_checks(bars, 0, minute, 3600) == [0, 12, 24, 36]
    assert refresh_checks(bars, 0, minute, 300) == list(range(len(bars)))      # expiry = the check interval
    assert refresh_checks(bars, 0, minute, 301) == list(range(0, len(bars), 2))
    assert refresh_checks(bars, None, minute, 3600) == []                     # a candidate without records
    assert refresh_checks(bars, 195, minute, 3600) == [39]


def test_switch_run_and_schedule():
    from ai_crypto_trader_b200.strategy_selection import switch_schedule
    from selection_ref import switch_run
    best = [-1, 2, 2, 1, 1, 0, 3, 3]
    score = [np.nan, 0.69, 0.71, 0.85, 0.87, 0.9, 0.95, 0.99]
    svc = host_service()
    sw, active, active_score = switch_run(svc, best, score)
    assert sw == [2, 4]
    assert active.tolist() == [-1, -1, 2, 2, 1, 1, 1, 1]
    assert active_score.tolist() == [0, 0, 0.71, 0.71, 0.87, 0.87, 0.87, 0.87]
    assert [h["new_strategy_id"] for h in svc.strategy_history] == [2, 1]
    assert all(h["previous_strategy_id"] == h["new_strategy_id"] for h in svc.strategy_history)   # the reference's quirk
    assert switch_schedule([10, 40], [2, 3], 100) == [(11, 41, 2), (41, 100, 3)]
    assert switch_schedule([10, 99], [2, 3], 100) == [(11, 100, 2)]         # a switch at the last bar trades nothing
    assert switch_schedule([], [], 100) == []
    # the segments are what WalkForward.score takes: contiguous, start < end, ending at N
    from ai_crypto_trader_b200.walk_forward import segment_tables
    seg, begin = segment_tables([switch_schedule([10, 40], [2, 3], 100)])
    assert seg["start"].tolist() == [11, 41] and seg["end"].tolist() == [41, 100] and begin.tolist() == [0, 2]


def test_gene_table():
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.strategy_selection import gene_table
    g = gene_table([{"ema_long": 20, "atr_period": 7}, {}])
    assert g.shape == (2, len(_lib.SEL_GENES))
    assert g[0, _lib.SEL_GENES.index("ema_long")] == 20 and g[0, _lib.SEL_GENES.index("atr_period")] == 7
    assert np.isnan(g[1]).all() and np.isnan(g[0, _lib.SEL_GENES.index("take_profit")])
