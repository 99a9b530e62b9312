"""The market-regime oracle (tests/regime_ref.py) and the host side of ai_crypto_trader_b200.regime against the
reference's own results (tests/golden/regime_reference.json, written by tests/golden/make_regime.py), without a GPU."""
import json
import math
from pathlib import Path

import numpy as np
import pytest

import regime_ref

GOLD = json.loads((Path(__file__).parent / "golden" / "regime_reference.json").read_text())


def _unjson(v):
    if isinstance(v, str):
        return float(v)
    if isinstance(v, dict):
        return {k: _unjson(x) for k, x in v.items()}
    return v


def test_thresholds_are_the_reference_defaults(monkeypatch):
    from ai_crypto_trader_b200 import regime
    for k in ("BULL_TREND_STRENGTH", "BULL_PRICE_CHANGE", "BULL_VOLATILITY", "BEAR_TREND_STRENGTH", "BEAR_PRICE_CHANGE",
              "BEAR_VOLATILITY", "VOLATILE_THRESHOLD", "RANGING_TREND_STRENGTH", "RANGING_PRICE_RANGE"):
        monkeypatch.delenv(k, raising=False)
    assert regime.thresholds_from_env() == GOLD["thresholds"] == regime_ref.DEFAULT_THRESHOLDS
    monkeypatch.setenv("VOLATILE_THRESHOLD", "2.25")
    assert regime.thresholds_from_env()["volatile"]["volatility"] == 2.25
    assert regime.regime_params(60).volatile_volatility == 2.25


def test_rule_reproduces_every_fixture_window():
    branches = set()
    for w in GOLD["windows"]:
        got = regime_ref.detect(w["prices"], w["trends"], w["strengths"], GOLD["thresholds"])
        assert regime_ref.NAMES[got["label"]] == w["label"], w["name"]
        branches.add(got["branch"])
    assert branches == {"unknown", "volatile", "bull", "bear", "ranging", "default bull", "default bear",
                        "default ranging"}
    sizes = {len(w["prices"]) for w in GOLD["windows"]}
    assert {0, 1, 2, 3} <= sizes


def test_windows_and_per_regime_performance_reproduce_the_update():
    u = GOLD["update"]
    rows = regime_ref.windows(u["minutes"], u["prices"], u["trends"], u["strengths"], GOLD["thresholds"])
    assert any(r["n_points"] == 0 for r in rows)                         # the gap leaves a window empty
    want = GOLD["update"]["strategy_performance_history"]
    got = {}
    for sid in u["strategies"]:
        trades = u["trades"].get(sid)
        if not trades:
            continue
        perf = regime_ref.performance_by_regime(rows, [(t["minute"], t["profit"]) for t in trades])
        if perf:
            got[sid] = perf
    assert set(got) == set(want)
    for sid in want:
        assert set(got[sid]) == set(want[sid]), sid
        for regime, w in want[sid].items():
            g = got[sid][regime]
            assert g["trade_count"] == w["trade_count"]
            for k in ("win_rate", "profit_factor"):
                assert g[k] == pytest.approx(w[k], rel=1e-12, abs=0), (sid, regime, k)


def test_bar_labels_follow_the_windows():
    u = GOLD["update"]
    rows = regime_ref.windows(u["minutes"], u["prices"], u["trends"], u["strengths"])
    minute0 = u["minutes"][0] - 125
    lab = regime_ref.bar_labels(10_000, minute0, 1, rows)
    m = minute0 + np.arange(10_000)
    assert np.all(lab[m < u["minutes"][0]] == regime_ref.UNKNOWN)
    assert np.all(lab[m >= rows[-1]["start_minute"] + 1440] == regime_ref.UNKNOWN)
    for r in rows:
        inside = lab[(m >= r["start_minute"]) & (m < r["start_minute"] + 1440)]
        assert np.all(inside == r["label"])


def test_regime_score_is_bit_equal_to_the_reference():
    from ai_crypto_trader_b200.regime import MarketRegimeService
    for case in GOLD["scores"]:
        perf = _unjson(case["perf"])
        got = MarketRegimeService._calculate_regime_score(None, perf, case["regime"])
        want = case["score"]
        assert got == want and type(got) is type(want), (case, got)
    assert any(c["score"] == 1 for c in GOLD["scores"]) and any(c["score"] == 0 for c in GOLD["scores"])


def test_points_restate_the_monitor_trend():
    close = np.array([10.0, 11.0, 12.0, 9.0, 10.0, 10.5], dtype=np.float32)
    s20 = np.array([np.nan, 10.0, 11.0, 10.0, 10.0, 10.0], dtype=np.float32)
    s50 = np.array([np.nan, 9.0, 10.0, 11.0, 10.0, 10.0], dtype=np.float32)
    s5 = np.array([np.nan, np.nan, 10.0, 10.0, 10.0, 10.0], dtype=np.float32)
    idx, m, p, tr, st = regime_ref.points(close, s20, s50, s5, minute0=0, bar_minutes=5, sample_minutes=10)
    assert idx.tolist() == [3, 5]                      # bars ending a 10-minute bucket, from the first defined one
    assert m.tolist() == [15, 25]
    assert tr.tolist() == [regime_ref.DOWN, regime_ref.SIDEWAYS]
    s1 = (9.0 - 10.0) / 10.0 * 100
    assert st[0] == abs(s1 * 0.6 + s1 * 0.4)
    assert math.isclose(st[1], 5.0, rel_tol=1e-12)
