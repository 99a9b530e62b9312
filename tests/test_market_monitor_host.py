"""CPU checks of the market monitor's restatement (tests/market_monitor_ref.py) against the reference's own outputs
(tests/golden/market_monitor_reference.json, made by tests/golden/make_market_monitor.py), and of the host's dict
assembly (ai_crypto_trader_b200/market_monitor.py)."""
import json
import math
from pathlib import Path

import numpy as np
import pytest

import market_monitor_ref as ref

FIXTURE = json.loads((Path(__file__).resolve().parent / "golden" / "market_monitor_reference.json").read_text())
TOL_ABS = ("bb_position", "stoch_k", "williams_r")       # denominators that are differences
# the dicts the fixture's combinations were computed on: the series' updates, then the crafted dicts (changes to base)
DICTS = [dict(s, current_price=1.0, avg_volume=1e6) for c in FIXTURE["series"] for s in c["snapshots"] if s] + \
    [{**{k: v for k, v in FIXTURE["base"].items() if k not in c["drop"]}, **c["set"]} for c in FIXTURE["crafted"]]


def fixture_bars(case) -> np.ndarray:
    """open / high / low / close [4][N] of a fixture series (open is the previous close)."""
    close = np.cumsum(case["close_steps"])
    open_ = np.concatenate([close[:1], close[:-1]])
    high = np.maximum(open_, close) + case["high_over"]
    low = np.minimum(open_, close) - case["low_under"]
    return np.stack([open_, high, low, close]).astype(np.float64) / FIXTURE["tick"]


def _same(a, b):
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))
    return a == b and type(a) is type(b) or (isinstance(a, (int, float)) and isinstance(b, (int, float)) and
                                             not isinstance(a, bool) and type(a) is type(b) and a == b)


def _leaves(result):
    if 'error' in result:
        return result
    return [None if v is None else list(v.values()) if isinstance(v, dict) else [v] for v in result.values()]


def _equal(got, want):
    if isinstance(want, dict) or want is None:
        return got == want
    if isinstance(want, list):
        return isinstance(got, list) and len(got) == len(want) and all(_equal(g, w) for g, w in zip(got, want))
    if isinstance(want, float):
        return isinstance(got, float) and _same(got, want)
    return type(got) is type(want) and got == want


def test_combinations_equal_the_reference_bit_for_bit():
    bad = []
    for k, (d, want) in enumerate(zip(DICTS, FIXTURE["combined"])):
        got = _leaves(ref.combinations(dict(d)))
        if not _equal(got, want):
            bad.append((k, d, got, want))
    assert not bad, bad[:3]


def test_fixture_covers_the_rounding_routes_and_the_none_entries():
    seen = set()
    for d in DICTS:
        raw = ref.combinations(dict(d), unrounded=True)
        if 'error' not in raw:
            seen |= {k for k, v in raw.items() if ref.roundings_disagree(v)}
    assert set(ref.combinations(DICTS[0], unrounded=True)) - seen == set(FIXTURE["no_midpoint"])
    flat = [c for c in FIXTURE["combined"] if isinstance(c, list)]
    assert any(c[2] is None for c in flat) and any(c[3] is None and c[11] is None for c in flat)
    assert sum(isinstance(c, dict) for c in FIXTURE["combined"]) >= 4           # missing required fields


def test_snapshot_matches_the_reference():
    near = 0
    for case in FIXTURE["series"]:
        bars = fixture_bars(case)
        ohlcv = np.zeros((5, 1, bars.shape[1]), dtype=np.float32)
        ohlcv[:4, 0] = bars
        ohlcv[4, 0] = 1.0
        for t, want in zip(case["picks"], case["snapshots"]):
            got = ref.row_at(ohlcv, case["minute0"], 0, t, case["W"])
            if want is None:
                assert got["valid"] == 0, (case["name"], t)
                continue
            assert got["valid"] == 1, (case["name"], t)
            for k, w in want.items():
                g = got[k]
                if k == "trend":
                    if g != w:
                        near += 1           # a deciding quantity within tolerance of its threshold
                        print(f"trend differs within tolerance: {case['name']} t={t} {g} vs {w}")
                    continue
                if isinstance(w, float) and math.isnan(w):
                    assert math.isnan(g), (case["name"], t, k)
                    continue
                tol = dict(rel=1e-12, abs=1e-9) if k in TOL_ABS else dict(rel=1e-12, abs=1e-300)
                assert g == pytest.approx(w, **tol), (case["name"], t, k, g, w)
    print(f"trend cases within tolerance of a threshold: {near}")
    assert near == 0


def test_market_update_dict_assembly():
    from ai_crypto_trader_b200 import _lib, market_monitor as mm
    row = np.zeros((), dtype=mm.ROW_DTYPE)
    d = dict(DICTS[0])
    for k in _lib.MM_SNAPSHOT_FIELDS:
        row[k] = d.get(k, 1.0)
    row["valid"], row["trend"] = 1, _lib.MM_TRENDS.index(d["trend"])

    class _M:
        symbols, minute0 = ["AUSDC"], 28_401_120

    class _H:
        market = _M()

    table = row[None, None]
    up = mm.market_update(_H(), 0, 0, table=table)
    assert list(up)[:4] == ["symbol", "current_price", "avg_volume", "timestamp"]
    assert list(up)[4:] == ['rsi', 'rsi_3m', 'rsi_5m', 'stoch_k', 'macd', 'macd_3m', 'macd_5m', 'williams_r',
                            'bb_position', 'trend', 'trend_strength', 'price_change_1m', 'price_change_3m',
                            'price_change_5m', 'price_change_15m', 'combined_indicators']
    assert up["timestamp"] == "2024-01-01T00:01:00+00:00" and up["trend"] == d["trend"]
    assert up["combined_indicators"] == {name: None for name in _lib.MM_COMBINATIONS}    # no combination computed
    table["valid"] = 0
    assert mm.market_update(_H(), 0, 0, table=table) is None


def test_snapshot_row_presence_and_errors():
    from ai_crypto_trader_b200 import _lib, market_monitor as mm
    d = dict(DICTS[0], ema_12=None, volume=3)
    row = mm.snapshot_row(d)
    assert row["present"] & _lib.MM_HAS["volume"] and not row["present"] & _lib.MM_HAS["ema_12"]
    assert row["volume"] == 3.0
    missing = {k: v for k, v in d.items() if k != "macd"}
    assert mm.calculate_indicator_combinations(missing) == {'error': "Missing required field: macd"}
    assert mm.LABEL_FIELDS[8] == "divergence_detector.divergence"
