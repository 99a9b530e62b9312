"""Generate the market-regime fixture by EXECUTING the reference's own code.

Run where a copy of the reference tree exists (as for make_golden.py):

    python tests/golden/make_regime.py

Writes tests/golden/regime_reference.json.  The reference module services/market_regime_service.py is imported with
the packages it imports but these functions do not use replaced by empty stubs (sklearn, hmmlearn, dotenv, redis,
matplotlib and the two services.utils.market_regime_* modules), and three of its functions run unmodified:
    detect_regime_from_data                 :503-603  on windows of points that reach every branch, 0-3 points, values
                                                      exactly at the thresholds, equal trend fractions, and random windows
    update_strategy_performance_by_regime   :829-993  end to end under asyncio.run, on a stub serving synthetic points
                                                      and trade records (gaps that leave windows empty, trades before the
                                                      first point and after the last window, a strategy without trades)
    _calculate_regime_score                 :734-827  every regime, with and without regime_performance, parameters on
                                                      both sides of each adjustment, and scores that clamp
Points are {timestamp, current_price, trend, trend_strength, price_change_24h}; timestamps are ISO strings of whole
minutes (the fixture stores the minutes).
"""
from __future__ import annotations

import asyncio
import json
import sys
import types
from datetime import datetime, timedelta, timezone
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
OUT = Path(__file__).resolve().parent / "regime_reference.json"
TRENDS = ("uptrend", "downtrend", "sideways")
MINUTE0 = 28_401_120          # 2024-01-01 00:00 UTC in minutes


def _load():
    from oracle import ref_runner
    ref_runner._prepare()
    names = ["sklearn", "sklearn.cluster", "sklearn.preprocessing", "sklearn.decomposition", "sklearn.ensemble",
             "sklearn.pipeline", "sklearn.model_selection", "hmmlearn", "hmmlearn.hmm", "dotenv",
             "services.utils.market_regime_detector", "services.utils.market_regime_data_collector"]
    for name in names:
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    for name in ("KMeans", "StandardScaler", "PCA", "RandomForestClassifier", "Pipeline", "train_test_split"):
        for mod in names[1:7]:
            setattr(sys.modules[mod], name, object)
    sys.modules["dotenv"].load_dotenv = lambda *a, **k: None
    sys.modules["services.utils.market_regime_detector"].MarketRegimeDetector = object
    sys.modules["services.utils.market_regime_data_collector"].MarketRegimeDataCollector = object
    import importlib
    return importlib.import_module("services.market_regime_service").MarketRegimeService


def iso(minute: int) -> str:
    return (datetime(1970, 1, 1, tzinfo=timezone.utc) + timedelta(minutes=int(minute))).strftime("%Y-%m-%dT%H:%M:%S")


def points(minutes, prices, trends, strengths):
    return [{"timestamp": iso(m), "current_price": float(p), "trend": TRENDS[t], "trend_strength": float(s),
             "price_change_24h": 0.0} for m, p, t, s in zip(minutes, prices, trends, strengths)]


def window_cases(rng):
    U, D, F = 0, 1, 2
    hourly = lambda n: [MINUTE0 + 60 * i for i in range(n)]
    rise = lambda n, r: [100.0 * (1 + r) ** i for i in range(n)]
    cases = [
        ("empty", [], [], []),
        ("one point", [100.0], [U], [0.5]),
        ("two points, bull", [100.0, 110.0], [U, U], [2.0, 2.0]),
        ("two points, ranging", [100.0, 100.5], [F, F], [0.1, 0.1]),
        ("three points, volatile", [100.0, 200.0, 90.0], [U, D, F], [5.0, 5.0, 5.0]),
        ("three points, bear", [100.0, 97.0, 94.0], [D, D, D], [1.0, 1.0, 1.0]),
        ("bull", rise(24, 0.003), [U] * 20 + [F] * 4, [1.2] * 24),
        ("bear", rise(24, -0.003), [D] * 20 + [F] * 4, [1.2] * 24),
        ("ranging", [100.0 + 0.1 * ((-1) ** i) for i in range(24)], [F] * 24, [0.1] * 24),
        ("default bull", rise(24, 0.0005), [U] * 14 + [D] * 5 + [F] * 5, [0.8] * 24),
        ("default bear", rise(24, -0.0005), [D] * 14 + [U] * 5 + [F] * 5, [0.8] * 24),
        ("default ranging", rise(24, 0.0005), [F] * 14 + [U] * 5 + [D] * 5, [0.8] * 24),
        ("change exactly +5", [100.0, 102.0, 105.0], [U, U, U], [1.0] * 3),
        ("change exactly -5", [100.0, 98.0, 95.0], [D, D, D], [1.0] * 3),
        ("up fraction exactly 0.6", [100.0, 102.0, 104.0, 105.0, 106.0], [U, U, U, F, F], [1.0] * 5),
        ("down fraction exactly 0.6", [100.0, 98.0, 96.0, 95.0, 94.0], [D, D, D, F, F], [1.0] * 5),
        ("|change| exactly 3", [100.0, 101.0, 103.0], [F, F, F], [0.1] * 3),
        ("strength exactly 0.3", [100.0, 100.5, 101.0], [F, F, F], [0.3] * 3),
        ("equal fractions", [100.0, 100.2, 100.1, 100.3, 100.2, 100.4], [U, U, D, D, F, F], [0.5] * 6),
        ("up = down > sideways", [100.0, 100.2, 100.1, 100.3, 100.2], [U, U, D, D, F], [0.5] * 5),
    ]
    out = [(name, hourly(len(p)), p, t, s) for name, p, t, s in cases]
    for k in range(60):
        n = int(rng.integers(0, 30))
        vol = float(rng.choice([0.001, 0.01, 0.05, 0.4]))
        drift = float(rng.choice([-0.004, -0.001, 0.0, 0.001, 0.004]))
        p = 100.0 * np.cumprod(1 + drift + vol * rng.standard_normal(n))
        t = rng.integers(0, 3, n).tolist()
        s = np.round(rng.uniform(0, 2, n), 3).tolist()
        out.append((f"random {k}", hourly(n), p.tolist(), t, s))
    return out


def update_case(rng):
    """Six days of hourly points with day 3 missing (an empty window), segments that trend up, down, flat and wild."""
    minutes, prices, trends, strengths = [], [], [], []
    p = 100.0
    for h in range(6 * 24):
        if 72 <= h < 96:
            continue
        day = h // 24
        drift, vol, tr, st = [(0.003, 0.001, 0, 1.5), (-0.003, 0.001, 1, 1.5), (0.0, 0.0005, 2, 0.1),
                              (0.0, 0.0, 2, 0.1), (0.0, 0.2, 2, 3.0), (0.0005, 0.001, 0, 0.8)][day]
        p *= 1 + drift + vol * rng.standard_normal()
        minutes.append(MINUTE0 + 37 + 60 * h)      # points off the hour: t0 is not midnight
        prices.append(float(p))
        trends.append(tr if rng.random() < 0.8 else int(rng.integers(0, 3)))
        strengths.append(float(st))
    first, last = minutes[0], minutes[-1]
    trades = {}
    for sid, n, lo, hi in (("s0", 300, first - 600, last + 3000), ("s1", 40, first + 1440, first + 2 * 1440)):
        tm = np.sort(rng.integers(lo, hi, n))
        profit = np.round(rng.normal(0.0, 5.0, n), 6)
        profit[::7] = 0.0                               # zero profit counts as a loss (:945) but not in total_loss
        trades[sid] = [{"timestamp": iso(m), "profit": float(x)} for m, x in zip(tm, profit)]
    trades["s0"].append({"timestamp": iso(first), "profit": 1.0})      # exactly on a window start
    return minutes, prices, trends, strengths, trades


def score_cases():
    base = {"sharpe_ratio": 0.8, "win_rate": 0.55, "max_drawdown": 0.2, "profit_factor": 1.3}
    rp = {"sharpe_ratio": 1.1, "win_rate": 0.6, "max_drawdown": 0.1, "profit_factor": 1.6, "trade_count": 12}
    params = [{}, {"ema_long": 20, "take_profit": 6, "stop_loss": 2, "rsi_oversold": 35, "bollinger_std": 2.5,
                   "rsi_period": 10, "atr_multiplier": 2.5, "atr_period": 7},
              {"ema_long": 30, "take_profit": 5, "stop_loss": 3, "rsi_oversold": 30, "bollinger_std": 2.0,
               "rsi_period": 14, "atr_multiplier": 2.0, "atr_period": 10}]
    out = []
    for regime in ("bull", "bear", "ranging", "volatile", "unknown"):
        for par in params:
            out.append({**base, "params": par})
            out.append({**base, "params": par, "regime_performance": {regime: dict(rp)}})
            out.append({"sharpe_ratio": 0.1, "win_rate": 0.3, "max_drawdown": 0.5, "profit_factor": 0.4, "params": par,
                        "regime_performance": {regime: {"win_rate": 0.2, "profit_factor": 0.3, "trade_count": 3}}})
    out += [{"sharpe_ratio": 5.0, "win_rate": 0.7, "max_drawdown": 0.1, "profit_factor": float("inf")},
            {"sharpe_ratio": -9.0, "win_rate": 0.1, "max_drawdown": 0.9, "profit_factor": 0.0},
            {}, {"regime_performance": {"bull": {"sharpe_ratio": 3.0}}}]
    return out


def _num(x):
    return x if np.isfinite(x) else repr(float(x))


def main():
    MRS = _load()
    inst = MRS()
    thresholds = inst.regime_thresholds
    rng = np.random.default_rng(2024)
    stub = types.SimpleNamespace(regime_thresholds=thresholds)
    windows = []
    for name, m, p, t, s in window_cases(rng):
        label = MRS.detect_regime_from_data(stub, points(m, p, t, s))
        windows.append({"name": name, "minutes": m, "prices": p, "trends": t, "strengths": s, "label": label})

    minutes, prices, trends, strengths, trades = update_case(rng)
    data = points(minutes, prices, trends, strengths)
    store = {f"strategy_trades_{k}": json.dumps(v) for k, v in trades.items()}

    class Redis:
        async def get(self, key):
            return store.get(key)

        async def set(self, key, value):
            store[key] = value

    async def historical(lookback_hours=168):
        return data

    async def strategies():
        return [{"worker_id": "s0"}, {"worker_id": "s1"}, {"worker_id": "s2"}]

    up = types.SimpleNamespace(regime_thresholds=thresholds, lookback_periods=inst.lookback_periods, redis=Redis(),
                               strategy_performance_history={}, get_historical_market_data=historical,
                               get_available_strategies=strategies)
    up.detect_regime_from_data = types.MethodType(MRS.detect_regime_from_data, up)
    asyncio.run(MRS.update_strategy_performance_by_regime(up))
    assert json.loads(store["strategy_regime_performance"]) == up.strategy_performance_history

    scores = []
    for perf in score_cases():
        for regime in ("bull", "bear", "ranging", "volatile", "unknown"):
            scores.append({"perf": {k: _num(v) if isinstance(v, float) else v for k, v in perf.items()},
                           "regime": regime, "score": MRS._calculate_regime_score(stub, perf, regime)})

    OUT.write_text(json.dumps({
        "thresholds": thresholds, "windows": windows,
        "update": {"minutes": minutes, "prices": prices, "trends": trends, "strengths": strengths,
                   "trades": {k: [{"minute": int((datetime.fromisoformat(t["timestamp"]).replace(tzinfo=timezone.utc)
                                                   - datetime(1970, 1, 1, tzinfo=timezone.utc)).total_seconds() // 60),
                                    "profit": t["profit"]} for t in v] for k, v in trades.items()},
                   "strategies": ["s0", "s1", "s2"],
                   "strategy_performance_history": up.strategy_performance_history},
        "scores": scores}, indent=1))
    print(f"wrote {OUT}: {len(windows)} windows, {len(scores)} scores, "
          f"labels {sorted(set(w['label'] for w in windows))}")


if __name__ == "__main__":
    main()
