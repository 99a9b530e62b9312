"""Writes selection_reference.json: the reference StrategySelectionService's scalar scoring and switch methods
(services/strategy_selection_service.py) on a spread of metrics dicts, hours and risk profiles.

Run from a checkout of the reference project:  python tests/golden/make_selection.py <reference root>
The reference module is imported with stub modules for redis, binance, matplotlib, seaborn, services.model_integration
and services.market_regime_service; the service is built with object.__new__ plus its attributes, reads a dict-backed fake
Redis, and sees "now" at a chosen UTC hour.  Only the JSON output is kept."""
import asyncio
import json
import math
import os
import sys
import tempfile
import types
from datetime import datetime as _dt
from pathlib import Path

HOURS = (0, 7, 8, 13, 14, 21, 22, 23)
PROFILES = ("conservative", "moderate", "aggressive")


class FakeRedis:
    def __init__(self, data):
        self.data = data

    async def get(self, key):
        return self.data.get(key)


def metrics_cases():
    inf = float("inf")
    base = {"win_rate": 0.55, "profit_factor": 1.4, "sharpe_ratio": 1.1, "max_drawdown": 0.04, "recovery_factor": 1.7}
    hourly = {str(h): {"win_rate": 0.3 + 0.05 * (h % 9), "trade_count": 9 + (h % 2)} for h in range(24)}
    return [
        {},
        dict(base),
        dict(base, profit_factor=inf, recovery_factor=inf),
        dict(base, max_drawdown=0.0, recovery_factor=inf),
        dict(base, sharpe_ratio=-0.8, win_rate=0.2, max_drawdown=0.3, recovery_factor=-0.4),
        dict(base, sharpe_ratio=4.5, win_rate=1.0, profit_factor=7.0, max_drawdown=0.12, recovery_factor=5.0),
        dict(base, hourly_performance=hourly),
        dict(base, hourly_performance={str(h): {"win_rate": 0.9, "trade_count": 10} for h in range(24)}),
        dict(base, profit_factor=0.0, win_rate=0.0, sharpe_ratio=0.0, max_drawdown=0.0, recovery_factor=inf),
    ]


def main(ref_root):
    ref_root = Path(ref_root).resolve()
    for name in ("redis", "binance", "binance.client", "matplotlib", "matplotlib.pyplot", "seaborn",
                 "services.model_integration", "services.market_regime_service"):
        mod = types.ModuleType(name)
        sys.modules[name] = mod
    sys.modules["services.model_integration"].FeatureImportanceIntegrator = object
    sys.modules["services.market_regime_service"].MarketRegimeService = object
    sys.path.insert(0, str(ref_root))
    cwd = os.getcwd()
    tmp = tempfile.mkdtemp()
    os.chdir(tmp)
    os.makedirs("logs", exist_ok=True)
    try:
        import services.strategy_selection_service as sss
    finally:
        os.chdir(cwd)

    class FixedClock(_dt):
        hour = 0

        @classmethod
        def now(cls, tz=None):
            return _dt(2024, 3, 5, cls.hour, 17, 0)

    sss.datetime = FixedClock
    cases = metrics_cases()
    params = [{"atr_multiplier": 2.8}, {"atr_multiplier": 1.0}, {}, None]
    out = {"cases": cases, "params": params, "hours": list(HOURS), "profiles": list(PROFILES), "results": []}
    for profile in PROFILES:
        for hour in HOURS:
            FixedClock.hour = hour
            svc = object.__new__(sss.StrategySelectionService)
            store = {}
            for i, m in enumerate(cases):
                if m:
                    store[f"strategy_performance_{i}"] = json.dumps(m)
                p = params[i % len(params)]
                if p is not None:
                    store[f"worker_parameters_{i}"] = json.dumps(p)
            svc.redis = FakeRedis(store)
            svc.strategy_metrics_cache, svc.cache_expiry = {}, 3600
            svc.selection_weights = {"market_regime": 0.3, "historical_performance": 0.25, "risk_profile": 0.15,
                                     "social_sentiment": 0.15, "market_volatility": 0.1, "feature_importance": 0.05}
            svc.min_improvement_threshold, svc.min_confidence_threshold = 0.15, 0.7
            svc.time_windows = {"high_volatility": {"start": "14:00", "end": "22:00"},
                                "low_activity": {"start": "00:00", "end": "08:00"}}
            svc.risk_profiles = {
                "conservative": {"max_drawdown": 0.05, "min_sharpe": 1.5, "volatility_preference": "low"},
                "moderate": {"max_drawdown": 0.10, "min_sharpe": 1.2, "volatility_preference": "medium"},
                "aggressive": {"max_drawdown": 0.15, "min_sharpe": 1.0, "volatility_preference": "high"}}
            svc.current_risk_profile = profile
            svc.sentiment_thresholds = {"very_bearish": -0.6, "bearish": -0.2, "neutral": 0.2, "bullish": 0.6,
                                        "very_bullish": 0.8}
            strategies = [{"worker_id": str(i)} for i in range(len(cases))]

            async def run():
                r = {"risk": await svc.calculate_risk_scores(strategies),
                     "historical": await svc.calculate_historical_performance_scores(strategies),
                     "social": await svc.calculate_social_sentiment_scores(strategies),
                     "volatility": await svc.calculate_volatility_scores(strategies)}
                r["time"] = await svc.apply_time_based_adjustments({str(i): 0.05 * i + 0.3 for i in range(len(cases))})
                return r
            res = asyncio.run(run())
            out["results"].append({"profile": profile, "hour": hour, **res})
    # the switch rule
    FixedClock.hour = 0
    svc.redis = FakeRedis({"strategy_selection_a": json.dumps({"selection_score": 0.6})})
    switch = []
    for cur, new in ((None, ("a", 0.71)), (None, ("a", 0.7)), ("a", ("a", 0.99)), ("a", ("b", 0.76)), ("a", ("b", 0.75)),
                     ("a", ("b", 0.7500001)), ("c", ("b", 0.72))):
        ok = asyncio.run(svc.should_switch_strategy(cur, {"worker_id": new[0], "selection_score": new[1],
                                                          "selection_confidence": new[1]}))
        switch.append({"current": cur, "new": new[0], "score": new[1], "switch": ok})
    out["switch"] = switch
    path = Path(__file__).with_name("selection_reference.json")
    path.write_text(json.dumps(out, indent=1))
    print("wrote", path)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "../reference")
