"""Run the REFERENCE's own code as the oracle of record (where a copy of the reference tree exists).

TEST INFRASTRUCTURE.  The reference tree is a checkout named `reference` beside this
repository, or the tree B200BT_REFERENCE_ROOT names; this
module is imported only by tests/golden/make_golden.py, which writes the
committed fixtures.  No test, smoke() or bench.py imports it.

The reference's numeric code runs UNMODIFIED; only modules it imports for
plotting / networking (matplotlib, seaborn, redis, binance) are replaced by
empty stubs, as verified in SURVEY.md section 8c.  The reference opens
`logs/*.log` and `config.json` relative to the cwd at import time
(services/genetic_algorithm.py:22, services/strategy_evaluation.py:23,513), so
we chdir into a scratch directory holding a copy of its config.json.
"""
from __future__ import annotations

import os
import shutil
import sys
import tempfile
import types
from pathlib import Path

REFERENCE_ROOT = Path(os.environ.get("B200BT_REFERENCE_ROOT", Path(__file__).resolve().parents[2] / "reference"))


def available() -> bool:
    return (REFERENCE_ROOT / "services" / "strategy_evaluation.py").exists()


_scratch = None


def _prepare():
    global _scratch
    if _scratch is not None:
        return _scratch
    if not available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    sys.dont_write_bytecode = True
    for name in ["matplotlib", "matplotlib.pyplot", "seaborn", "redis", "redis.asyncio", "redis.exceptions",
                 "binance", "binance.client"]:
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["matplotlib"].use = lambda *a, **k: None
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["redis.asyncio"].Redis = object
    sys.modules["redis.exceptions"].ConnectionError = Exception
    sys.modules["binance.client"].Client = object
    _scratch = Path(tempfile.mkdtemp(prefix="b200bt_ref_"))
    (_scratch / "logs").mkdir()
    shutil.copy(REFERENCE_ROOT / "config.json", _scratch / "config.json")
    os.chdir(_scratch)
    if str(REFERENCE_ROOT) not in sys.path:
        sys.path.insert(0, str(REFERENCE_ROOT))
    return _scratch


def strategy_evaluation():
    """(StrategyEvaluationSystem instance, StrategyPerformanceMetrics class) of the reference."""
    _prepare()
    import logging
    from services.strategy_evaluation import StrategyEvaluationSystem, StrategyPerformanceMetrics
    logging.getLogger("strategy_evaluation").setLevel(logging.ERROR)
    return StrategyEvaluationSystem("config.json"), StrategyPerformanceMetrics


def genetic_algorithm_class():
    _prepare()
    import logging
    from services.genetic_algorithm import GeneticAlgorithm
    logging.getLogger("genetic_algorithm").setLevel(logging.ERROR)
    return GeneticAlgorithm


def portfolio_risk_service():
    """A PortfolioRiskService built without __init__ (Redis / Binance clients, portfolio_risk_service.py:47-110);
    only the pure numeric methods (:217-396) are used."""
    _prepare()
    import logging
    from services.portfolio_risk_service import PortfolioRiskService
    logging.getLogger().setLevel(logging.ERROR)
    svc = object.__new__(PortfolioRiskService)
    svc.historical_data = {}
    svc.asset_correlations = {}
    svc.risk_config = {}
    return svc


def monte_carlo_service(mc_params: dict):
    """A MonteCarloService built without __init__ (which needs Binance keys and
    rewrites config.json, monte_carlo_service.py:47-108)."""
    _prepare()
    import logging
    from services.monte_carlo_service import MonteCarloService
    logging.getLogger().setLevel(logging.ERROR)
    svc = object.__new__(MonteCarloService)
    svc.mc_params = dict(mc_params)
    svc.historical_data = {}
    svc.simulation_results = {}
    svc.last_simulation_time = {}
    return svc


def optimization_goals() -> dict:
    import json
    return json.loads((REFERENCE_ROOT / "config.json").read_text())["evolution"]["optimization_goals"]


# ---------------------------------------------------------------------------------
# BASELINE configs[0]: the reference's own StrategyTester bar loop
# ---------------------------------------------------------------------------------
def _install_ta_shim():
    """`ta` (third-party, not installed, unpinned) -> thin classes over oracle.indicators_ref,
    exposing exactly the constructors / methods binance_ml_strategy.py:5-8,67-179 uses."""
    from oracle import indicators_ref as R

    class SMAIndicator:
        def __init__(self, close, window): self.c, self.w = close, window
        def sma_indicator(self): return R.sma(self.c, self.w)

    class EMAIndicator:
        def __init__(self, close, window): self.c, self.w = close, window
        def ema_indicator(self): return R.ema(self.c, self.w)

    class MACD:
        def __init__(self, close, window_slow=26, window_fast=12, window_sign=9):
            self.l, self.s, self.d = R.macd(close, window_fast, window_slow, window_sign)
        def macd(self): return self.l
        def macd_signal(self): return self.s
        def macd_diff(self): return self.d

    class IchimokuIndicator:
        def __init__(self, high, low, window1=9, window2=26, window3=52): self.a, self.b = R.ichimoku(high, low, window1, window2, window3)
        def ichimoku_a(self): return self.a
        def ichimoku_b(self): return self.b

    class RSIIndicator:
        def __init__(self, close, window=14): self.c, self.w = close, window
        def rsi(self): return R.rsi(self.c, self.w)

    class StochasticOscillator:
        def __init__(self, high, low, close, window=14, smooth_window=3): self.k, self.d = R.stochastic(high, low, close, window, smooth_window)
        def stoch(self): return self.k
        def stoch_signal(self): return self.d

    class WilliamsRIndicator:
        def __init__(self, high, low, close, lbp=14): self.v = R.williams_r(high, low, close, lbp)
        def williams_r(self): return self.v

    class BollingerBands:
        def __init__(self, close, window=20, window_dev=2): self.h, self.m, self.l = R.bollinger(close, window, window_dev)
        def bollinger_hband(self): return self.h
        def bollinger_mavg(self): return self.m
        def bollinger_lband(self): return self.l

    class AverageTrueRange:
        def __init__(self, high, low, close, window=14): self.v = R.atr(high, low, close, window)
        def average_true_range(self): return self.v

    class VolumeWeightedAveragePrice:
        def __init__(self, high, low, close, volume, window=14): self.v = R.vwap(high, low, close, volume, window)
        def volume_weighted_average_price(self): return self.v

    mods = {"ta": {}, "ta.trend": dict(SMAIndicator=SMAIndicator, EMAIndicator=EMAIndicator, MACD=MACD, IchimokuIndicator=IchimokuIndicator),
            "ta.momentum": dict(RSIIndicator=RSIIndicator, StochasticOscillator=StochasticOscillator, WilliamsRIndicator=WilliamsRIndicator),
            "ta.volatility": dict(BollingerBands=BollingerBands, AverageTrueRange=AverageTrueRange),
            "ta.volume": dict(VolumeWeightedAveragePrice=VolumeWeightedAveragePrice)}
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m


class _Anything:
    """Stub object for plotting modules: every attribute / call returns itself."""
    def __getattr__(self, name): return self
    def __call__(self, *a, **k): return self


def strategy_tester():
    """The reference's StrategyTester, its numeric code unmodified, with
      * `ta` replaced by the oracle restatement (the package is not installed / not pinned),
      * TechnicalAnalyzer._handle_nan_values re-expressed for pandas 3 (`fillna(method=)` was removed),
      * the two OpenAI calls of AITrader replaced by the deterministic stub documented in
        DESIGN.md: analyze_trade_opportunity -> the technical signal with confidence 1.0,
        analyze_risk_setup -> None (no AI risk opinion, so the tester keeps the technical sizing,
        strategy_tester.py:259-265)."""
    _prepare()
    _install_ta_shim()
    os.environ.setdefault("OPENAI_API_KEY", "not-a-key")
    for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.dates", "seaborn"):
        m = sys.modules.get(name) or types.ModuleType(name)
        m.__getattr__ = lambda attr, _m=m: _Anything()
        sys.modules[name] = m
    import logging
    logging.getLogger().setLevel(logging.ERROR)
    import binance_ml_strategy as bms
    from backtesting.strategy_tester import StrategyTester

    def _handle_nan_values(self):
        import numpy as np
        cols = self.data.select_dtypes(include=[np.number]).columns
        self.data[cols] = self.data[cols].ffill().bfill().fillna(0)
    bms.TechnicalAnalyzer._handle_nan_values = _handle_nan_values

    tester = StrategyTester("config.json")

    async def analyze_trade_opportunity(market_data):
        sig = bms.TradingSignal(symbol=market_data["symbol"], price=market_data["current_price"], rsi=market_data["rsi"],
                                stoch_k=market_data["stoch_k"], macd=market_data["macd"], volume=market_data["avg_volume"],
                                volatility=market_data["volatility"], williams_r=market_data["williams_r"],
                                trend=market_data["trend"], trend_strength=market_data["trend_strength"],
                                bb_position=market_data["bb_position"])
        return {"decision": sig.signal, "confidence": 1.0, "reasoning": "deterministic stub"}

    async def analyze_risk_setup(risk_setup):
        return None
    tester.ai_trader.analyze_trade_opportunity = analyze_trade_opportunity
    tester.ai_trader.analyze_risk_setup = analyze_risk_setup
    return tester, bms


def run_reference_backtest(df, symbol="SYNUSDC", initial_balance=10000.0):
    """Execute StrategyTester.backtest_strategy on an in-memory OHLCV DataFrame (timestamp index)."""
    import asyncio
    tester, bms = strategy_tester()
    tester.data_manager.merge_market_and_social_data = lambda *a, **k: df
    start, end = df.index[0].to_pydatetime(), df.index[-1].to_pydatetime()
    stats = asyncio.run(tester.backtest_strategy(symbol, "1m", start, end, initial_balance))
    return stats, tester, bms
