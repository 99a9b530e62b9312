"""Market regimes on the GPU engine: regime labels of a market's bars, trade metrics of a population per regime, and
regime-based strategy selection.

Reference: services/market_regime_service.py.
  regime_thresholds                       :100-118
  detect_regime_from_data                 :503-603  (b200bt_regime_labels, one window at a time)
  select_strategy_for_regime              :637-732
  _calculate_regime_score                 :734-827
  update_strategy_performance_by_regime   :829-993  (windows :844-889; the per-regime backtest its TODO at :909-911
                                                     leaves out is b200bt_class_stats on the sweep's records)
The reference classifies monitor snapshots; here one point per `sample_minutes` bucket of the market's own bars carries
the monitor's trend fields (indicators.multi_timeframe_indicators at that bar).  The ML detectors, the live rolling
detection and Redis are out of scope.

Mirrored quirks (kept, not fixed): max_drawdown is calculate_metrics' fraction while the score divides it by 100
(:753), so the drawdown term is nearly constant; the clamp to [0, 1] makes many strategies tie at 1.0, and the stable
descending sort then picks the first of them.
"""
from __future__ import annotations

import ctypes as C
import logging
import os
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib
from .sweep import DEFAULT_GOALS, MarketData, PopulationSweep

logger = logging.getLogger("b200bt.regime")

REGIMES = _lib.REGIMES
SCORED_REGIMES = REGIMES[:4]


def thresholds_from_env() -> Dict:
    """regime_thresholds of the reference (:100-118): the same environment variables and defaults."""
    return {
        "bull": {"trend_strength": float(os.getenv("BULL_TREND_STRENGTH", "0.6")),
                 "price_change": float(os.getenv("BULL_PRICE_CHANGE", "5.0")),
                 "volatility": float(os.getenv("BULL_VOLATILITY", "0.5"))},
        "bear": {"trend_strength": float(os.getenv("BEAR_TREND_STRENGTH", "0.6")),
                 "price_change": float(os.getenv("BEAR_PRICE_CHANGE", "-5.0")),
                 "volatility": float(os.getenv("BEAR_VOLATILITY", "0.5"))},
        "volatile": {"volatility": float(os.getenv("VOLATILE_THRESHOLD", "1.5"))},
        "ranging": {"trend_strength": float(os.getenv("RANGING_TREND_STRENGTH", "0.3")),
                    "price_range": float(os.getenv("RANGING_PRICE_RANGE", "3.0"))},
    }


def regime_params(sample_minutes: int = 60, thresholds: Optional[Dict] = None) -> _lib.RegimeParams:
    """b200bt_regime_params of a thresholds dict in the reference's nested form (default: thresholds_from_env()).  The
    bull / bear `volatility` entries are not read by the rule (:571-597) and have no field."""
    t = thresholds or thresholds_from_env()
    return _lib.RegimeParams(sample_minutes=int(sample_minutes), reserved=0,
                             volatile_volatility=float(t["volatile"]["volatility"]),
                             bull_price_change=float(t["bull"]["price_change"]),
                             bull_trend_strength=float(t["bull"]["trend_strength"]),
                             bear_price_change=float(t["bear"]["price_change"]),
                             bear_trend_strength=float(t["bear"]["trend_strength"]),
                             ranging_price_range=float(t["ranging"]["price_range"]),
                             ranging_trend_strength=float(t["ranging"]["trend_strength"]))


def trend_rows(market: MarketData) -> torch.Tensor:
    """float32 [4][S][N] on the device: close, SMA20, SMA50 (base clock) and the SMA20 of the 5-minute closes at the last
    completed 5-minute bar (b200bt_sma_bank, b200bt_resample, b200bt_align; NaN where undefined)."""
    from . import indicators as ind
    if 5 % market.bar_minutes:
        raise ValueError(f"regime labels need 5-minute bars derived from the market's clock (bar_minutes = "
                         f"{market.bar_minutes} does not divide 5)")
    sma = ind.sma_bank(market.close, [20, 50], fill=False)
    m5 = ind.resample(market, 5)
    sma5 = ind.align_to_base(ind.sma_bank(m5.close, [20], fill=False)[:, 0].contiguous(), market, 5)
    return torch.stack([market.close, sma[:, 0], sma[:, 1], sma5])


def label_rows(labels: torch.Tensor, S: int, N: int, what: str = "regime labels") -> Tuple[torch.Tensor, int]:
    """Per-bar labels as the kernels read them: (labels, ld_labels) from a device uint8 tensor [S or 1][N].  One row shared by
    every symbol ([1][N], or a row expanded to [S][N]) comes back as a contiguous [1][N] with ld_labels = 0, per-symbol
    rows as a contiguous [S][N] with ld_labels = N.  `what` names the argument in the ValueError of any other tensor."""
    if not (isinstance(labels, torch.Tensor) and labels.is_cuda and labels.dtype == torch.uint8 and labels.dim() == 2
            and labels.shape[0] in (1, S) and labels.shape[1] == N):
        raise ValueError(f"{what} must be a device uint8 tensor [{S} or 1][{N}]")
    if labels.shape[0] == 1 or labels.stride(0) == 0:
        return labels[:1].contiguous(), 0
    return labels.contiguous(), N


def regime_labels(market: MarketData, sample_minutes: int = 60, thresholds: Optional[Dict] = None,
                  primary: Optional[Union[int, str]] = None) -> Tuple[torch.Tensor, List[np.ndarray]]:
    """(labels uint8 [S][N] on the device, windows): the regime (an index into REGIMES) of every bar, and per symbol the
    rows of its 24-hour windows (a structured array of _lib.REGIME_WINDOW_DTYPE; n_points = 0 marks a skipped window).
    `primary` (a symbol index or name): that symbol's labels for every symbol (an expanded view), as the reference
    watches one PRIMARY_TRADING_SYMBOL.  sample_minutes: minutes per point, a multiple of 5 and of the bar clock; 60 by
    default, as the rule scales volatility by sqrt(24) "to a 24-hour scale" (:543)."""
    rows = trend_rows(market)
    if primary is not None:
        p = market.symbols.index(primary) if isinstance(primary, str) else int(primary)
        rows = rows[:, p:p + 1].contiguous()
    S, N = rows.shape[1], rows.shape[2]
    lib = _lib.load()
    K = int(lib.b200bt_regime_max_windows(N, market.bar_minutes))
    labels = torch.empty((S, N), dtype=torch.uint8, device=market.device)
    win = torch.empty((S, K, 8), dtype=torch.float64, device=market.device)          # 64-byte rows
    params = regime_params(sample_minutes, thresholds)
    plane = S * N
    base = rows.data_ptr()
    with torch.cuda.device(market.device):
        _lib.call("b200bt_regime_labels", base, base + 4 * plane, base + 8 * plane, base + 12 * plane, S, N, N,
                  market.minute0, market.bar_minutes, C.byref(params), labels.data_ptr(), N, win.data_ptr(), K,
                  _lib.current_stream())
    table = win.cpu().numpy().view(np.dtype(_lib.REGIME_WINDOW_DTYPE)).reshape(S, K)
    windows = [table[s][table[s]["start_minute"] >= 0] for s in range(S)]
    if primary is not None:
        return labels.expand(market.S, N), windows * market.S
    return labels, windows


class MarketRegimeService:
    """The regime service of the reference on the GPU engine: labels the market once, backtests a population per regime
    (PopulationSweep.class_stats) and selects the best strategy for a regime with the reference's score."""

    def __init__(self, market: MarketData, config: Optional[Dict] = None, thresholds: Optional[Dict] = None,
                 sample_minutes: int = 60):
        self.config = config or {}
        self.market = market
        self.current_regime = None
        self.regime_history: List = []
        self.strategy_performance_history: Dict = {}
        self.regime_strategy_mapping: Dict = {}
        self.regime_thresholds = thresholds or thresholds_from_env()
        self.primary_symbol = os.getenv("PRIMARY_TRADING_SYMBOL", "BTCUSDC")
        self.sample_minutes = int(sample_minutes)
        goals = self.config.get("evolution", {}).get("optimization_goals") or DEFAULT_GOALS
        self.sweep = PopulationSweep(market, optimization_goals=goals)
        self._labels = None
        self.windows = None

    def labels(self) -> torch.Tensor:
        """The market's bar labels (computed on first use): the primary symbol's labels for every symbol when
        PRIMARY_TRADING_SYMBOL is one of the market's symbols, else each symbol's own."""
        if self._labels is None:
            primary = self.primary_symbol if self.primary_symbol in self.market.symbols else None
            self._labels, self.windows = regime_labels(self.market, self.sample_minutes, self.regime_thresholds, primary)
        return self._labels

    def regime_performance(self, population: List[Dict]) -> List[Dict]:
        """One dict per individual in the shape _calculate_regime_score reads.  Overall sharpe_ratio, win_rate,
        max_drawdown and profit_factor are the means over symbols of the lane stats (the default fitness rule).
        regime_performance[regime] pools the individual's records on every symbol whose bar carries that regime:
        trade_count = sum of n_records, win_rate = sum of n_wins / trade_count, profit_factor = the net sum / |sum of
        the losses|, or 1 without losses (:947-954); sharpe_ratio and max_drawdown are the means over symbols of the
        class stats.  Regimes without records are left out, as the reference leaves them out."""
        _, classes = self.sweep.class_stats(population, self.labels(), len(SCORED_REGIMES))
        lanes = self.sweep.lane_stats()
        out = []
        for i, params in enumerate(population):
            perf = {"strategy_id": i, "params": params,
                    "sharpe_ratio": float(np.mean(lanes["sharpe_ratio"][i])),
                    "win_rate": float(np.mean(lanes["win_rate"][i])),
                    "max_drawdown": float(np.mean(lanes["max_drawdown"][i])),
                    "profit_factor": float(np.mean(lanes["profit_factor"][i])),
                    "regime_performance": {}}
            for r, name in enumerate(SCORED_REGIMES):
                st = classes[r]
                n = float(np.sum(st["n_records"][i]))
                if n <= 0:
                    continue
                loss = float(np.sum(st["total_loss"][i]))
                perf["regime_performance"][name] = {
                    "trade_count": int(n),
                    "win_rate": float(np.sum(st["n_wins"][i])) / n,
                    "profit_factor": float(np.sum(st["net_profit"][i])) / abs(loss) if loss != 0 else 1,
                    "sharpe_ratio": float(np.mean(st["sharpe_ratio"][i])),
                    "max_drawdown": float(np.mean(st["max_drawdown"][i])),
                }
            out.append(perf)
        return out

    def regime_scores(self, population: List[Dict]) -> np.ndarray:
        """_calculate_regime_score of every individual for bull, bear, ranging, volatile: float64 [pop][4]."""
        perf = self.regime_performance(population)
        return np.array([[self._calculate_regime_score(p, r) for r in SCORED_REGIMES] for p in perf], dtype=np.float64)

    async def select_strategy_for_regime(self, regime: str, population: List[Dict]) -> Optional[Dict]:
        """The individual of `population` with the highest regime score (a stable descending sort: the first of a tie
        wins); regime_strategy_mapping[regime] becomes its index.  Every call scores the population it is given.
        Errors: logged, None returned (the reference's convention)."""
        try:
            if not population:
                logger.warning("No available strategies found")
                return None
            perf = self.regime_performance(population)
            scored = sorted(({"strategy_id": p["strategy_id"], "score": self._calculate_regime_score(p, regime)}
                             for p in perf), key=lambda x: x["score"], reverse=True)
            best = scored[0]["strategy_id"]
            self.regime_strategy_mapping[regime] = best
            logger.info("Selected strategy %d for %s regime with score %.4f", best, regime, scored[0]["score"])
            return population[best]
        except Exception as e:
            logger.error("Error selecting strategy for regime %s: %s", regime, e)
            return None

    def _calculate_regime_score(self, perf_data: Dict, regime: str) -> float:
        """The reference's expression (:734-827) verbatim."""
        try:
            sharpe_ratio = perf_data.get('sharpe_ratio', 0)
            win_rate = perf_data.get('win_rate', 0)
            max_drawdown = perf_data.get('max_drawdown', 100)
            profit_factor = perf_data.get('profit_factor', 0)
            norm_drawdown = 1 - (max_drawdown / 100)
            base_score = (
                sharpe_ratio * 0.3 +
                win_rate * 0.2 +
                norm_drawdown * 0.2 +
                profit_factor * 0.3
            ) / 1.0
            regime_perf = perf_data.get('regime_performance', {}).get(regime, {})
            if regime_perf:
                regime_sharpe = regime_perf.get('sharpe_ratio', sharpe_ratio)
                regime_win_rate = regime_perf.get('win_rate', win_rate)
                regime_drawdown = regime_perf.get('max_drawdown', max_drawdown)
                regime_profit_factor = regime_perf.get('profit_factor', profit_factor)
                regime_norm_drawdown = 1 - (regime_drawdown / 100)
                regime_score = (
                    regime_sharpe * 0.3 +
                    regime_win_rate * 0.2 +
                    regime_norm_drawdown * 0.2 +
                    regime_profit_factor * 0.3
                ) / 1.0
                final_score = (base_score * 0.3) + (regime_score * 0.7)
            else:
                final_score = base_score
            strategy_params = perf_data.get('params', {})
            if regime == 'bull':
                if strategy_params.get('ema_long', 0) < 30:
                    final_score *= 1.1
                if strategy_params.get('take_profit', 0) > 5:
                    final_score *= 1.05
            elif regime == 'bear':
                if strategy_params.get('stop_loss', 100) < 3:
                    final_score *= 1.1
                if strategy_params.get('rsi_oversold', 0) > 30:
                    final_score *= 1.05
            elif regime == 'ranging':
                if strategy_params.get('bollinger_std', 0) > 2.0:
                    final_score *= 1.1
                if strategy_params.get('rsi_period', 0) < 14:
                    final_score *= 1.05
            elif regime == 'volatile':
                if strategy_params.get('atr_multiplier', 0) > 2.0:
                    final_score *= 1.1
                if strategy_params.get('atr_period', 0) < 10:
                    final_score *= 1.05
            return max(0, min(1, final_score))
        except Exception as e:
            logger.error("Error calculating regime score: %s", e)
            return 0.0
