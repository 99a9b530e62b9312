"""The strategy selection service on the GPU engine: which candidate would the reference's selection rule have made live at
every check of a market's history, and how would the selected strategies have traded it.

Reference: services/strategy_selection_service.py.
  weights and thresholds from the environment          :56-128
  get_strategy_metrics (the per-candidate cache)       :159-264
  calculate_risk_scores                                 :299-369
  calculate_historical_performance_scores               :371-423
  calculate_social_sentiment_scores                     :425-485
  calculate_volatility_scores                           :487-575
  calculate_feature_importance_scores                   :577-687
  apply_time_based_adjustments                          :689-770
  select_optimal_strategy                               :772-882
  should_switch_strategy / switch_strategy              :884-1002
  update_risk_profile                                   :1004-1029
with _calculate_regime_score (market_regime_service.py:734-827, regime.MarketRegimeService).

replay() runs the service over the market: check c at the close of bar start_bar + c * check_bars, each candidate's
metrics snapshot refreshed on its own cache clock, every candidate scored (b200bt_selection_replay), the switch rule
applied in check order (b200bt_selection_switch), and the stitched run of the active candidates scored with
WalkForward.score.  The candidates' records are those of one population sweep over the whole series: a replay over the
history the candidates were evolved on is in-sample.

Supplied keys of a snapshot (the reference reads them from Redis keys nothing writes): params, regime_performance (per
scored regime of the regime label row) and hourly_performance (with a record's pnl as its profit).  Defaults: no
average_trade, avg_volatility, avg_trades_per_hour, volatility_performance or social_performance; no social metrics,
market conditions or feature-importance data.  The social, volatility and feature-importance factors are therefore
constants (0.5, 0.5 / 0.6, 0.5).
"""
from __future__ import annotations

import ctypes as C
import logging
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .population import iso_minute
from .regime import REGIMES, MarketRegimeService
from .sweep import BOOK_CAP_HEADROOM, MarketData
from .walk_forward import STAT_FIELDS, WalkForward

logger = logging.getLogger("b200bt.strategy_selection")

FACTORS = ("market_regime", "historical_performance", "risk_profile", "social_sentiment", "market_volatility",
           "feature_importance")
WEIGHT_ENV = (("market_regime", "WEIGHT_MARKET_REGIME", "0.30"), ("historical_performance", "WEIGHT_HISTORICAL_PERF", "0.25"),
              ("risk_profile", "WEIGHT_RISK_PROFILE", "0.15"), ("social_sentiment", "WEIGHT_SOCIAL_SENTIMENT", "0.15"),
              ("market_volatility", "WEIGHT_MARKET_VOLATILITY", "0.10"),
              ("feature_importance", "WEIGHT_FEATURE_IMPORTANCE", "0.05"))
RISK_PROFILES = {
    "conservative": {"max_drawdown": 0.05, "min_sharpe": 1.5, "volatility_preference": "low"},
    "moderate": {"max_drawdown": 0.10, "min_sharpe": 1.2, "volatility_preference": "medium"},
    "aggressive": {"max_drawdown": 0.15, "min_sharpe": 1.0, "volatility_preference": "high"},
}
VOLATILITY_PREFERENCES = ("low", "medium", "high")          # B200BT_SEL_P_RISK_VOLATILITY = index
TIME_WINDOWS = {"high_volatility": {"start": "14:00", "end": "22:00"}, "low_activity": {"start": "00:00", "end": "08:00"}}
CACHE_EXPIRY = 3600
SENTIMENT_THRESHOLDS = {"very_bearish": -0.6, "bearish": -0.2, "neutral": 0.2, "bullish": 0.6, "very_bullish": 0.8}
ROW_DTYPE = np.dtype([(n, "<f8") for n in _lib.SEL_ROW])
SWITCH_REASON = "Automated strategy selection"


def selection_weights_from_env() -> Dict[str, float]:
    """The WEIGHT_* environment weights, normalised to sum 1 (:71-83)."""
    w = {k: float(os.getenv(env, default)) for k, env, default in WEIGHT_ENV}
    total = sum(w.values())
    for k in w:
        w[k] /= total
    return w


def check_bars(check_interval_s: float, bar_minutes: int) -> int:
    """Bars between checks: STRATEGY_CHECK_INTERVAL seconds over the bar's seconds, which must be a positive integer."""
    q = float(check_interval_s) / 60.0 / bar_minutes
    if not (q >= 1 and q == int(q)):
        raise ValueError(f"STRATEGY_CHECK_INTERVAL = {check_interval_s} s is not a positive whole number of "
                         f"{bar_minutes}-minute bars")
    return int(q)


def n_checks(N: int, start_bar: int, every: int) -> int:
    """Checks at bars start_bar + c * every <= N - 1."""
    if not 0 <= start_bar < N:
        raise ValueError(f"start_bar {start_bar} outside [0, {N})")
    return (N - 1 - start_bar) // every + 1


def switch_schedule(switch_bars: Sequence[int], actives: Sequence[int], N: int) -> List[Tuple[int, int, int]]:
    """The stitched run: the candidate made active at bar t trades bars t + 1 up to and including the bar of the next
    switch, the last one to N - 1; nothing trades before the first switch.  [(start, end, candidate)], empty segments
    (a switch at the last bar) left out."""
    out = []
    for i, (t, k) in enumerate(zip(switch_bars, actives)):
        end = switch_bars[i + 1] + 1 if i + 1 < len(switch_bars) else N
        if t + 1 < end:
            out.append((int(t) + 1, int(end), int(k)))
    return out


def gene_table(candidates: Sequence[Dict]) -> np.ndarray:
    """float64 [K][B200BT_SEL_GENES]: the genes the scores read, NaN where a candidate lacks the key."""
    return np.array([[float(p[g]) if p.get(g) is not None else math.nan for g in _lib.SEL_GENES] for p in candidates],
                    dtype=np.float64).reshape(len(candidates), len(_lib.SEL_GENES))


class StrategySelectionService:
    """The reference's selection service over a fixed list of candidate parameter dicts (index = strategy id) trading
    every symbol of `market`.  The scalar scoring methods take metrics dicts the caller puts in `strategy_metrics`
    ({strategy id: dict}), parameters in `worker_parameters`, and the hour of "now" in `current_hour`; replay() computes
    every snapshot itself."""

    def __init__(self, market: MarketData, candidates: Sequence[Dict], config: Optional[Dict] = None):
        self.config = config or {}
        self.market = market
        self.candidates = [dict(p) for p in candidates]
        self.check_interval = int(os.getenv("STRATEGY_CHECK_INTERVAL", "300"))
        self.selection_weights = selection_weights_from_env()
        self.min_improvement_threshold = float(os.getenv("MIN_STRATEGY_IMPROVEMENT", "0.15"))
        self.min_confidence_threshold = float(os.getenv("MIN_STRATEGY_CONFIDENCE", "0.7"))
        self.time_windows = {k: dict(v) for k, v in TIME_WINDOWS.items()}
        self.risk_profiles = {k: dict(v) for k, v in RISK_PROFILES.items()}
        self.current_risk_profile = os.getenv("RISK_PROFILE", "moderate")
        self.sentiment_thresholds = dict(SENTIMENT_THRESHOLDS)
        self.cache_expiry = CACHE_EXPIRY
        self.active_strategy_id = None
        self.strategy_history: List[Dict] = []
        self.strategy_selection: Dict = {}        # strategy_selection_{id}: the selection dict of each switch
        self.strategy_metrics: Dict = {}
        self.worker_parameters: Dict = {i: p for i, p in enumerate(self.candidates)}
        self.current_hour = 0
        self.market_regime_service = MarketRegimeService(market, self.config)
        self.sweep = self.market_regime_service.sweep
        self._event_cap = 0                       # learnt from the previous replay (0: count first)

    # -- the reference's scalar methods -------------------------------------------------------------------------------
    async def get_strategy_metrics(self, strategy_id) -> Dict:
        return self.strategy_metrics.get(strategy_id) or {}

    async def calculate_risk_scores(self, strategies: List[Dict]) -> Dict:
        try:
            risk_scores = {}
            risk_profile = self.risk_profiles[self.current_risk_profile]
            for strategy in strategies:
                strategy_id = strategy["worker_id"]
                metrics = await self.get_strategy_metrics(strategy_id)
                if not metrics:
                    risk_scores[strategy_id] = 0.0
                    continue
                max_drawdown = metrics.get("max_drawdown", 1.0)
                sharpe_ratio = metrics.get("sharpe_ratio", 0.0)
                recovery_factor = metrics.get("recovery_factor", 0.0)
                avg_vol = metrics.get("avg_volatility", 0.5)
                dd_score = 1.0 - (max_drawdown / risk_profile["max_drawdown"]) if max_drawdown > 0 else 1.0
                volatility_score = 0.5
                vol_pref = risk_profile["volatility_preference"]
                if vol_pref == "low":
                    volatility_score = 1.0 - min(avg_vol, 1.0)
                elif vol_pref == "medium":
                    volatility_score = 1.0 - abs(avg_vol - 0.5)
                elif vol_pref == "high":
                    volatility_score = min(avg_vol, 1.0)
                sharpe_score = min(sharpe_ratio / risk_profile["min_sharpe"], 1.0)
                recovery_score = min(recovery_factor, 2.0) / 2.0
                combined_score = dd_score * 0.3 + sharpe_score * 0.3 + recovery_score * 0.2 + volatility_score * 0.2
                risk_scores[strategy_id] = max(0.0, min(1.0, combined_score))
            return risk_scores
        except Exception as e:
            logger.error("Error calculating risk scores: %s", e)
            return {strategy["worker_id"]: 0.0 for strategy in strategies}

    async def calculate_historical_performance_scores(self, strategies: List[Dict]) -> Dict:
        try:
            performance_scores = {}
            for strategy in strategies:
                strategy_id = strategy["worker_id"]
                metrics = await self.get_strategy_metrics(strategy_id)
                if not metrics:
                    performance_scores[strategy_id] = 0.0
                    continue
                win_rate = metrics.get("win_rate", 0.0)
                profit_factor = metrics.get("profit_factor", 0.0)
                sharpe_ratio = metrics.get("sharpe_ratio", 0.0)
                avg_trade = metrics.get("average_trade", 0.0)
                win_rate_score = min(win_rate, 1.0)
                pf_score = min(profit_factor / 3.0, 1.0)
                sharpe_score = min(sharpe_ratio / 3.0, 1.0)
                avg_trade_score = 0.5
                if avg_trade > 0:
                    avg_trade_score = min(0.5 + (avg_trade / 0.02), 1.0)
                elif avg_trade < 0:
                    avg_trade_score = max(0.0, 0.5 + (avg_trade / 0.02))
                performance_scores[strategy_id] = (win_rate_score * 0.25 + pf_score * 0.25 + sharpe_score * 0.3 +
                                                   avg_trade_score * 0.2)
            return performance_scores
        except Exception as e:
            logger.error("Error calculating performance scores: %s", e)
            return {strategy["worker_id"]: 0.0 for strategy in strategies}

    async def calculate_social_sentiment_scores(self, strategies: List[Dict]) -> Dict:
        """No social metrics reach a replay (:439-441): every candidate scores 0.5."""
        return {strategy["worker_id"]: 0.5 for strategy in strategies}

    async def calculate_volatility_scores(self, strategies: List[Dict]) -> Dict:
        """No market conditions reach a replay: the category is "medium" (:502-513), so a candidate without metrics
        scores 0.5 and one with metrics but no volatility_performance 0.6 (:521-566)."""
        try:
            volatility_scores = {}
            for strategy in strategies:
                strategy_id = strategy["worker_id"]
                metrics = await self.get_strategy_metrics(strategy_id)
                if not metrics:
                    volatility_scores[strategy_id] = 0.5
                    continue
                volatility_performance = metrics.get("volatility_performance", {})
                if "medium" in volatility_performance:
                    category_perf = volatility_performance["medium"]
                    volatility_scores[strategy_id] = (category_perf.get("win_rate", 0.5) * 0.6 +
                                                      min(category_perf.get("profit_factor", 1.0) / 2.0, 1.0) * 0.4)
                else:
                    volatility_scores[strategy_id] = 0.6
            return volatility_scores
        except Exception as e:
            logger.error("Error calculating volatility scores: %s", e)
            return {strategy["worker_id"]: 0.5 for strategy in strategies}

    async def calculate_feature_importance_scores(self, strategies: List[Dict]) -> Dict:
        """No feature-importance data reaches a replay (:593-595): every candidate scores 0.5."""
        return {strategy["worker_id"]: 0.5 for strategy in strategies}

    async def apply_time_based_adjustments(self, scores: Dict) -> Dict:
        """The hour of "now" is current_hour (a replay's check bar, UTC)."""
        try:
            adjusted_scores = scores.copy()
            current_hour = self.current_hour
            in_high_volatility = in_low_activity = False
            for window_name, window in self.time_windows.items():
                start_hour = int(window["start"].split(":")[0])
                end_hour = int(window["end"].split(":")[0])
                if start_hour <= current_hour < end_hour:
                    if window_name == "high_volatility":
                        in_high_volatility = True
                    elif window_name == "low_activity":
                        in_low_activity = True
            for strategy_id in adjusted_scores:
                metrics = await self.get_strategy_metrics(strategy_id)
                if "hourly_performance" in metrics:
                    hourly_perf = metrics["hourly_performance"].get(str(current_hour), {})
                    if hourly_perf:
                        win_rate = hourly_perf.get("win_rate", 0.5)
                        if hourly_perf.get("trade_count", 0) >= 10:
                            adjusted_scores[strategy_id] += (win_rate - 0.5) * 2 * 0.1
                if in_high_volatility:
                    volatility_handling = 0.0
                    params = self.worker_parameters.get(strategy_id)
                    if params is not None:
                        volatility_handling = min(params.get("atr_multiplier", 1.0) / 2.0, 1.0)
                    adjusted_scores[strategy_id] += volatility_handling * 0.05
                if in_low_activity:
                    frequency_score = max(0, 1.0 - (metrics.get("avg_trades_per_hour", 10.0) / 20.0))
                    adjusted_scores[strategy_id] += frequency_score * 0.05
            for strategy_id in adjusted_scores:
                adjusted_scores[strategy_id] = max(0.0, min(1.0, adjusted_scores[strategy_id]))
            return adjusted_scores
        except Exception as e:
            logger.error("Error applying time-based adjustments: %s", e)
            return scores

    async def should_switch_strategy(self, current_strategy_id, new_strategy: Dict) -> bool:
        """The rule of :896-927; the current strategy's score is its score at its own switch (strategy_selection_{id})."""
        try:
            if current_strategy_id is None or current_strategy_id != new_strategy["worker_id"]:
                new_score = new_strategy.get("selection_score", 0.0)
                new_confidence = new_strategy.get("selection_confidence", 0.0)
                current_score = 0.0
                if current_strategy_id is not None and current_strategy_id in self.strategy_selection:
                    current_score = self.strategy_selection[current_strategy_id].get("selection_score", 0.0)
                improvement = new_score - current_score
                return improvement > self.min_improvement_threshold and new_confidence > self.min_confidence_threshold
            return False
        except Exception as e:
            logger.error("Error in should_switch_strategy: %s", e)
            return False

    async def switch_strategy(self, new_strategy: Dict) -> bool:
        """switch_strategy (:946-998) without Redis: the active id, the selection dict and the switch record.  The record's
        previous_strategy_id is the new id, as in the reference, which assigns the active id before it records."""
        strategy_id = new_strategy["worker_id"]
        self.active_strategy_id = strategy_id
        self.strategy_selection[strategy_id] = new_strategy
        self.strategy_history.append({
            "timestamp": new_strategy.get("selection_time"), "previous_strategy_id": self.active_strategy_id,
            "new_strategy_id": strategy_id, "selection_score": new_strategy.get("selection_score", 0.0),
            "factor_scores": new_strategy.get("factor_scores", {}),
            "market_regime": new_strategy.get("market_regime", "unknown"), "reason": SWITCH_REASON})
        return True

    async def update_risk_profile(self, profile: str) -> bool:
        if profile not in self.risk_profiles:
            logger.error("Invalid risk profile: %s", profile)
            return False
        self.current_risk_profile = profile
        return True

    # -- the replay ---------------------------------------------------------------------------------------------------
    def params_array(self, start_bar: int, every: int):
        """The B200BT_SEL_P_* slots of this service's settings."""
        prof = self.risk_profiles[self.current_risk_profile]
        hours = [int(self.time_windows[w][e].split(":")[0]) for w in ("high_volatility", "low_activity")
                 for e in ("start", "end")]
        vals = [start_bar, every, self.cache_expiry, *[self.selection_weights[f] for f in FACTORS],
                self.min_improvement_threshold, self.min_confidence_threshold, prof["max_drawdown"], prof["min_sharpe"],
                VOLATILITY_PREFERENCES.index(prof["volatility_preference"]), *hours]
        return (C.c_double * len(vals))(*[float(v) for v in vals])

    def _replay_rows(self, start_bar: int, count: Optional[int], with_scores: bool):
        """(rows [C][ROW_WORDS], scores [C][K] or None, switch checks) on the device."""
        m, sw = self.market, self.sweep
        every = check_bars(self.check_interval, m.bar_minutes)
        total = n_checks(m.N, start_bar, every)
        Cn = total if count is None else min(int(count), total)
        K = len(self.candidates)
        dev = m.device
        labels = self.market_regime_service.labels()[:1].contiguous()
        params = self.params_array(start_bar, every)
        genes = torch.from_numpy(gene_table(self.candidates)).to(dev)
        rows = torch.empty((Cn, len(_lib.SEL_ROW)), dtype=torch.float64, device=dev)
        locks = torch.empty(Cn, dtype=torch.int32, device=dev)
        scores = torch.empty((Cn, K), dtype=torch.float64, device=dev) if with_scores else None
        packed, unique, expand = sw._unique(self.candidates)
        row_of = np.arange(K) if expand is None else np.asarray(expand)
        calls = [0]

        def launch(indiv: torch.Tensor, lo: int, hi: int, cap: int) -> None:
            sel = np.nonzero((row_of >= lo) & (row_of < hi))[0]
            idx = torch.from_numpy(sel.astype(np.int32)).to(dev)
            row = torch.from_numpy((row_of[sel] - lo).astype(np.int32)).to(dev)
            g = genes[torch.from_numpy(sel).to(dev)].contiguous()
            _lib.call("b200bt_selection_replay", m.close.data_ptr(), _lib.ld(m.close), m.S, m.N, indiv.data_ptr(), hi - lo,
                      C.byref(sw.cfg), sw._stats.data_ptr(), sw._events.data_ptr(), cap, labels.data_ptr(), 0,
                      row.data_ptr(), idx.data_ptr(), g.data_ptr(), len(sel), K, params, Cn, int(calls[0] > 0),
                      rows.data_ptr(), _lib.ptr(scores), locks.data_ptr(), _lib.current_stream())
            calls[0] += 1

        sw._record_pass(packed, unique, expand, self._event_cap, launch)
        busiest = sw._exact_cap(sw._stats)
        self._event_cap = busiest + busiest // BOOK_CAP_HEADROOM + 2
        self.last_batches = calls[0]
        switches = torch.empty(Cn, dtype=torch.int32, device=dev)
        n_sw = torch.empty(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.call("b200bt_selection_switch", rows.data_ptr(), Cn, params, switches.data_ptr(), n_sw.data_ptr(),
                      _lib.current_stream())
        return rows, scores, switches[:int(n_sw.item())]

    def _selection(self, row) -> Dict:
        k = int(row["best"])
        return {"worker_id": k, "parameters": dict(self.candidates[k]), "selection_score": float(row["score"]),
                "selection_confidence": float(row["score"]), "market_regime": REGIMES[int(row["regime"])],
                "selection_time": iso_minute(self.market.minute0 + int(row["bar"]) * self.market.bar_minutes),
                "factor_scores": {f: float(row[f]) for f in FACTORS}}

    async def select_optimal_strategy(self, bar: int) -> Optional[Dict]:
        """The reference's selection at the close of `bar`, by a service that starts there (every candidate fetches its
        snapshot of the records with bar <= `bar`): the best candidate's dict with worker_id, parameters,
        selection_score, selection_confidence, market_regime, selection_time and factor_scores; None when no candidate
        is valid.  Errors: logged, None returned."""
        try:
            rows, _, _ = self._replay_rows(int(bar), 1, False)
            row = rows.cpu().numpy().view(ROW_DTYPE)[0, 0]
            if row["best"] < 0:
                logger.warning("No strategy scores available")
                return None
            return self._selection(row)
        except Exception as e:
            logger.error("Error selecting optimal strategy: %s", e)
            return None

    def replay(self, start_bar: int = 0, rows: bool = True, scores: bool = False) -> Optional[Dict]:
        """The service over bars [start_bar, N) (see the module docstring):
          checks         structured rows (ROW_DTYPE: bar, regime, best, score, the six factor scores, active,
                         active_score) when `rows`
          scores         float64 [C][K] of every candidate's final score when `scores` (small replays only)
          switches       the switch records (switch_strategy :974-982, quirk included) with their check and bar
          active_share   float64 [K]: the fraction of checks each candidate was active
          stitched       {field: [S]} lane stats of the stitched run (None without a switch), stitched_mean the means
          candidates     {field: [K][S]} each candidate's own lane stats over [start_bar, N), candidates_mean [K] means
        Errors: logged, None returned."""
        try:
            m = self.market
            dev_rows, dev_scores, dev_sw = self._replay_rows(int(start_bar), None, scores)
            table = dev_rows.cpu().numpy().view(ROW_DTYPE)[:, 0]
            sw_checks = dev_sw.cpu().numpy().tolist()
            K = len(self.candidates)
            act = table["active"].astype(np.int64)
            share = np.bincount(act[act >= 0], minlength=K)[:K] / len(table)
            switches = []
            for c in sw_checks:
                sel = self._selection(table[c])
                switches.append({"timestamp": sel["selection_time"], "previous_strategy_id": sel["worker_id"],
                                 "new_strategy_id": sel["worker_id"], "selection_score": sel["selection_score"],
                                 "factor_scores": sel["factor_scores"], "market_regime": sel["market_regime"],
                                 "reason": SWITCH_REASON, "check": int(c), "bar": int(table[c]["bar"])})
            sched = switch_schedule([s["bar"] for s in switches], [s["new_strategy_id"] for s in switches], m.N)
            schedules = ([sched] if sched else []) + [[(int(start_bar), m.N, k)] for k in range(K)]
            st = WalkForward(self.sweep, {}).score(schedules, self.candidates)
            off = 1 if sched else 0
            stitched = {f: st[f][0] for f in st} if sched else None
            cand = {f: st[f][off:] for f in st}
            return {
                "checks": table.copy() if rows else None,
                "scores": dev_scores.cpu().numpy() if scores else None,
                "switches": switches,
                "active_share": share,
                "schedule": sched,
                "stitched": stitched,
                "stitched_mean": {f: float(np.mean(stitched[f])) for f in STAT_FIELDS} if sched else None,
                "candidates": cand,
                "candidates_mean": {f: np.mean(cand[f], axis=1) for f in STAT_FIELDS},
            }
        except Exception as e:
            logger.error("Error replaying strategy selection: %s", e)
            return None
