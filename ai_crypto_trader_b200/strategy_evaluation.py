"""StrategyEvaluationSystem / StrategyPerformanceMetrics call surface on the GPU engine.

Reference: services/strategy_evaluation.py.
  StrategyEvaluationSystem._simulate_trades(strategy_id, parameters, market_data)   :746-878
  StrategyPerformanceMetrics.calculate_metrics(trades, initial_capital)             :32-228
  StrategyEvaluationSystem._calculate_strategy_score(metrics)                       :579-633

`_simulate_trades` keeps the reference's signature and returns the reference's trade
records (one dict per entry and per exit, keys timestamp/symbol/side/price/quantity/
fees/pnl); the bar-by-bar state machine runs in the sweep kernel (one lane), the host
only formats the O(#trades) records.  `evaluate_population` is the batched form the GA
uses.  Market data contract: price and rsi are fp32 (values are rounded to fp32 on
upload; DESIGN.md "Data contract").
"""
from __future__ import annotations

import json
import logging
from datetime import datetime
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib
from .sweep import DEFAULT_GOALS, MarketData, PopulationSweep
from .synth import bar_timestamp

logger = logging.getLogger("b200bt.strategy_evaluation")


class StrategyPerformanceMetrics:
    """Host-side metrics over an arbitrary list of trade records (e.g. live trades handed in
    by a caller).  The GA path never calls this: there the same quantities are reduced inside
    the sweep kernel.  Restates calculate_metrics (:32-228) for the scalar fields."""

    @staticmethod
    def calculate_metrics(trades: List[Dict], initial_capital: float = 10000.0) -> Dict:
        base = {"total_trades": 0, "win_rate": 0.0, "profit_factor": 0.0, "sharpe_ratio": 0.0, "max_drawdown": 0.0,
                "average_profit": 0.0, "average_loss": 0.0, "largest_profit": 0.0, "largest_loss": 0.0,
                "total_profit": 0.0, "total_loss": 0.0, "net_profit": 0.0, "return_pct": 0.0,
                "avg_trade_duration": 0, "risk_reward_ratio": 0.0, "profitable_symbols": {},
                "unprofitable_symbols": {}, "monthly_returns": {}, "daily_returns": {}}
        if not trades:
            return base
        recs = sorted(trades, key=lambda t: t.get("timestamp", ""))
        pnl = [t.get("pnl", 0) for t in recs]
        if len(recs) < 2:
            p = pnl[0]
            base.update(total_trades=1, win_rate=1.0 if p > 0 else 0.0, net_profit=p,
                        return_pct=(p / initial_capital) * 100)
            for key, cond in (("average_profit", p > 0), ("largest_profit", p > 0), ("total_profit", p > 0),
                              ("average_loss", p < 0), ("largest_loss", p < 0), ("total_loss", p < 0)):
                base[key] = p if cond else 0.0
            return base
        wins = [p for p in pnl if p > 0]
        losses = [p for p in pnl if p < 0]
        tp, tl = sum(wins), sum(losses)
        equity, peak, dds = [initial_capital], initial_capital, []
        daily, monthly, by_symbol = {}, {}, {}
        for t, p in zip(recs, pnl):
            cur = equity[-1] + p
            equity.append(cur)
            if cur > peak:
                peak = cur
            else:
                dds.append((peak - cur) / peak)
            ts = t.get("timestamp", "")
            if ts:
                try:
                    d = datetime.fromisoformat(ts.replace("Z", "+00:00"))
                    for key, bucket in ((d.strftime("%Y-%m-%d"), daily), (d.strftime("%Y-%m"), monthly)):
                        bucket[key] = bucket[key] + p if key in bucket else p
                except ValueError:
                    pass
            sym = t.get("symbol", "UNKNOWN")
            by_symbol[sym] = by_symbol.get(sym, 0) + p
        durs = []
        for i in range(0, len(recs) - 1, 2):
            try:
                a = datetime.fromisoformat(recs[i].get("timestamp", "").replace("Z", "+00:00"))
                b = datetime.fromisoformat(recs[i + 1].get("timestamp", "").replace("Z", "+00:00"))
                durs.append((b - a).total_seconds() / 60)
            except ValueError:
                pass
        vals = list(daily.values())
        sharpe = 0
        if len(vals) > 1:
            sd = np.std(vals)
            sharpe = (np.mean(vals) / sd) * np.sqrt(252) if sd > 0 else 0
        avg_p = tp / len(wins) if wins else 0
        avg_l = tl / len(losses) if losses else 0
        net = tp + tl
        return {
            "total_trades": len(recs), "win_rate": len(wins) / len(recs),
            "profit_factor": abs(tp / tl) if tl != 0 else float("inf"), "sharpe_ratio": sharpe,
            "max_drawdown": max(dds) if dds else 0, "average_profit": avg_p, "average_loss": avg_l,
            "largest_profit": max(wins) if wins else 0, "largest_loss": min(losses) if losses else 0,
            "total_profit": tp, "total_loss": tl, "net_profit": net, "return_pct": (net / initial_capital) * 100,
            "avg_trade_duration": sum(durs) / len(durs) if durs else 0,
            "risk_reward_ratio": abs(avg_p / avg_l) if avg_l != 0 else float("inf"),
            "profitable_symbols": {s: v for s, v in by_symbol.items() if v > 0},
            "unprofitable_symbols": {s: v for s, v in by_symbol.items() if v <= 0},
            "monthly_returns": monthly, "daily_returns": daily, "equity_curve": equity,
        }


    @staticmethod
    def calculate_advanced_metrics(metrics: Dict) -> Dict:
        """calculate_advanced_metrics (:231-319): Calmar, Sortino, recovery factor, expectancy, profit per day
        from a calculate_metrics dict; the streak fields appear only when the caller added a 'trades' list (:267-288)."""
        import numpy as np
        out = dict(metrics)
        dd = metrics.get("max_drawdown", 0)
        out["calmar_ratio"] = (metrics.get("return_pct", 0) / 100) / dd if dd > 0 else float("inf")
        daily = list(metrics.get("daily_returns", {}).values())
        if daily:
            neg = [r for r in daily if r < 0]
            downside = np.std(neg) if neg else 0
            out["sortino_ratio"] = (np.mean(daily) / downside) * np.sqrt(252) if downside > 0 else float("inf")
        else:
            out["sortino_ratio"] = 0
        trades = metrics.get("trades", []) if metrics.get("total_trades", 0) > 0 else []
        if trades:
            win = loss = best_win = best_loss = 0
            for t in sorted(trades, key=lambda x: x.get("timestamp", "")):
                if t.get("pnl", 0) > 0:
                    win, loss = win + 1, 0
                    best_win = max(best_win, win)
                else:
                    loss, win = loss + 1, 0
                    best_loss = max(best_loss, loss)
            out["max_consecutive_wins"], out["max_consecutive_losses"] = best_win, best_loss
        out["recovery_factor"] = (metrics.get("net_profit", 0) / (dd * metrics.get("initial_capital", 10000))
                                  if dd > 0 else float("inf"))
        if metrics.get("total_trades", 0) > 0:
            wr = metrics.get("win_rate", 0)
            out["expectancy"] = wr * metrics.get("average_profit", 0) - (1 - wr) * abs(metrics.get("average_loss", 0))
        else:
            out["expectancy"] = 0
        out["profit_per_day"] = np.mean(daily) if daily else 0
        return out


class StrategyEvaluationSystem:
    def __init__(self, config_path: Optional[str] = "config.json", config: Optional[Dict] = None):
        if config is None:
            try:
                with open(config_path, "r") as f:
                    config = json.load(f)
            except (OSError, TypeError):
                config = {}
        self.config = config
        self.optimization_goals = self.config.get("evolution", {}).get("optimization_goals", {}) or dict(DEFAULT_GOALS)
        self.performance_metrics = self.config.get("evolution", {}).get("performance_metrics", {})

    # -- reference-compatible single-strategy call -----------------------------------
    def _lane_sweep(self, parameters: Dict, market_data: List[Dict], event_cap: int):
        """(one-lane sweep over the points' own price and rsi fields, fp32 prices) for one parameter set."""
        n = len(market_data)
        price = np.array([d.get("price", 50000) for d in market_data], dtype=np.float32)
        rsi = np.array([d.get("rsi", 50) for d in market_data], dtype=np.float32)
        ohlcv = np.zeros((5, 1, n), dtype=np.float32)
        ohlcv[3, 0] = price
        market = MarketData(ohlcv)
        period = int(parameters.get("rsi_period", 14))
        sweep = PopulationSweep.from_bank(market, torch.from_numpy(rsi).to(market.device).view(1, 1, n), [period],
                                          self.optimization_goals, event_cap=event_cap)
        return sweep, price

    def _simulate_trades(self, strategy_id: str, parameters: Dict, market_data: List[Dict]) -> List[Dict]:
        if not market_data:
            return []
        n = len(market_data)
        sweep, price = self._lane_sweep(parameters, market_data, event_cap=n + 1)
        sweep.evaluate([dict(parameters)])
        n_rec = int(sweep.lane_stats()["n_records"][0, 0])
        ev = sweep.events()[0, 0, :n_rec]
        size = 10000 * (min(parameters.get("max_position_size", 5), 20) / 100)     # :761-764
        out, entry = [], 0.0
        for w in ev.tolist():
            bar, is_exit, sell = w & _lib.EVENT_BAR_MASK, bool(w & _lib.EVENT_EXIT), bool(w & _lib.EVENT_SELL)
            d = market_data[bar]
            px = float(price[bar])
            if not is_exit:
                entry = px
                qty, pnl = size / px, -size * 0.001
            else:
                qty = size / entry
                pnl = qty * ((px - entry) if sell else (entry - px)) - size * 0.002
            out.append({"timestamp": d.get("timestamp", f"2023-01-{bar + 1:02d}T00:00:00Z"),
                        "symbol": d.get("symbol", "BTCUSDT"), "side": "sell" if sell else "buy", "price": px,
                        "quantity": qty, "fees": size * 0.001, "pnl": pnl})
        return out

    # -- k-fold cross-validation (:635-744) -----------------------------------------------------------
    CV_METRICS = ("sharpe_ratio", "win_rate", "max_drawdown", "profit_factor", "return_pct")

    def cross_validate_population(self, population: List[Dict], close: torch.Tensor, bank: torch.Tensor, periods,
                                  minute0: int, bar_minutes: int = 1, k_folds: int = 5,
                                  initial_capital: float = 10000.0) -> Dict[str, np.ndarray]:
        """The numeric core of cross_validate_strategy for a whole population at once.

        close [S][N] fp32 and bank [S][P][N] (RSI rows for `periods`) are device tensors.  The bars are cut into
        k contiguous folds (:659-666); for each fold every individual is simulated on the fold ("test") and on
        the other folds glued together ("train", :674-682 -- the state machine runs straight across the seam,
        as the reference's does, and the records keep their own calendar days).  Returns arrays [k][pop][S] for
        the lane metrics `CV_METRICS` and `score`, prefixed train_ / test_."""
        S, N = close.shape
        if N < k_folds:
            k_folds = N
        fold = N // k_folds
        bounds = [(i * fold, (i + 1) * fold if i < k_folds - 1 else N) for i in range(k_folds)]
        out = {f"{side}_{m}": np.zeros((k_folds, len(population), S)) for side in ("train", "test")
               for m in self.CV_METRICS + ("score", "n_records")}

        def run(side, f, c, bk, m0, gap_bar=0, gap_minutes=0):
            market = MarketData.from_close(c.contiguous(), minute0=m0, bar_minutes=bar_minutes)
            sweep = PopulationSweep.from_bank(market, bk.contiguous(), periods, self.optimization_goals,
                                              initial_capital=initial_capital, mode="auto")
            sweep.set_gap(gap_bar, gap_minutes)
            sweep.evaluate(population)
            st = sweep.lane_stats()
            for m in ("sharpe_ratio", "win_rate", "max_drawdown", "profit_factor", "score", "n_records"):
                out[f"{side}_{m}"][f] = st[m]
            out[f"{side}_return_pct"][f] = st["net_profit"] / initial_capital * 100

        for f, (a, b) in enumerate(bounds):
            run("test", f, close[:, a:b], bank[:, :, a:b], minute0 + a * bar_minutes)
            if a == 0 and b == N:
                continue                                               # k = 1: nothing to train on (:672 gives [])
            if a == 0:
                run("train", f, close[:, b:], bank[:, :, b:], minute0 + b * bar_minutes)
            elif b == N:
                run("train", f, close[:, :a], bank[:, :, :a], minute0)
            else:
                run("train", f, torch.cat([close[:, :a], close[:, b:]], dim=1), torch.cat([bank[:, :, :a], bank[:, :, b:]], dim=2),
                    minute0, gap_bar=a, gap_minutes=(b - a) * bar_minutes)
        out["fold_bounds"] = np.array(bounds)
        return out

    @staticmethod
    def _summarize_market_conditions(market_data: List[Dict]) -> Dict:
        """:880-935 (host; a fold's worth of points)."""
        if not market_data:
            return {"trend": "unknown", "volatility": 0, "volume": 0, "period_start": None, "period_end": None}
        prices = [d.get("price", 0) for d in market_data if d.get("price", 0) > 0]
        volumes = [d.get("volume", 0) for d in market_data if d.get("volume", 0) > 0]
        trend, volatility = "unknown", 0
        if len(prices) >= 2:
            change = (prices[-1] - prices[0]) / prices[0] if prices[0] > 0 else 0
            trend = "uptrend" if change > 0.05 else "downtrend" if change < -0.05 else "ranging"
            p = np.asarray(prices, dtype=np.float64)
            volatility = np.std((p[1:] - p[:-1]) / p[:-1])
        return {"trend": trend, "volatility": float(volatility), "volume": float(np.mean(volumes) if volumes else 0),
                "period_start": market_data[0].get("timestamp"), "period_end": market_data[-1].get("timestamp")}

    @staticmethod
    def _calculate_cv_summary(fold_results: List[Dict], test_metric: str, normalize: bool) -> Dict:
        """:937-990."""
        tr = [f["train_score"] for f in fold_results]
        te = [f["test_score"] for f in fold_results]
        summary = {"mean_train_score": float(np.mean(tr)), "std_train_score": float(np.std(tr)),
                   "mean_test_score": float(np.mean(te)), "std_test_score": float(np.std(te)),
                   "train_test_gap": float(np.mean(tr) - np.mean(te)),
                   "relative_overfitting": float((np.mean(tr) - np.mean(te)) / np.mean(tr)) if np.mean(tr) > 0 else 0}
        for side in ("train", "test"):
            for metric in (fold_results[0][f"{side}_metrics"] if fold_results else {}):
                vals = [f[f"{side}_metrics"][metric] for f in fold_results]
                summary[f"mean_{side}_{metric}"] = float(np.mean(vals))
                summary[f"std_{side}_{metric}"] = float(np.std(vals))
        summary["consistency"] = (1.0 - min(1.0, summary["std_test_score"] / summary["mean_test_score"])
                                  if summary["mean_test_score"] > 0 else 0.0)
        return summary

    def cross_validate_strategy(self, strategy_id: str, parameters: Dict, market_data_periods: List[Dict],
                                k_folds: int = 5, test_metric: str = "sharpe_ratio",
                                normalize_results: bool = True) -> Dict:
        """Drop-in for cross_validate_strategy (:635-744) on a flat list of market-data points (keys timestamp,
        symbol, price, rsi[, volume]) on a uniform time grid.  JSON dump and plots (:732-739) are out of scope."""
        pts = market_data_periods
        if len(pts) < k_folds:
            k_folds = len(pts)
        n = len(pts)
        t0 = datetime.fromisoformat(pts[0]["timestamp"].replace("Z", "+00:00"))
        minute0 = int((t0.replace(tzinfo=None) - datetime(1970, 1, 1)).total_seconds() // 60)   # calendar days as written (:151)
        step = 1
        if n > 1:
            t1 = datetime.fromisoformat(pts[1]["timestamp"].replace("Z", "+00:00"))
            step = max(1, int(round((t1 - t0).total_seconds() / 60)))
        dev = torch.device("cuda", torch.cuda.current_device())
        close = torch.from_numpy(np.array([d.get("price", 50000) for d in pts], dtype=np.float32)).to(dev).view(1, n)
        bank = torch.from_numpy(np.array([d.get("rsi", 50) for d in pts], dtype=np.float32)).to(dev).view(1, 1, n)
        period = int(parameters.get("rsi_period", 14))
        cv = self.cross_validate_population([dict(parameters)], close, bank, [period], minute0, step, k_folds)
        fold_results = []
        for f, (a, b) in enumerate(cv["fold_bounds"].tolist()):
            block = {}
            for side in ("train", "test"):
                m = {k: float(cv[f"{side}_{k}"][f, 0, 0]) for k in self.CV_METRICS}
                m["test_metric"] = m.get(test_metric, 0)
                block[f"{side}_metrics"] = m
                block[f"{side}_score"] = float(cv[f"{side}_score"][f, 0, 0])
            fold_results.append({"fold": f + 1, **block, "market_conditions": self._summarize_market_conditions(pts[a:b])})
        return {"strategy_id": strategy_id, "parameters": parameters, "k_folds": len(fold_results),
                "test_metric": test_metric,
                "cv_summary": self._calculate_cv_summary(fold_results, test_metric, normalize_results),
                "fold_results": fold_results, "timestamp": datetime.now().isoformat()}

    def _calculate_strategy_score(self, metrics: Dict) -> float:
        goals = self.optimization_goals
        score = metrics.get(goals.get("primary", "sharpe_ratio"), 0)
        for name in goals.get("secondary", []):
            if name == "max_drawdown":
                score *= (1 - metrics.get("max_drawdown", 0))
            elif name == "win_rate":
                score *= (1 + metrics.get("win_rate", 0))
            elif name == "profit_factor":
                score *= (metrics.get("profit_factor", 1) / 2)
            elif name == "expectancy":
                score *= (1 + min(metrics.get("expectancy", 0) / 100, 1))
        floor = goals.get("constraints", {}).get("min_trades_per_day", 0)
        per_day = metrics.get("trades_per_day", floor)
        if per_day < floor:
            score *= per_day / floor
        return score

    # -- trade-sequence Monte-Carlo (BACKLOG.md:194 "BACK-04") --------------------------------------------------------
    def monte_carlo_trades(self, strategy_id: str, parameters: Dict, market_data: List[Dict],
                           num_simulations: int = 1000, simulation_method: str = "bootstrap", block_len: int = 1,
                           confidence_level: float = 0.95, seed: int = 2024) -> Dict:
        """How much of a strategy's result is the luck of its trade order: the round trips of _simulate_trades'
        records on `market_data` (same flat list of points) are resampled `num_simulations` times on the GPU
        ("bootstrap": with replacement, in circular blocks of `block_len` trips; "shuffle": every trip once, in a keyed
        pseudo-random order) and the equity walked as calculate_metrics walks it.  Returns a dict shaped like
        run_monte_carlo_simulation's (monte_carlo_service.py:339-374) with equity in place of price; `original` holds
        the unresampled sequence's values, `num_trades` counts round trips (two records each).  Logs and returns {} on
        failure (:392)."""
        from .monte_carlo import risk_statistics, statistics_blocks
        from .trade_monte_carlo import TradeMonteCarlo
        try:
            if not market_data:
                logger.error("No market data for the trade Monte-Carlo of %s", strategy_id)
                return {}
            if simulation_method not in _lib.TRADE_MC_METHODS:
                logger.error("Unknown trade simulation method: %s", simulation_method)
                return {}
            sweep, _ = self._lane_sweep(parameters, market_data, event_cap=0)
            trip, n_trips, fee = sweep.trade_pnl([dict(parameters)])
            st = sweep.lane_stats()
            capital = float(sweep.cfg.initial_capital)
            mc = TradeMonteCarlo(sweep.market.device)
            finals, maxdd = mc.simulate(trip, n_trips, fee, num_simulations, simulation_method, block_len, capital, seed)
            blocks = statistics_blocks(risk_statistics(mc.engine, finals[0], maxdd[0], capital, confidence_level,
                                                       mdd_percentiles=(95,)), capital, "equity")
            net = float(st["net_profit"][0, 0])
            return {
                "strategy_id": strategy_id, "symbol": market_data[0].get("symbol", "BTCUSDT"),
                "initial_capital": capital, "num_trades": int(n_trips[0, 0].item()),
                "num_simulations": int(num_simulations), "simulation_method": simulation_method,
                "block_len": int(block_len), "seed": int(seed), "timestamp": datetime.now().isoformat(),
                "original": {"final_equity": capital + net, "return_pct": net / capital * 100,
                             "max_drawdown": float(st["max_drawdown"][0, 0])},
                **blocks,
            }
        except Exception as e:  # reference convention: log, return {}
            logger.error("Error running trade Monte-Carlo simulation for %s: %s", strategy_id, e, exc_info=True)
            return {}

    MC_POPULATION_FIELDS = ("expected_equity", "expected_pct_change", "var", "cvar", "prob_profit", "prob_loss",
                            "mdd_mean", "mdd_median", "mdd_p95", "mdd_max")

    def monte_carlo_population(self, population: List[Dict], market: MarketData,
                               sweep: Optional[PopulationSweep] = None, num_simulations: int = 1000,
                               simulation_method: str = "bootstrap", block_len: int = 1,
                               confidence_level: float = 0.95, seed: int = 2024,
                               max_path_bytes: int = 1 << 30) -> Dict[str, np.ndarray]:
        """monte_carlo_trades for every (individual, symbol) lane of a population -- meant for its top, e.g. to rank it
        by the 5th-percentile return or the 95th-percentile drawdown.  Lane id of (i, s) = i * S + s.  Returns [pop][S]
        arrays of the scalars of monte_carlo_trades' dict: num_trades, original_final_equity / return_pct / max_drawdown,
        MC_POPULATION_FIELDS, and [pop][S][9] arrays percentile_equity / percentile_pct_change at `percentiles`."""
        from .monte_carlo import PERCENTILES, risk_statistics
        from .trade_monte_carlo import TradeMonteCarlo
        sweep = sweep or PopulationSweep(market, optimization_goals=self.optimization_goals)
        trip, n_trips, fee = sweep.trade_pnl(population)
        st = sweep.lane_stats()
        P, S = len(population), market.S
        capital = float(sweep.cfg.initial_capital)
        net = st["net_profit"]
        out = {"num_trades": n_trips.cpu().numpy().astype(np.int64), "original_final_equity": capital + net,
               "original_return_pct": net / capital * 100, "original_max_drawdown": st["max_drawdown"].copy(),
               "percentiles": np.array(PERCENTILES),
               "percentile_equity": np.zeros((P, S, len(PERCENTILES))),
               "percentile_pct_change": np.zeros((P, S, len(PERCENTILES)))}
        for k in self.MC_POPULATION_FIELDS:
            out[k] = np.zeros((P, S))
        mc = TradeMonteCarlo(market.device)
        rows = trip.view(P * S, -1)
        per_call = max(1, int(max_path_bytes) // (8 * int(num_simulations)))     # finals + maxdd fp32 per lane
        for lo in range(0, P * S, per_call):
            hi = min(P * S, lo + per_call)
            finals, maxdd = mc.simulate(rows[lo:hi], n_trips.view(-1)[lo:hi], fee.view(-1)[lo:hi], num_simulations,
                                        simulation_method, block_len, capital, seed, lane_ids=np.arange(lo, hi))
            for r in range(hi - lo):
                i, s = divmod(lo + r, S)
                q = risk_statistics(mc.engine, finals[r], maxdd[r], capital, confidence_level, mdd_percentiles=(95,))
                pv = np.asarray(q["percentile_values"])
                out["percentile_equity"][i, s] = pv
                out["percentile_pct_change"][i, s] = (pv / capital - 1) * 100
                out["expected_equity"][i, s], out["expected_pct_change"][i, s] = q["expected_price"], q["expected_pct"]
                out["var"][i, s], out["cvar"][i, s] = abs(q["var"]), abs(q["cvar"])
                out["prob_profit"][i, s], out["prob_loss"][i, s] = q["prob_profit"], 1 - q["prob_profit"]
                for k in ("mdd_mean", "mdd_median", "mdd_p95", "mdd_max"):
                    out[k][i, s] = q[k]
        return out

    # -- batched form -------------------------------------------------------------
    def evaluate_population(self, population: List[Dict], market: MarketData,
                            sweep: Optional[PopulationSweep] = None, aggregation: str = "mean") -> np.ndarray:
        """aggregation "mean": fitness[i] = mean over symbols of score(metrics(simulate(population[i], symbol)));
        "book": fitness[i] = score(metrics(records of population[i] on every symbol, as one trade list)).  A given
        `sweep` evaluates under its own aggregation."""
        sweep = sweep or PopulationSweep(market, optimization_goals=self.optimization_goals, aggregation=aggregation)
        return sweep.evaluate(population)

    def evaluate_book(self, strategy_id: str, parameters: Dict, market: MarketData) -> Dict:
        """evaluate_strategy (:528-577) on the book of one strategy: its records on every symbol of `market`, in symbol
        order, as ONE trade list.  Returns calculate_metrics + calculate_advanced_metrics of that list (daily / monthly
        returns, equity curve and symbol dicts included, built on the host from the records, formatted as
        _simulate_trades formats them) and `score`, the GPU book pass's score on the advanced dict (the composition of
        evaluate_strategy).  Errors: logged, {} returned (the reference's convention)."""
        try:
            sweep = PopulationSweep(market, optimization_goals=self.optimization_goals, aggregation="book",
                                    score_on_advanced=True)
            fitness = sweep.evaluate([dict(parameters)])
            lanes = sweep.lane_stats()["n_records"][0]
            events = sweep.events()
            close = market.close.cpu().numpy()
            size = 10000 * (min(parameters.get("max_position_size", 5), 20) / 100)      # :761-764
            trades = []
            for s in range(market.S):
                entry = 0.0
                for w in events[0, s, :int(lanes[s])].tolist():
                    bar, is_exit, sell = w & _lib.EVENT_BAR_MASK, bool(w & _lib.EVENT_EXIT), bool(w & _lib.EVENT_SELL)
                    px = float(close[s, bar])
                    if not is_exit:
                        entry = px
                        qty, pnl = size / px, -size * 0.001
                    else:
                        qty = size / entry
                        pnl = qty * ((px - entry) if sell else (entry - px)) - size * 0.002
                    trades.append({"timestamp": bar_timestamp(bar, market.minute0, market.bar_minutes),
                                   "symbol": market.symbols[s], "side": "sell" if sell else "buy", "price": px,
                                   "quantity": qty, "fees": size * 0.001, "pnl": pnl})
            metrics = StrategyPerformanceMetrics.calculate_metrics(trades, sweep.cfg.initial_capital)
            out = StrategyPerformanceMetrics.calculate_advanced_metrics(metrics)
            out.update(strategy_id=strategy_id, parameters=parameters, score=float(fitness[0]),
                       timestamp=datetime.now().isoformat())
            return out
        except Exception as e:        # reference convention: log, return an empty result
            logger.error("Error evaluating the book of strategy %s: %s", strategy_id, e)
            return {}

    def backtest_overfitting(self, population: List[Dict], market: MarketData, n_blocks: int = 16,
                             sweep: Optional[PopulationSweep] = None) -> Dict:
        """How much of the best backtest of `population` is selection bias: CSCV and the Deflated Sharpe Ratio on the
        per-day PnL of every individual's book (its records on every symbol of `market`, PopulationSweep.daily_pnl).  The
        trials are the distinct decoded individuals; the rows hold every calendar day of the series, zeros included, and
        the Sharpe ratios are calculate_metrics' daily rule over all those days (overfitting.cscv).

        Returns pbo, prob_oos_loss, degradation {slope, intercept, r2}, n_trials, n_combinations, n_blocks, block_days,
        dropped_days, first_day, the per-combination arrays sel (a trial index), is_sr, oos_sr, n_below, n_tied, omega,
        logit; [pop] arrays sharpe (annualised, all kept days) and deflated_sharpe; and best {index, sharpe,
        deflated_sharpe}, the individual of highest full-sample Sharpe (the first one on ties).  Errors: logged, {}
        returned (the reference's convention)."""
        from .overfitting import cscv, deflated_sharpe
        try:
            sweep = sweep or PopulationSweep(market, optimization_goals=self.optimization_goals)
            _, unique, expand = sweep._unique(population)
            book, _, first_day = sweep.daily_pnl(unique)
            res = cscv(book, n_blocks)
            dsr = deflated_sharpe(res, res["n_trials"])
            idx = np.arange(len(population)) if expand is None else np.asarray(expand)
            out = {k: v for k, v in res.items() if k not in ("mu", "m2", "m3", "m4", "sharpe")}
            out.update(first_day=first_day, sharpe=res["sharpe"][idx], deflated_sharpe=dsr[idx])
            best = int(np.argmax(out["sharpe"]))
            out["best"] = {"index": best, "sharpe": float(out["sharpe"][best]),
                           "deflated_sharpe": float(out["deflated_sharpe"][best])}
            return out
        except Exception as e:        # reference convention: log, return an empty result
            logger.error("Error measuring the backtest overfitting of a population: %s", e)
            return {}

    def data_snooping(self, population: List[Dict], market: MarketData, benchmark: Optional[Dict] = None,
                      n_boot: int = 10_000, block_len=10.0, alpha: float = 0.05, seed: int = 0,
                      sweep: Optional[PopulationSweep] = None) -> Dict:
        """Is the best of `population` really better than `benchmark` once the search over the population is accounted
        for?  White's Reality Check, Hansen's SPA and Romano and Wolf's StepM (overfitting.spa) on the per-day PnL of
        every individual's book (PopulationSweep.daily_pnl), against the book row of `benchmark` -- the incumbent
        strategy's parameter dict, swept on the same calendar -- or a flat, zero PnL when it is None.  The trials are the
        distinct decoded individuals.

        Returns spa()'s result with the per-trial arrays mean, omega, t_stat and stepm.rejected expanded to `population`
        order, best.index an index into `population` (the first individual of the best trial), and first_day.  Errors:
        logged, {} returned (the reference's convention)."""
        from .overfitting import spa
        try:
            sweep = sweep or PopulationSweep(market, optimization_goals=self.optimization_goals)
            _, unique, expand = sweep._unique(population)
            book, _, first_day = sweep.daily_pnl(unique)
            bench = None if benchmark is None else sweep.daily_pnl([benchmark])[0][0]
            res = spa(book, bench, n_boot=n_boot, block_len=block_len, alpha=alpha, seed=seed)
            idx = np.arange(len(population)) if expand is None else np.asarray(expand)
            for k in ("mean", "omega", "t_stat"):
                res[k] = res[k][idx]
            res["stepm"]["rejected"] = res["stepm"]["rejected"][idx]
            if res["best"] is not None:
                res["best"]["index"] = int(np.flatnonzero(idx == res["best"]["index"])[0])
            res["first_day"] = first_day
            return res
        except Exception as e:        # reference convention: log, return an empty result
            logger.error("Error testing a population for data snooping: %s", e)
            return {}

    def model_confidence_set(self, population: List[Dict], market: MarketData, incumbent: Optional[Dict] = None,
                             alpha: float = 0.10, statistic: str = "R", n_boot: int = 10_000, block_len=10.0,
                             seed: int = 0, sweep: Optional[PopulationSweep] = None) -> Dict:
        """Which individuals of `population` cannot be told apart from the best?  Hansen, Lunde and Nason's Model
        Confidence Set (overfitting.mcs) at level `alpha` on the per-day PnL of every individual's book
        (PopulationSweep.daily_pnl).  The models are the distinct decoded individuals; `incumbent`, the running
        strategy's parameter dict, is swept on the same calendar and added as one more model.

        Returns mcs()'s result with p_values, included, mean and model_of expanded to `population` order; its rows are
        the distinct individuals, then the incumbent (row n_trials - 1), and elimination_order indexes them.  Rows with
        the same book, such as individuals whose differing genes never change a trade, are one model and share one
        p-value.  Also first_day, and incumbent {p_value, included}: is the running strategy still among the best?
        Errors: logged, {} returned (the reference's convention)."""
        from .overfitting import mcs
        try:
            sweep = sweep or PopulationSweep(market, optimization_goals=self.optimization_goals)
            _, unique, expand = sweep._unique(population)
            book, _, first_day = sweep.daily_pnl(unique)
            if incumbent is not None:
                book = torch.cat([book, sweep.daily_pnl([incumbent])[0]], dim=0)
            res = mcs(book, alpha=alpha, statistic=statistic, n_boot=n_boot, block_len=block_len, seed=seed)
            idx = np.arange(len(population)) if expand is None else np.asarray(expand)
            if incumbent is not None:
                res["incumbent"] = dict(p_value=float(res["p_values"][-1]), included=bool(res["included"][-1]))
            for k in ("p_values", "included", "mean", "model_of"):
                res[k] = res[k][idx]
            res["first_day"] = first_day
            return res
        except Exception as e:        # reference convention: log, return an empty result
            logger.error("Error computing the model confidence set of a population: %s", e)
            return {}
