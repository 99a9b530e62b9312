"""ResultAnalyzer drop-in: the JSON / dict side of the reference class, the part `run_backtest.py analyze` drives.

Reference: backtesting/result_analyzer.py -- load_results (:23-30), get_available_results (:32-49),
filter_results (:51-72), generate_summary_report (:226-328), compare_results (:330-424),
save_summary_report (:426-437); caller run_backtest.py:152-186.  Error convention kept: never raise, log and
return {} / [] / None.

Charts: the reference draws with matplotlib + seaborn, which this image does not have and which are no part of the
hot path.  `compare_results` builds the same comparison table and writes it as `comparison_<metric>.csv` under
`plots_dir` (a PNG bar chart as well when matplotlib happens to be importable); `plot_equity_curve` /
`plot_trade_analysis` return None without matplotlib, the value the reference returns when plotting fails
(:146-148, :223-225).
"""
from __future__ import annotations

import csv
import json
import logging
from pathlib import Path
from typing import Dict, List, Optional, Union

logger = logging.getLogger("b200bt.result_analyzer")


def _return_pct(stats: Dict) -> float:
    ib, fb = stats.get("initial_balance", 0), stats.get("final_balance", 0)
    return ((fb / ib) - 1) * 100 if ib > 0 else 0                      # :277-280, :348-351


class ResultAnalyzer:
    def __init__(self, results_dir: str = "backtesting/results", plots_dir: Optional[str] = None):
        self.results_dir = Path(results_dir)
        self.results_dir.mkdir(parents=True, exist_ok=True)
        self.plots_dir = Path(plots_dir) if plots_dir is not None else Path("backtesting/plots")     # :19-20

    # -- files ---------------------------------------------------------------------------
    def load_results(self, result_path: Union[str, Path]) -> Dict:
        try:
            with open(result_path, "r") as f:
                return json.load(f)
        except Exception as e:
            logger.error("Error loading result file %s: %s", result_path, e)
            return {}

    def get_available_results(self) -> List[Dict]:
        results = []
        for file_path in self.results_dir.glob("*.json"):
            try:
                with open(file_path, "r") as f:
                    data = json.load(f)
                data["file_path"] = str(file_path)
                results.append(data)
            except Exception as e:
                logger.error("Error loading result file %s: %s", file_path, e)
        return results

    def filter_results(self, strategy: str = None, symbol: str = None, interval: str = None,
                       min_trades: int = 0) -> List[Dict]:
        out = []
        for result in self.get_available_results():
            if strategy and result.get("strategy") != strategy:
                continue
            if symbol and result.get("symbol") != symbol:
                continue
            if interval and result.get("interval") != interval:
                continue
            if min_trades and result.get("stats", {}).get("total_trades", 0) < min_trades:
                continue
            out.append(result)
        return out

    # -- reports -------------------------------------------------------------------------
    def generate_summary_report(self, results: List[Dict]) -> Dict:
        if not results:
            return {}
        rows, strategies, symbols, intervals = [], set(), set(), set()
        tot_wr = tot_pf = tot_sh = 0
        total_trades = profitable = 0
        best = worst = None
        best_ret, worst_ret = -float("inf"), float("inf")
        for i, r in enumerate(results):
            st = r.get("stats", {})
            strategies.add(r.get("strategy", "Unknown")); symbols.add(r.get("symbol", "Unknown")); intervals.add(r.get("interval", "Unknown"))
            ret = _return_pct(st)
            profitable += 1 if st.get("final_balance", 0) > st.get("initial_balance", 0) else 0
            if ret > best_ret:
                best_ret, best = ret, i
            if ret < worst_ret:
                worst_ret, worst = ret, i
            total_trades += st.get("total_trades", 0)
            tot_wr += st.get("win_rate", 0); tot_pf += st.get("profit_factor", 0); tot_sh += st.get("sharpe_ratio", 0)
            rows.append({"strategy": r.get("strategy", "Unknown"), "symbol": r.get("symbol", "Unknown"),
                         "interval": r.get("interval", "Unknown"), "trades": st.get("total_trades", 0),
                         "win_rate": st.get("win_rate", 0), "profit_factor": st.get("profit_factor", 0),
                         "sharpe_ratio": st.get("sharpe_ratio", 0), "return_pct": ret,
                         "max_drawdown": st.get("max_drawdown_pct", 0), "file_path": r.get("file_path", "")})
        n = len(results)
        return {"strategies": list(strategies), "symbols": list(symbols), "intervals": list(intervals), "total_results": n,
                "average_win_rate": tot_wr / n, "average_profit_factor": tot_pf / n, "average_sharpe_ratio": tot_sh / n,
                "best_result": results[best] if best is not None else None,
                "worst_result": results[worst] if worst is not None else None,
                "total_trades": total_trades, "profitable_strategies": profitable, "results": rows}

    def comparison_table(self, results: List[Dict]) -> List[Dict]:
        """The rows compare_results charts (:338-361)."""
        rows = []
        for result in results:
            st = result.get("stats", {})
            rows.append({"strategy": result.get("strategy", "Unknown"), "symbol": result.get("symbol", "Unknown"),
                         "interval": result.get("interval", "Unknown"), "win_rate": st.get("win_rate", 0),
                         "profit_factor": st.get("profit_factor", 0), "sharpe_ratio": st.get("sharpe_ratio", 0),
                         "max_drawdown": st.get("max_drawdown_pct", 0), "return_pct": _return_pct(st),
                         "total_trades": st.get("total_trades", 0)})
        return rows

    def compare_results(self, results: List[Dict], metric: str = "return_pct", save_path: Optional[str] = None) -> Optional[str]:
        try:
            if not results:
                logger.error("No results provided for comparison")
                return None
            rows = self.comparison_table(results)
            if metric not in rows[0]:
                logger.error("Metric %s not found in result data", metric)
                return None
            self.plots_dir.mkdir(parents=True, exist_ok=True)
            path = Path(save_path) if save_path else self.plots_dir / f"comparison_{metric}.csv"
            try:
                import matplotlib
                matplotlib.use("Agg")
                import matplotlib.pyplot as plt
            except Exception:
                plt = None
            if plt is not None and (save_path is None or path.suffix.lower() == ".png"):
                png = path.with_suffix(".png")
                vals = [r[metric] for r in rows]
                plt.figure(figsize=(14, 8))
                plt.bar(range(len(rows)), vals, color=["green" if v >= 0 else "red" for v in vals])
                plt.title(f"Comparison by {metric}")
                plt.xticks(range(len(rows)), [f"{r['strategy']}\n{r['symbol']}\n{r['interval']}" for r in rows], rotation=45)
                plt.ylabel(metric); plt.grid(True, axis="y"); plt.tight_layout(); plt.savefig(png); plt.close()
                return str(png)
            with open(path, "w", newline="") as f:
                w = csv.DictWriter(f, fieldnames=list(rows[0]))
                w.writeheader()
                w.writerows(rows)
            return str(path)
        except Exception as e:
            logger.error("Error comparing results: %s", e)
            return None

    def plot_equity_curve(self, result: Dict, save_path: Optional[str] = None) -> Optional[str]:
        logger.error("Error plotting equity curve: matplotlib is not part of the H100 drop-in")
        return None

    def plot_trade_analysis(self, result: Dict, save_path: Optional[str] = None) -> Optional[str]:
        logger.error("Error plotting trade analysis: matplotlib is not part of the H100 drop-in")
        return None

    def save_summary_report(self, summary: Dict, filename: str = "backtest_summary.json") -> Optional[str]:
        path = self.results_dir / filename
        try:
            with open(path, "w") as f:
                json.dump(summary, f, indent=2, default=float)
            return str(path)
        except Exception as e:
            logger.error("Error saving summary report: %s", e)
            return None
