"""Generate the book fixture by EXECUTING the reference's own code on multi-symbol trade lists.

Run where a copy of the reference tree exists (as for make_golden.py, whose goal sets and JSON conventions it shares):

    python tests/golden/make_book.py

Writes tests/golden/book_reference.json (reference metrics per book) and book_reference.npz (fp32 close / RSI rows of every
symbol and the merged record order of every book).  For each case, S synthetic symbols share one timestamp grid; per
individual the reference's own
    StrategyEvaluationSystem._simulate_trades      services/strategy_evaluation.py:746   (per symbol)
produces the records, which are concatenated in symbol order (the list evaluate_strategy :528-577 hands on), then
    StrategyPerformanceMetrics.calculate_metrics   :32    (sorts the mixed list by timestamp, :67)
    calculate_advanced_metrics                     :231
    _calculate_strategy_score                      :579   (config goals and the 12 goal sets of make_golden.ALT_GOALS)
Cases: records of different symbols on the same bar (symbols that copy one series), an entry on the last bar with its
force-close, a book with 0 records, a symbol that never trades (RSI NaN), merged pairs (2k, 2k+1) that cross symbols, a
1-minute and a 1440-minute grid.  A book of exactly 1 record cannot come out of _simulate_trades (every entry is closed),
so the 1-record short dict (:68-92) is recorded on the first record of a book, fed to calculate_metrics directly.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
OUT = Path(__file__).resolve().parent

from ai_crypto_trader_b200 import synth  # noqa: E402
from oracle import indicators_ref, ref_runner, simulate_ref  # noqa: E402
from make_golden import ALT_GOALS, SCALARS, jsonable  # noqa: E402

PERIODS = [5, 9, 14]
SOURCE = [0, 1, 0, 2]          # symbols 0 and 2 copy one series (ties); symbol 3's RSI is NaN (never trades)
QUIET = 3
POPULATION = [
    {"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30, "take_profit": 3, "stop_loss": 2},
    {"rsi_period": 5, "rsi_overbought": 65, "rsi_oversold": 35, "take_profit": 1, "stop_loss": 1},
    {"rsi_period": 9, "rsi_overbought": 71, "rsi_oversold": 33, "take_profit": 2.7312, "stop_loss": 0.5519,
     "max_position_size": 12},
    {"rsi_period": 5, "rsi_overbought": 101, "rsi_oversold": 99, "take_profit": 0.0001, "stop_loss": 0.0001},  # dense
    {"rsi_period": 9, "rsi_overbought": 100, "rsi_oversold": 0},                                                 # 0 records
    {"rsi_period": 14, "rsi_overbought": 40, "rsi_oversold": 60, "take_profit": 2, "stop_loss": 2},
]
DENSE = 3


def _market(n_bars):
    close = np.ascontiguousarray(synth.synth_ohlcv(3, n_bars)[3][SOURCE])
    rsi = np.stack([indicators_ref.rsi_bank(close[s], PERIODS) for s in range(len(SOURCE))]).astype(np.float32)
    rsi[QUIET] = np.nan
    return close, rsi


def _last_bar_entry_length(lo, hi):
    """A series length at which the dense individual enters on the last bar (and is force-closed there)."""
    for n in range(lo, hi):
        close, rsi = _market(n)
        recs = simulate_ref.simulate_trades(POPULATION[DENSE], simulate_ref.market_points(
            close[0], rsi[0, PERIODS.index(5)], "S0", synth.EPOCH_2024_MINUTES))
        if len(recs) >= 2 and recs[-1]["timestamp"] == recs[-2]["timestamp"]:
            return n
    raise RuntimeError("no length puts an entry on the last bar")


def make_book():
    ses, metrics_cls = ref_runner.strategy_evaluation()
    goals = ref_runner.optimization_goals()
    arrays, cases = {}, []
    for name, bar_minutes, n_bars in (("grid_1m", 1, _last_bar_entry_length(2000, 2100)), ("grid_1440m", 1440, 500)):
        close, rsi = _market(n_bars)
        arrays[f"close_{name}"] = close
        arrays[f"rsi_{name}"] = rsi
        books = []
        for i, params in enumerate(POPULATION):
            trades, symbol_of = [], {}
            for s in range(len(SOURCE)):
                sym = f"SYN{s:03d}USDT"
                symbol_of[sym] = s
                points = simulate_ref.market_points(close[s], rsi[s, PERIODS.index(params["rsi_period"])], sym,
                                                    synth.EPOCH_2024_MINUTES, bar_minutes)
                trades += ses._simulate_trades(f"{name}_{i}", dict(params), points)       # REFERENCE, per symbol
            m = metrics_cls.calculate_metrics(trades)                                      # REFERENCE, one mixed list
            adv = metrics_cls.calculate_advanced_metrics(m)                                # REFERENCE
            score = ses._calculate_strategy_score(m)                                       # REFERENCE
            alt = []
            for g, on_advanced in ALT_GOALS:                                               # REFERENCE
                ses.optimization_goals = g
                alt.append(jsonable(ses._calculate_strategy_score(adv if on_advanced else m)))
            ses.optimization_goals = goals
            # the merged order: calculate_metrics' own stable sort of the concatenated list
            merged = sorted(trades, key=lambda x: x.get("timestamp", ""))
            t0 = simulate_ref.market_points(close[0][:1], rsi[0, 0][:1], "x", synth.EPOCH_2024_MINUTES, bar_minutes)[0]
            from datetime import datetime
            base = datetime.fromisoformat(t0["timestamp"])
            arrays[f"bar_{name}_{i}"] = np.array(
                [int((datetime.fromisoformat(t["timestamp"]) - base).total_seconds() // 60) // bar_minutes for t in merged],
                dtype=np.int64)
            arrays[f"sym_{name}_{i}"] = np.array([symbol_of[t["symbol"]] for t in merged], dtype=np.int64)
            arrays[f"pnl_{name}_{i}"] = np.array([t["pnl"] for t in merged], dtype=np.float64)
            daily = m.get("daily_returns", {})
            books.append({
                "params": params, "n_records": len(trades),
                "metrics": {k: jsonable(m[k]) for k in SCALARS},
                "advanced": {k: jsonable(adv[k]) for k in simulate_ref.ADVANCED_KEYS},
                "score": jsonable(score), "alt_scores": alt,
                "daily_returns": [jsonable(daily[k]) for k in sorted(daily)],
                "profitable_symbols": {k: jsonable(v) for k, v in m.get("profitable_symbols", {}).items()},
                "unprofitable_symbols": {k: jsonable(v) for k, v in m.get("unprofitable_symbols", {}).items()},
            })
            print(f"{name} #{i}: records={len(trades):5d} score={float(score):.6g}")
        one = metrics_cls.calculate_metrics(trades[:1]) if trades else None
        cases.append({"name": name, "bar_minutes": bar_minutes, "n_bars": int(n_bars), "books": books,
                      "one_record": None if one is None else {k: jsonable(one[k]) for k in SCALARS}})
    np.savez_compressed(OUT / "book_reference.npz", **arrays)
    (OUT / "book_reference.json").write_text(json.dumps(
        {"periods": PERIODS, "source": SOURCE, "quiet": QUIET, "minute0": synth.EPOCH_2024_MINUTES, "goals": goals,
         "alt_goals": [{"goals": g, "advanced": a} for g, a in ALT_GOALS], "cases": cases}, indent=1))


if __name__ == "__main__":
    if not ref_runner.available():
        raise SystemExit("the reference tree is not available (see oracle/ref_runner.py)")
    make_book()
