"""NumPy / pandas restatement of the market-regime contract (b200bt_regime_labels, b200bt_class_stats;
include/b200bt.h): the points of a market's bars, the 24-hour windows and the rule of detect_regime_from_data
(services/market_regime_service.py:503-603), the bar labels, the per-regime performance of
update_strategy_performance_by_regime (:829-993), and the trade metrics of a lane's records per label (tests/book_ref.book
on the filtered records of an oracle/sim_oracle.c lane)."""
from __future__ import annotations

import numpy as np
import pandas as pd

import book_ref

BULL, BEAR, RANGING, VOLATILE, UNKNOWN = range(5)
NAMES = ("bull", "bear", "ranging", "volatile", "unknown")
UP, DOWN, SIDEWAYS = 0, 1, 2
TREND_NAMES = ("uptrend", "downtrend", "sideways")
BAR_MASK = 0x3FFFFFFF

DEFAULT_THRESHOLDS = {"bull": {"trend_strength": 0.6, "price_change": 5.0, "volatility": 0.5},
                      "bear": {"trend_strength": 0.6, "price_change": -5.0, "volatility": 0.5},
                      "volatile": {"volatility": 1.5},
                      "ranging": {"trend_strength": 0.3, "price_range": 3.0}}


def points(close, sma20, sma50, sma5, minute0: int, bar_minutes: int, sample_minutes: int):
    """(bar index, minute, price, trend code, trend_strength) of the points of one symbol: the last bar of every
    epoch-aligned sample bucket that a later bar leaves, from the first one where the three averages are defined.
    float64 arithmetic in the order of market_monitor_service.py:263-280."""
    N = len(close)
    t = np.arange(N, dtype=np.int64)
    m = minute0 + t * bar_minutes
    is_pt = (m + bar_minutes) // sample_minutes != m // sample_minutes
    c, s20, s50, s5 = (np.asarray(x, dtype=np.float64) for x in (close, sma20, sma50, sma5))
    ok = is_pt & ~np.isnan(s20) & ~np.isnan(s50) & ~np.isnan(s5)
    if not ok.any():
        e = np.zeros(0)
        return e.astype(np.int64), e.astype(np.int64), e, e.astype(np.int64), e
    idx = np.nonzero(is_pt & (t >= np.argmax(ok)))[0]
    c, s20, s50, s5 = c[idx], s20[idx], s50[idx], s5[idx]
    st1 = (c - s20) / s20 * 100
    st5 = (c - s5) / s5 * 100
    strength = np.abs(st1 * 0.6 + st5 * 0.4)
    trend = np.where((c > s20) & (s20 > s50), UP, np.where((c < s20) & (s20 < s50), DOWN, SIDEWAYS))
    return idx, m[idx], c, trend, strength


def detect(prices, trends, strengths, thr=None) -> dict:
    """detect_regime_from_data on one window's points (in time order): its statistics, label and the branch taken."""
    thr = thr or DEFAULT_THRESHOLDS
    n = len(prices)
    out = dict(n_points=n, volatility=np.nan, change_pct=np.nan, mean_strength=np.nan, up_frac=np.nan,
               down_frac=np.nan, sideways_frac=np.nan, label=UNKNOWN, branch="unknown")
    if n == 0:
        return out
    p = pd.Series(np.asarray(prices, dtype=np.float64))
    vol = p.pct_change().std() * np.sqrt(24)
    change = ((p.iloc[-1] - p.iloc[0]) / p.iloc[0]) * 100
    ts = pd.Series(np.asarray(strengths, dtype=np.float64)).mean()
    tr = np.asarray(trends)
    up, down, side = (float(np.sum(tr == k)) / n for k in (UP, DOWN, SIDEWAYS))
    out.update(volatility=vol, change_pct=change, mean_strength=ts, up_frac=up, down_frac=down, sideways_frac=side)
    if n < 2:
        return out
    if vol > thr["volatile"]["volatility"]:
        label, branch = VOLATILE, "volatile"
    elif change > thr["bull"]["price_change"] and up > thr["bull"]["trend_strength"]:
        label, branch = BULL, "bull"
    elif change < thr["bear"]["price_change"] and down > thr["bear"]["trend_strength"]:
        label, branch = BEAR, "bear"
    elif abs(change) < thr["ranging"]["price_range"] and ts < thr["ranging"]["trend_strength"]:
        label, branch = RANGING, "ranging"
    elif up > down and up > side:
        label, branch = BULL, "default bull"
    elif down > up and down > side:
        label, branch = BEAR, "default bear"
    else:
        label, branch = RANGING, "default ranging"
    out.update(label=label, branch=branch)
    return out


def windows(minutes, prices, trends, strengths, thr=None) -> list:
    """The 24-hour windows [t0 + 1440 k, t0 + 1440 (k + 1)) from the first point's minute t0, while their start < the
    last point's minute (:863-885); each row: start_minute plus detect()'s fields (n_points 0: skipped)."""
    minutes = np.asarray(minutes, dtype=np.int64)
    if len(minutes) == 0:
        return []
    t0, last = int(minutes[0]), int(minutes[-1])
    rows = []
    k = 0
    while t0 + 1440 * k < last:
        w0 = t0 + 1440 * k
        sel = (minutes >= w0) & (minutes < w0 + 1440)
        row = detect(np.asarray(prices)[sel], np.asarray(trends)[sel], np.asarray(strengths)[sel], thr)
        row["start_minute"] = w0
        rows.append(row)
        k += 1
    return rows


def bar_labels(N: int, minute0: int, bar_minutes: int, rows: list) -> np.ndarray:
    """uint8 [N]: the label of the window holding each bar's minute, UNKNOWN outside every window."""
    m = minute0 + np.arange(N, dtype=np.int64) * bar_minutes
    out = np.full(N, UNKNOWN, dtype=np.uint8)
    for r in rows:
        out[(m >= r["start_minute"]) & (m < r["start_minute"] + 1440)] = r["label"]
    return out


def symbol_labels(close, sma20, sma50, sma5, minute0, bar_minutes, sample_minutes, thr=None):
    """(labels uint8 [N], window rows) of one symbol."""
    _, m, p, tr, st = points(close, sma20, sma50, sma5, minute0, bar_minutes, sample_minutes)
    rows = windows(m, p, tr, st, thr)
    return bar_labels(len(close), minute0, bar_minutes, rows), rows


def performance_by_regime(rows: list, trades: list) -> dict:
    """update_strategy_performance_by_regime's per-regime entry of one strategy: trades = [(minute, profit)] matched to
    the windows with points by their minute; win_rate, profit_factor, trade_count (:928-985)."""
    out = {}
    for regime in ("bull", "bear", "ranging", "volatile"):
        wins = [r for r in rows if r["n_points"] > 0 and NAMES[r["label"]] == regime]
        if not wins:
            continue
        sel = [p for m, p in trades if any(w["start_minute"] <= m < w["start_minute"] + 1440 for w in wins)]
        if not sel:
            continue
        n = len(sel)
        win_rate = sum(1 for p in sel if p > 0) / n
        total_loss = abs(sum(p for p in sel if p < 0))
        pf = sum(sel) / total_loss if total_loss > 0 else 1
        out[regime] = {"win_rate": win_rate * n / n, "profit_factor": pf * n / n, "trade_count": n}
    return out


def _equal_days(out: dict, ev, pn, cfg) -> dict:
    """The metrics step's daily moments are shifted to the first day (csrc/sweep_dev.cuh day_complete): days whose sums
    are all equal have exactly 0 variance, so Sharpe is 0 (and with equal negative days the downside deviation is 0 and
    Sortino +inf), where np.std of equal values may leave a rounding residue.  A class list of one kind of record (all
    entries, each day -fee) makes such days common."""
    n = len(ev)
    if n < 2:
        return out
    bars = (np.asarray(ev, dtype=np.int64) & BAR_MASK)
    gap = np.where((cfg.gap_bar > 0) & (bars >= cfg.gap_bar), cfg.gap_minutes, 0)
    day = (cfg.minute0 + bars * cfg.bar_minutes + gap) // 1440
    daily = np.add.reduceat(np.asarray(pn, dtype=np.float64), np.concatenate([[0], np.nonzero(day[1:] != day[:-1])[0] + 1]))
    changed = False
    if len(daily) > 1 and np.all(daily == daily[0]):
        out["sharpe_ratio"], changed = 0.0, True
    neg = daily[daily < 0]
    if len(neg) and np.all(neg == neg[0]):
        out["downside_deviation"], out["sortino_ratio"], changed = 0.0, float("inf"), True
    if changed:
        out["score"] = book_ref.score(out, cfg)
    return out


def class_stats(events, pnls, labels_row, R: int, cfg) -> list:
    """book_ref.book of the records of one lane whose bar carries label r, for r = 0 .. R - 1."""
    ev = np.asarray(events, dtype=np.uint32)
    pn = np.asarray(pnls, dtype=np.float64)
    lab = np.asarray(labels_row)[(ev & BAR_MASK).astype(np.int64)] if len(ev) else np.zeros(0, np.uint8)
    return [_equal_days(book_ref.book([ev[lab == r]], [pn[lab == r]], cfg), ev[lab == r], pn[lab == r], cfg)
            for r in range(R)]
