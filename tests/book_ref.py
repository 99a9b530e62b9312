"""Float64 restatement of the book metrics (b200bt_book_metrics, include/b200bt.h): the lanes of one
individual, as oracle/sim_oracle.c emits them (event words and record pnl), merged in the order (bar, symbol, record index)
and walked the way calculate_metrics (services/strategy_evaluation.py:32-228) walks one mixed trade list, in numpy so that
full-size books (10^5..10^6 records) take milliseconds."""
from __future__ import annotations

import math

import numpy as np

SYMBOL_TAG = 0x9E3779B1
BAR_MASK = 0x3FFFFFFF


def _order(events: list):
    """(bars, symbols, words, index into the concatenated lanes) in book order: lexicographic on (bar, symbol, record)."""
    words = np.concatenate([np.asarray(ev, dtype=np.uint32) for ev in events]) if events else np.zeros(0, np.uint32)
    syms = np.concatenate([np.full(len(ev), s, dtype=np.int64) for s, ev in enumerate(events)]) if events else \
        np.zeros(0, np.int64)
    bars = (words & BAR_MASK).astype(np.int64)
    idx = np.lexsort((np.arange(len(words)), syms, bars))        # stable: record index breaks the remaining ties
    return bars[idx], syms[idx], words[idx], idx


def merged(events: list, pnls: list) -> list:
    """[(bar, symbol, word, pnl)] of the lanes' records in book order."""
    bars, syms, words, idx = _order(events)
    pnl = np.concatenate([np.asarray(p, dtype=np.float64) for p in pnls])[idx] if len(idx) else np.zeros(0)
    return list(zip(bars.tolist(), syms.tolist(), words.tolist(), pnl.tolist()))


def _hash(words: np.ndarray, syms: np.ndarray) -> int:
    """xor over records r of event_hash(r, word_r ^ (symbol_r * SYMBOL_TAG)), in uint32 lanes."""
    if len(words) == 0:
        return 0
    with np.errstate(over="ignore"):
        idx = np.arange(len(words), dtype=np.uint32)
        w = words.astype(np.uint32) ^ (syms.astype(np.uint32) * np.uint32(SYMBOL_TAG))
        a = (idx * np.uint32(0x9E3779B1)) ^ w
        a = a * np.uint32(0x85EBCA77)
        a ^= a >> np.uint32(15)
        b = (w * np.uint32(0xC2B2AE3D)) ^ ((idx << np.uint32(13)) | (idx >> np.uint32(19)))
        b = b * np.uint32(0x27D4EB2F)
        b ^= b >> np.uint32(16)
    return (int(np.bitwise_xor.reduce(b)) << 32) | int(np.bitwise_xor.reduce(a))


def book(events: list, pnls: list, cfg) -> dict:
    """Book stats (the b200bt_lane_stats fields) of one individual: events[s] / pnls[s] = its records on symbol s.
    `cfg`: an oracle.sim_oracle.Config.  The equity is the running float64 sum in book order (np.cumsum adds in order,
    as the record loop of calculate_metrics :128-139 does); a record that does not set a new peak (strict >) is a
    drawdown candidate (peak - equity) / peak."""
    bars, syms, words, idx = _order(events)
    p = np.concatenate([np.asarray(x, dtype=np.float64) for x in pnls])[idx] if len(idx) else np.zeros(0)
    n = len(p)
    cap = cfg.initial_capital
    eq = np.cumsum(np.concatenate([[cap], p]))[1:]
    peak_before = np.maximum.accumulate(np.concatenate([[cap], eq]))[:-1]
    cand = ~(eq > peak_before)
    peak_at = np.maximum(peak_before, eq)
    maxdd = float(np.max((peak_at[cand] - eq[cand]) / peak_at[cand])) if cand.any() else 0.0
    win, loss = p > 0, p < 0
    tot_p, tot_l = float(np.sum(p[win])) if win.any() else 0.0, float(np.sum(p[loss])) if loss.any() else 0.0
    gap = np.where((cfg.gap_bar > 0) & (bars >= cfg.gap_bar), cfg.gap_minutes, 0)
    day = (cfg.minute0 + bars * cfg.bar_minutes + gap) // 1440
    if n:
        starts = np.concatenate([[0], np.nonzero(day[1:] != day[:-1])[0] + 1])
        daily = np.add.reduceat(p, starts)
    else:
        daily = np.zeros(0)
    dur = int(np.sum(bars[1:n - n % 2:2] - bars[0:n - n % 2:2])) if n >= 2 else 0
    out = dict(n_records=float(n), n_wins=float(win.sum()), n_losses=float(loss.sum()), total_profit=tot_p,
               total_loss=tot_l, net_profit=tot_p + tot_l, max_drawdown=maxdd, n_days=float(len(daily)),
               largest_profit=float(p[win].max()) if win.any() else 0.0,
               largest_loss=float(p[loss].min()) if loss.any() else 0.0, sum_duration_bars=float(dur),
               trade_hash=_hash(words, syms))
    sharpe = win_rate = pf = 0.0
    if n >= 2:
        win_rate = float(win.sum()) / n
        pf = abs(tot_p / tot_l) if tot_l != 0 else math.inf
        if len(daily) > 1:
            sd = float(np.std(daily))
            sharpe = float(np.mean(daily)) / sd * math.sqrt(252) if sd > 0 else 0.0
    out.update(sharpe_ratio=sharpe, win_rate=win_rate, profit_factor=pf)
    mean_daily = downside = sortino = 0.0
    n_neg = 0
    if n >= 2 and len(daily) > 0:
        mean_daily = float(np.mean(daily))
        neg = daily[daily < 0]
        n_neg = len(neg)
        downside = float(np.std(neg)) if n_neg else 0.0
        sortino = mean_daily / downside * math.sqrt(252) if downside > 0 else math.inf
    out.update(sortino_ratio=sortino, n_negative_days=float(n_neg), downside_deviation=downside, mean_daily_pnl=mean_daily)
    out["score"] = score(out, cfg)
    return out


def score(o: dict, cfg) -> float:
    """_calculate_strategy_score (:579-633) under the codes of include/b200bt.h (as oracle/sim_oracle.c)."""
    ret_pct = o["net_profit"] / cfg.initial_capital * 100
    avg_p = o["total_profit"] / o["n_wins"] if o["n_wins"] > 0 else 0.0
    avg_l = o["total_loss"] / o["n_losses"] if o["n_losses"] > 0 else 0.0
    wr, pf, dd = o["win_rate"], o["profit_factor"], o["max_drawdown"]
    expectancy = wr * avg_p - (1 - wr) * abs(avg_l) if o["n_records"] > 0 else 0.0
    primary = {
        1: ret_pct, 2: pf, 3: wr, 4: o["net_profit"], 5: o["n_records"], 6: dd, 7: o["total_profit"], 8: o["total_loss"],
        9: o["largest_profit"], 10: o["largest_loss"], 11: avg_p, 12: avg_l, 13: o["sortino_ratio"], 14: expectancy,
        15: (ret_pct / 100) / dd if dd > 0 else math.inf, 16: o["mean_daily_pnl"],
        17: o["net_profit"] / (dd * 10000) if dd > 0 else math.inf, 99: 0.0,
    }.get(cfg.primary, o["sharpe_ratio"])
    s = primary
    if cfg.secondary_mask & 1:
        s *= (1 - dd)
    if cfg.secondary_mask & 2:
        s *= (1 + wr)
    if cfg.secondary_mask & 4:
        s *= (pf / 2)
    if cfg.secondary_mask & 8:
        s *= (1 + min(expectancy / 100, 1.0))
    return s
