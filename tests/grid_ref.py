"""Plain Python / NumPy restatement of the grid service's simulation loop (services/grid_trading_strategy.py run()
:122-233 in simulation mode), pinned to tests/golden/grid_reference.json, which the reference's own run() wrote.  The
oracle of the GPU tests of b200bt_grid_sweep.

simulate       tick by tick with the reference's expressions (list comprehensions over the levels, levels.index, the
               strict-> checks written as tick periods); exact
simulate_fast  the same rule with NumPy over the ticks between two checks (searchsorted and prefix sums over the
               levels): same counts, regenerations and levels; profit and cash summed in another order
"""
from __future__ import annotations

import bisect
from typing import Dict, List, Optional

import numpy as np

FIELDS = ("total_profit", "total_trades", "profitable_trades", "win_rate", "profit_per_day", "up_crossings",
          "down_crossings", "n_regenerations", "num_grids", "lower", "upper", "cash", "position", "mark_to_market",
          "max_position", "min_position", "n_rebalance_checks", "n_adjustments", "n_ticks", "near_ties")


def levels(lower: float, upper: float, n: int, kind: int) -> List[float]:
    """_generate_grid_levels (:347-385); kind 0 arithmetic, 1 geometric."""
    if kind == 0:
        step = (upper - lower) / n
        return [lower + i * step for i in range(n + 1)]
    ratio = (upper / lower) ** (1 / n)
    return [lower * (ratio ** i) for i in range(n + 1)]


def _near(x: float, lv: List[float]) -> bool:
    """x within |L| * 2^-50 of a level a bound on x compares it with last (the kernel's near-tie rule)."""
    for strict in (False, True):
        e = bisect.bisect_right(lv, x) if strict else bisect.bisect_left(lv, x)
        for j in (e - 1, e):
            if 0 <= j < len(lv) and abs(x - lv[j]) <= abs(lv[j]) * 2.0 ** -50:
                return True
    return False


def _finish(st: Dict, T: int, bar_seconds: int, last_price: float) -> Dict:
    total = st["up_crossings"] + st["down_crossings"]
    secs = (T - 1) * bar_seconds
    st["total_trades"] = total
    st["win_rate"] = st["profitable_trades"] / total if total > 0 else 0.0
    st["profit_per_day"] = st["total_profit"] / (secs / 86400) if secs > 0 else 0.0
    st["mark_to_market"] = st["cash"] + st["position"] * last_price
    st["n_ticks"] = T
    return st


def simulate(prices, lower: float, upper: float, n: int, kind: int, qty: float, lower_pct: float, upper_pct: float,
             rebalance_ticks: int, adjust_ticks: int, adapt: bool = False, labels=None, table: Optional[Dict] = None,
             bar_seconds: int = 60, days=None) -> Dict:
    """One lane, tick by tick.  prices: the tick prices (floats, tick 0 = the start bar); labels: per-tick labels
    (B200BT_REGIME_* ints) or None; table: {label: (num_grids, lower_pct, upper_pct)}; days: per-tick day index, for the
    per-day snapshots.  Returns the stats fields plus "regenerations" [(tick, lower, upper, n)] (tick 0 = the initial
    grid), "levels" (the final ones), "day_profit" {day: realised profit} and "snapshots" [(day, tick, total_trades,
    profitable_trades, total_profit)] at each day's last tick."""
    prices = [float(p) for p in prices]
    T = len(prices)
    lv = levels(lower, upper, n, kind)
    n_cur, lo_pct, up_pct = n, lower_pct, upper_pct
    st = {f: 0 for f in FIELDS}
    st.update(total_profit=0.0, cash=0.0)
    regens = [(0, lower, upper, n)]
    net = nmax = nmin = 0
    ties = 0
    day_profit: Dict[int, float] = {}
    snaps = []
    last = prices[0]
    for k in range(T):
        cur = prices[k]
        p_day = 0.0
        if (cur > last or cur < last) and kind == 1 and (_near(last, lv) or _near(cur, lv)):
            ties += 1
        if cur > last:
            for level in [lv_ for lv_ in lv if last <= lv_ <= cur]:
                profit = (level - lv[lv.index(level) - 1]) * qty if lv.index(level) > 0 else 0
                if profit > 0:
                    st["profitable_trades"] += 1
                st["total_profit"] += profit
                st["up_crossings"] += 1
                p_day += profit
                st["cash"] += level * qty
                net -= 1
        elif cur < last:
            for level in [lv_ for lv_ in lv if cur <= lv_ <= last]:
                st["down_crossings"] += 1
                st["cash"] -= level * qty
                net += 1
        last = cur
        nmax, nmin = max(nmax, net), min(nmin, net)
        if days is not None:
            day_profit[days[k]] = day_profit.get(days[k], 0.0) + p_day
        if k > 0 and k % rebalance_ticks == 0:
            st["n_rebalance_checks"] += 1
            if cur < lower * 1.05 or cur > upper * 0.95:
                lower = cur * (1 - lo_pct / 100)
                upper = cur * (1 + up_pct / 100)
                lv = levels(lower, upper, n_cur, kind)
                regens.append((k, lower, upper, n_cur))
        if k > 0 and k % adjust_ticks == 0:
            st["n_adjustments"] += 1
            if adapt and labels is not None and table and int(labels[k]) in table:
                n_cur, lo_pct, up_pct = table[int(labels[k])]
            total = st["up_crossings"] + st["down_crossings"]
            if total > 10:
                wr = st["profitable_trades"] / total
                if wr < 0.4:
                    n_cur = max(5, n_cur - 2)
                elif wr > 0.7:
                    n_cur = min(20, n_cur + 2)
        if days is not None and (k == T - 1 or days[k + 1] != days[k]):
            snaps.append((int(days[k]), k, st["up_crossings"] + st["down_crossings"], st["profitable_trades"],
                          st["total_profit"]))
    st.update(n_regenerations=len(regens) - 1, num_grids=n_cur, lower=lower, upper=upper, position=net * qty,
              max_position=nmax * qty, min_position=nmin * qty, near_ties=ties)
    out = _finish(st, T, bar_seconds, prices[-1])
    out.update(regenerations=regens, levels=lv, day_profit=day_profit, snapshots=snaps)
    return out


def simulate_fast(prices, lower: float, upper: float, n: int, kind: int, qty: float, lower_pct: float, upper_pct: float,
                  rebalance_ticks: int, adjust_ticks: int, adapt: bool = False, labels=None, table: Optional[Dict] = None,
                  bar_seconds: int = 60) -> Dict:
    """simulate() with NumPy over each run of ticks between two checks (no per-day output, no near-tie count)."""
    p = np.asarray(prices, dtype=np.float64)
    T = len(p)
    lv = np.array(levels(lower, upper, n, kind))
    n_cur, lo_pct, up_pct = n, lower_pct, upper_pct
    up = down = prof = 0
    profit = cash = 0.0
    net = nmax = nmin = 0
    n_regen = n_reb = n_adj = 0
    k = 1
    next_reb, next_adj = rebalance_ticks, adjust_ticks
    while k < T:
        stop = min(next_reb, next_adj, T - 1)
        last, cur = p[k - 1:stop], p[k:stop + 1]
        f = np.searchsorted(lv, lv, "left")     # levels.index: a repeated level earns the step under its first copy
        pl = np.where(f > 0, (lv - lv[np.maximum(f - 1, 0)]) * qty, 0.0)
        cum_p = np.concatenate([[0.0], np.cumsum(pl)])
        cum_w = np.concatenate([[0], np.cumsum(pl > 0)])
        cum_l = np.concatenate([[0.0], np.cumsum(lv * qty)])
        upm, dnm = cur > last, cur < last
        a = np.where(upm, np.searchsorted(lv, last, "left"), np.searchsorted(lv, cur, "left"))
        b = np.where(upm, np.searchsorted(lv, cur, "right"), np.searchsorted(lv, last, "right"))
        cnt = np.where(upm | dnm, np.maximum(b - a, 0), 0)
        a_, b_ = a, np.maximum(a, b)
        up += int(cnt[upm].sum())
        down += int(cnt[dnm].sum())
        prof += int((cum_w[b_] - cum_w[a_])[upm].sum())
        profit += float((cum_p[b_] - cum_p[a_])[upm].sum())
        cash += float((cum_l[b_] - cum_l[a_])[upm].sum() - (cum_l[b_] - cum_l[a_])[dnm].sum())
        dn = np.where(upm, -cnt, cnt)
        path = net + np.cumsum(dn)
        if len(path):
            nmax, nmin = max(nmax, int(path.max())), min(nmin, int(path.min()))
            net = int(path[-1])
        k = stop + 1
        c = float(p[stop])
        if stop == next_reb:
            n_reb += 1
            next_reb += rebalance_ticks
            if c < lower * 1.05 or c > upper * 0.95:
                lower, upper = c * (1 - lo_pct / 100), c * (1 + up_pct / 100)
                lv = np.array(levels(lower, upper, n_cur, kind))
                n_regen += 1
        if stop == next_adj:
            n_adj += 1
            next_adj += adjust_ticks
            if adapt and labels is not None and table and int(labels[stop]) in table:
                n_cur, lo_pct, up_pct = table[int(labels[stop])]
            if up + down > 10:
                wr = prof / (up + down)
                if wr < 0.4:
                    n_cur = max(5, n_cur - 2)
                elif wr > 0.7:
                    n_cur = min(20, n_cur + 2)
    st = {f: 0 for f in FIELDS}
    st.update(total_profit=profit, up_crossings=up, down_crossings=down, profitable_trades=prof, cash=cash,
              n_regenerations=n_regen, num_grids=n_cur, lower=lower, upper=upper, position=net * qty,
              max_position=nmax * qty, min_position=nmin * qty, n_rebalance_checks=n_reb, n_adjustments=n_adj)
    return _finish(st, T, bar_seconds, float(p[-1]))
