"""Plain Python restatement of the multi-symbol grid service (services/grid_trading_strategy.py run() :160-206 with
several symbols in simulation mode): one instance, num_grids and the boundary pcts shared by its symbols.  Built on
grid_ref's lane functions; the oracle of the GPU tests of b200bt_grid_service_sweep.

simulate_service   tick by tick: every symbol's crossings, then every symbol's rebalance check with the shared values,
                   then _adjust_grid_parameters for the symbols in order, each mutating the shared values (regime rule,
                   then that symbol's win-rate rule)
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import grid_ref

def fixture_series(fx: Dict, case: Dict):
    """(closes [S][N] as the engine's float32 values in Python floats, labels [N] or None) of a case of
    tests/golden/grid_service_reference.json: ticks stored as the first one and the differences, labels as runs."""
    closes = []
    for name in case["closes"]:
        t = np.cumsum(fx["series"][name])
        closes.append([float(v) for v in (t / 16).astype(np.float32)])
    labels = None
    if case["labels"]:
        labels = [v for v, n in fx["label_runs"][case["labels"]] for _ in range(n)]
    return closes, labels


SERVICE_FIELDS = ("total_profit", "total_trades", "profitable_trades", "win_rate", "profit_per_day", "num_grids",
                  "lower_pct", "upper_pct", "n_adjustments", "n_num_grids_changes", "min_num_grids", "max_num_grids")


def simulate_service(prices: Sequence[Sequence[float]], bounds: Sequence[Tuple[float, float]], n: int, kind: int,
                     qty: Sequence[float], lower_pct: float, upper_pct: float, rebalance_ticks: int, adjust_ticks: int,
                     adapt: bool = False, labels=None, table: Optional[Dict] = None, bar_seconds: int = 60,
                     days=None) -> Dict:
    """prices [S][T] tick prices; bounds [S] initial (lower, upper); labels: ONE per-tick label row (the service reads
    one market_regime_history key) or None; table {label: (num_grids, lower_pct, upper_pct)}; days: per-tick day index.
    Returns {"lanes": [S] grid_ref-shaped dicts (num_grids = the lane's final grid), "service": SERVICE_FIELDS,
    "adjustments": [(tick, num_grids, lower_pct, upper_pct after it)], "day_profit": {day: profit summed over symbols
    in order}}."""
    S, T = len(prices), len(prices[0])
    px = [[float(p) for p in row] for row in prices]
    lanes = []
    for s in range(S):
        lo, up = bounds[s]
        st = {f: 0 for f in grid_ref.FIELDS}
        st.update(total_profit=0.0, cash=0.0)
        lanes.append({"lower": lo, "upper": up, "n": n, "lv": grid_ref.levels(lo, up, n, kind), "st": st, "net": 0,
                      "nmax": 0, "nmin": 0, "ties": 0, "last": px[s][0], "regens": [(0, lo, up, n)], "day": {}})
    n_cur, lo_pct, up_pct = n, lower_pct, upper_pct
    n_adj = n_changed = 0
    n_min = n_max = n
    adjustments = []
    for k in range(T):
        for s, ln in enumerate(lanes):                      # _process_grid_simulation, symbols in order
            cur, last, lv, st = px[s][k], ln["last"], ln["lv"], ln["st"]
            p_day = 0.0
            if (cur > last or cur < last) and kind == 1 and (grid_ref._near(last, lv) or grid_ref._near(cur, lv)):
                ln["ties"] += 1
            if cur > last:
                for level in [x for x in lv if last <= x <= cur]:
                    profit = (level - lv[lv.index(level) - 1]) * qty[s] if lv.index(level) > 0 else 0
                    if profit > 0:
                        st["profitable_trades"] += 1
                    st["total_profit"] += profit
                    st["up_crossings"] += 1
                    p_day += profit
                    st["cash"] += level * qty[s]
                    ln["net"] -= 1
            elif cur < last:
                for level in [x for x in lv if cur <= x <= last]:
                    st["down_crossings"] += 1
                    st["cash"] -= level * qty[s]
                    ln["net"] += 1
            ln["last"] = cur
            ln["nmax"], ln["nmin"] = max(ln["nmax"], ln["net"]), min(ln["nmin"], ln["net"])
            if days is not None:
                ln["day"][days[k]] = ln["day"].get(days[k], 0.0) + p_day
        if k > 0 and k % rebalance_ticks == 0:              # _rebalance_grid with the shared values
            for s, ln in enumerate(lanes):
                ln["st"]["n_rebalance_checks"] += 1
                cur = px[s][k]
                if cur < ln["lower"] * 1.05 or cur > ln["upper"] * 0.95:
                    ln["lower"], ln["upper"] = cur * (1 - lo_pct / 100), cur * (1 + up_pct / 100)
                    ln["n"] = n_cur
                    ln["lv"] = grid_ref.levels(ln["lower"], ln["upper"], n_cur, kind)
                    ln["regens"].append((k, ln["lower"], ln["upper"], n_cur))
        if k > 0 and k % adjust_ticks == 0:                 # _adjust_grid_parameters, symbols in order
            n_adj += 1
            before = n_cur
            rule = table.get(int(labels[k])) if adapt and labels is not None and table else None
            for ln in lanes:
                if rule is not None:
                    n_cur, lo_pct, up_pct = rule
                    n_min, n_max = min(n_min, n_cur), max(n_max, n_cur)
                total = ln["st"]["up_crossings"] + ln["st"]["down_crossings"]
                if total > 10:
                    wr = ln["st"]["profitable_trades"] / total
                    if wr < 0.4:
                        n_cur = max(5, n_cur - 2)
                    elif wr > 0.7:
                        n_cur = min(20, n_cur + 2)
                    n_min, n_max = min(n_min, n_cur), max(n_max, n_cur)
            n_changed += n_cur != before
            adjustments.append((k, n_cur, lo_pct, up_pct))
    out: List[Dict] = []
    for s, ln in enumerate(lanes):
        st = ln["st"]
        st.update(n_regenerations=len(ln["regens"]) - 1, num_grids=ln["n"], lower=ln["lower"], upper=ln["upper"],
                  position=ln["net"] * qty[s], max_position=ln["nmax"] * qty[s], min_position=ln["nmin"] * qty[s],
                  near_ties=ln["ties"], n_adjustments=n_adj)
        r = grid_ref._finish(st, T, bar_seconds, px[s][-1])
        r.update(regenerations=ln["regens"], levels=ln["lv"], day_profit=ln["day"])
        out.append(r)
    total_profit = 0.0
    for r in out:
        total_profit += r["total_profit"]
    trades = sum(r["total_trades"] for r in out)
    prof = sum(r["profitable_trades"] for r in out)
    secs = (T - 1) * bar_seconds
    service = {"total_profit": total_profit, "total_trades": trades, "profitable_trades": prof,
               "win_rate": prof / trades if trades > 0 else 0.0,
               "profit_per_day": total_profit / (secs / 86400) if secs > 0 else 0.0,
               "num_grids": n_cur, "lower_pct": lo_pct, "upper_pct": up_pct, "n_adjustments": n_adj,
               "n_num_grids_changes": n_changed, "min_num_grids": n_min, "max_num_grids": n_max}
    day_profit: Dict[int, float] = {}
    for r in out:
        for d, v in r["day_profit"].items():
            day_profit[d] = day_profit.get(d, 0.0) + v
    return {"lanes": out, "service": service, "adjustments": adjustments, "day_profit": day_profit}
