"""Plain Python / NumPy restatements of the DCA service's simulation loop (services/dca_strategy.py run() :140-239 in
simulation mode), pinned to tests/golden/dca_reference.json, which the reference's own run() wrote.  The oracle of the
GPU tests of b200bt_dca_dip_pct and b200bt_dca_sweep.

klines_high     the literal kline rule of _check_for_dips at one bar (the days, their highs, their count)
dip_series      the drop series of every bar from day highs (NumPy), equal to the literal rule
simulate_ticks  tick by tick, symbol by symbol, with the reference's datetime arithmetic and expressions; exact
simulate        the same rule jumping from event to event over the kernel's decoded tables (for 1M-bar series); exact

Both return {"stats": [S] dicts of the b200bt_dca_stats fields, "service": the service totals, "purchases": [S] lists of
(tick, kind, price, quantity, amount), "day": {calendar day: the change of sum_s (Q_s * c_s - I_s)}, "order_total": the
service's own total_invested (the orders, in purchase order)}.
"""
from __future__ import annotations

import math
from datetime import datetime, timedelta
from typing import Dict, List, Optional, Sequence

import numpy as np

EPOCH = datetime(1970, 1, 1)
KINDS = ("scheduled", "dip", "rebalance")
BEAR = 1


def fmix32(h: int) -> int:
    h &= 0xFFFFFFFF
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    h ^= h >> 16
    return h


def klines_high(high: Sequence[float], minute0: int, bar_minutes: int, b: int) -> List[float]:
    """The day highs get_historical_klines(1d, "7 days ago UTC") serves at bar b: the UTC days whose start is >= now - 7
    days and that hold a bar with start <= now, each the max high of those bars."""
    now = minute0 + b * bar_minutes
    lo = now - 7 * 1440
    out = []
    for d in range(-(-lo // 1440), now // 1440 + 1):
        bars = [j for j in range(max(0, -(-(d * 1440 - minute0) // bar_minutes)), b + 1)
                if d * 1440 <= minute0 + j * bar_minutes < (d + 1) * 1440]
        if bars:
            out.append(max(float(high[j]) for j in bars))
    return out


def dip_of(klines: List[float], price: float) -> float:
    """_check_for_dips' drop (:841-855), NaN where it makes no check."""
    if not klines or len(klines) < 2:
        return math.nan
    recent_high = float(max(klines))                 # a Python float: a 0 high raises, as in the reference
    try:
        return ((recent_high - price) / recent_high) * 100
    except ZeroDivisionError:
        return math.nan


def dip_series(high: np.ndarray, close: np.ndarray, minute0: int, bar_minutes: int) -> np.ndarray:
    """dip_of(klines_high(...)) at every bar of one symbol, from per-day prefix maxima."""
    N = len(close)
    minutes = minute0 + np.arange(N, dtype=np.int64) * bar_minutes
    day = minutes // 1440
    first = int(day[0])
    nd = int(day[-1]) - first + 1
    h = high.astype(np.float64)
    dmax = np.full(nd, -np.inf)
    np.maximum.at(dmax, day - first, h)
    pre = h.copy()                                   # prefix max within the day
    starts = np.r_[True, day[1:] != day[:-1]]
    out = np.empty(N)
    idx = np.flatnonzero(starts)
    for a, z in zip(idx, list(idx[1:]) + [N]):
        pre[a:z] = np.maximum.accumulate(h[a:z])
    for b in range(N):
        d = int(day[b]) - first
        lo_day = -(-(int(minutes[b]) - 7 * 1440) // 1440) - first
        prev = [dmax[j] for j in range(max(0, lo_day), d) if dmax[j] > -np.inf]
        kl = prev + [pre[b]]
        out[b] = dip_of(kl, float(close[b]))
    return out


def _label(labels, s, bar):
    if labels is None:
        return None
    row = labels[0] if len(labels) == 1 else labels[s]
    return int(row[bar])


def simulate_ticks(close: np.ndarray, high: np.ndarray, minute0: int, bar_minutes: int, start_bar: int, svc,
                   labels=None, precision: Optional[Sequence[int]] = None, usdc_balance: float = 0.0,
                   dip: Optional[np.ndarray] = None) -> Dict:
    """The loop tick by tick.  svc: dca.Service (the parameters as the reference reads them).  dip: the drop series
    [S][N] (default: the literal kline rule at every visited bar)."""
    S, N = close.shape
    symbols = svc.symbols
    precision = list(precision) if precision is not None else [6] * S
    T = N - start_bar
    t0 = EPOCH + timedelta(minutes=minute0 + start_bar * bar_minutes)
    now_of = lambda k: t0 + timedelta(minutes=k * bar_minutes)
    pos = [{"I": 0.0, "Q": 0.0, "avg": 0.0, "last_price": 0.0, "last_tick": -1, "cv": 0.0, "pl": 0.0, "pct": 0.0}
           for _ in range(S)]
    purchases = [[] for _ in range(S)]
    last_dip = {}
    order_total = 0
    counts = [dict(n_sched=0, n_dip=0, n_reb=0, n_zero=0, order=0.0, hash=0, min_day=math.inf) for _ in range(S)]
    # _initialize_dca_strategy: symbols_config is replaced per symbol, the first interval uses the symbol's own settings
    next_buy = []
    symbols_config = {}
    for s, sym in enumerate(symbols):
        symbols_config = {sym: svc.settings(sym)}
        h = symbols_config[sym]["interval_hours"]
        next_buy.append(t0 + timedelta(hours=svc.interval_hours_at(h, _label(labels, s, start_bar), t0.weekday())))
    conf = lambda sym: symbols_config.get(sym, {})
    last_rebalance = t0 - timedelta(days=svc.rebalance_interval_days)
    n_checks = 0
    days = {}
    v_prev = [0.0] * S

    def purchase(s, k, kind, order, price):
        nonlocal order_total
        quantity = order / price
        factor = 10 ** precision[s]
        q = math.floor(quantity * factor) / factor
        p = pos[s]
        amount = price * q
        new_i = p["I"] + amount
        new_q = p["Q"] + q
        p.update(I=new_i, Q=new_q, avg=new_i / new_q if new_q > 0 else 0, last_price=price, last_tick=k,
                 cv=new_q * price, pl=new_q * price - new_i, pct=((new_q * price - new_i) / new_i) * 100 if new_i > 0 else 0.0)
        purchases[s].append((k, KINDS[kind], price, q, amount))
        c = counts[s]
        c["hash"] ^= fmix32(4 * k + kind)
        if q == 0:
            c["n_zero"] += 1
        if kind != 2:
            order_total += order
            c["order"] += order

    def order_of(s, k, dip_buy):
        sym = symbols[s]
        base = conf(sym).get("base_order_size_usdc", svc.base_order_size_usdc)
        return svc.order_size(base, dip_buy, _label(labels, s, start_bar + k) == BEAR)

    for k in range(T):
        now = now_of(k)
        bar = start_bar + k
        for s, sym in enumerate(symbols):                                       # _process_dca
            price = float(close[s, bar])
            p = pos[s]
            p["cv"] = p["Q"] * price
            if p["I"] > 0:
                p["pl"] = p["cv"] - p["I"]
                p["pct"] = (p["pl"] / p["I"]) * 100
            if now >= next_buy[s]:
                purchase(s, k, 0, order_of(s, k, False), price)
                counts[s]["n_sched"] += 1
                h = conf(sym).get("interval_hours", svc.interval_hours)
                next_buy[s] = now + timedelta(hours=svc.interval_hours_at(h, _label(labels, s, bar), now.weekday()))
        if svc.periodic_rebalancing and (now - last_rebalance).days >= svc.rebalance_interval_days:
            n_checks += 1
            total_value = 0.0
            for s in range(S):
                total_value += pos[s]["cv"]
            total_value += usdc_balance
            actions = []
            for s, sym in enumerate(symbols):
                current_alloc = pos[s]["cv"] / total_value if total_value > 0 else 0
                target_alloc = conf(sym).get("allocation", 1.0 / len(symbols))
                deviation_pct = abs((current_alloc - target_alloc) / target_alloc) * 100 if target_alloc > 0 else 0
                if deviation_pct > svc.max_deviation_pct:
                    target_value = total_value * target_alloc
                    if pos[s]["cv"] < target_value:
                        actions.append((s, target_value - pos[s]["cv"]))
            for s, buy_value in actions:
                purchase(s, k, 2, buy_value, float(close[s, bar]))
                counts[s]["n_reb"] += 1
            last_rebalance = now
        if svc.price_dip_detection:                                             # _check_for_dips
            for s, sym in enumerate(symbols):
                if s in last_dip and (now - last_dip[s]).days < svc.max_dip_frequency_days:
                    continue
                price = float(close[s, bar])
                drop = float(dip[s, bar]) if dip is not None else dip_of(
                    klines_high(high[s], minute0, bar_minutes, bar), price)
                if drop >= svc.dip_threshold_pct:
                    purchase(s, k, 1, order_of(s, k, True), price)
                    counts[s]["n_dip"] += 1
                    last_dip[s] = now
        for s in range(S):                                                      # _update_performance_metrics
            price = float(close[s, bar])
            p = pos[s]
            p["cv"] = p["Q"] * price
            if p["I"] > 0:
                p["pl"] = p["cv"] - p["I"]
                p["pct"] = (p["pl"] / p["I"]) * 100
        day = (minute0 + bar * bar_minutes) // 1440
        if k == T - 1 or (minute0 + (bar + 1) * bar_minutes) // 1440 != day:      # the day's last tick
            acc = 0.0
            for s in range(S):
                v = pos[s]["Q"] * float(close[s, bar]) - pos[s]["I"]
                counts[s]["min_day"] = min(counts[s]["min_day"], v)
                acc = acc + (v - v_prev[s])
                v_prev[s] = v
            days[day] = acc
    stats = []
    for s in range(S):
        p, c = pos[s], counts[s]
        stats.append({
            "total_invested": p["I"], "total_quantity": p["Q"], "average_price": float(p["avg"]),
            "current_value": p["cv"], "profit_loss": p["pl"], "profit_loss_pct": p["pct"],
            "n_scheduled": c["n_sched"], "n_dip": c["n_dip"], "n_rebalance": c["n_reb"], "order_usdc": float(c["order"]),
            "last_purchase_price": p["last_price"], "last_purchase_tick": p["last_tick"],
            "next_scheduled_us": (next_buy[s] - t0) // timedelta(microseconds=1),
            "last_dip_tick": int((last_dip[s] - t0) / timedelta(minutes=bar_minutes)) if s in last_dip else -1,
            "n_zero_quantity": c["n_zero"], "n_rebalance_checks": n_checks, "min_day_profit_loss": c["min_day"],
            "purchase_hash": c["hash"], "n_ticks": T, "reserved": 0.0,
        })
    return {"stats": stats, "service": service_of(stats), "purchases": purchases, "day": days,
            "order_total": order_total}


def service_of(stats: List[Dict]) -> Dict:
    """_update_performance_metrics' totals (:1047-1056), symbols in order."""
    total_invested = 0.0
    total_value = 0.0
    for st in stats:
        total_invested += st["total_invested"]
        total_value += st["current_value"]
    total_profit = total_value - total_invested
    return {"total_purchases": sum(st["n_scheduled"] + st["n_dip"] for st in stats), "total_invested": total_invested,
            "total_value": total_value, "total_profit": total_profit,
            "total_profit_pct": (total_profit / total_invested) * 100 if total_invested > 0 else 0.0}


def simulate(close: np.ndarray, dip: np.ndarray, minute0: int, bar_minutes: int, start_bar: int, decoded: Dict,
             labels=None, precision: Optional[Sequence[int]] = None, usdc_balance: float = 0.0) -> Dict:
    """The same rule from event to event over the kernel's tables (dca.decode_individual's dict): per symbol the next
    scheduled tick, the next dip tick (np.flatnonzero over the drop series) and the next rebalance tick; day ends only
    where a day's value is needed."""
    S, N = close.shape
    T = N - start_bar
    iv = decoded["individual"]
    first_us = decoded["first_us"]
    target = decoded["target"]
    precision = list(precision) if precision is not None else [6] * S
    pw = [float(10 ** p) for p in precision]
    tick_us = bar_minutes * 60_000_000
    minutes = minute0 + (start_bar + np.arange(T, dtype=np.int64)) * bar_minutes
    weekend = ((minutes // 1440 + 3) % 7 >= 5).astype(np.int64)
    dayv = minutes // 1440
    day_end = np.flatnonzero(np.r_[dayv[1:] != dayv[:-1], True])
    lab = np.full((S, T), 4, dtype=np.int64)
    if labels is not None:
        for s in range(S):
            row = np.asarray(labels[0] if len(labels) == 1 else labels[s])[start_bar:].astype(np.int64)
            lab[s] = np.where(row < 5, row, 4)
    flags = iv.flags
    cool = iv.dip_cooldown_minutes
    cool_ticks = 1 if cool <= 0 else max(1, -(-cool // bar_minutes))
    st = []
    purchases = [[] for _ in range(S)]
    for s in range(S):
        last = int(s == S - 1)
        L = dict(Q=0.0, I=0.0, order=0.0, last_price=0.0, last_tick=-1, last_dip=-1, n_sched=0, n_dip=0, n_reb=0,
                 n_zero=0, hash=0, min_day=math.inf)
        L["next_us"] = int(first_us[s][lab[s, 0]][weekend[0]])
        L["ks"] = 0 if L["next_us"] <= 0 else -(-L["next_us"] // tick_us)
        hits = np.flatnonzero(dip[s, start_bar:] >= iv.dip_threshold_pct) if flags & 1 else np.zeros(0, np.int64)
        L["hits"] = hits
        L["kd"] = int(hits[0]) if len(hits) else T
        st.append(L)

    def buy(s, k, kind, order):
        L = st[s]
        p = float(close[s, start_bar + k])
        q = math.floor(order / p * pw[s]) / pw[s]
        amount = p * q
        L["I"] = L["I"] + amount
        L["Q"] = L["Q"] + q
        L["last_price"], L["last_tick"] = p, k
        L["hash"] ^= fmix32(4 * k + kind)
        L["n_zero"] += q == 0.0
        purchases[s].append((k, KINDS[kind], p, q, amount))

    def advance(s, stop, upto_sched):
        """every event of symbol s before tick stop (and the scheduled one at stop when upto_sched)"""
        L = st[s]
        last = int(s == S - 1)
        while True:
            k = min(L["ks"], L["kd"])
            if k > stop or (k == stop and not (upto_sched and L["ks"] == stop)):
                break
            if L["ks"] == k:
                order = iv.order[last][0][int(lab[s, k] == BEAR)]
                buy(s, k, 0, order)
                L["order"] = L["order"] + order
                L["n_sched"] += 1
                now = k * tick_us
                L["next_us"] = now + iv.later_us[last][lab[s, k]][weekend[k]]
                L["ks"] = k + 1 if L["next_us"] <= now else max(k + 1, -(-L["next_us"] // tick_us))
            if k == stop:
                break
            if L["kd"] == k:
                dip_buy(s, k)

    def dip_buy(s, k):
        L = st[s]
        last = int(s == S - 1)
        order = iv.order[last][1][int(lab[s, k] == BEAR)]
        buy(s, k, 1, order)
        L["order"] = L["order"] + order
        L["n_dip"] += 1
        L["last_dip"] = k
        hits = L["hits"]
        j = np.searchsorted(hits, k + cool_ticks)
        L["kd"] = int(hits[j]) if j < len(hits) else T

    reb = bool(flags & 2)
    reb_ticks = range(iv.rebalance_first, T, iv.rebalance_period) if reb else range(0)
    stops = sorted(set(day_end.tolist()) | set(reb_ticks))
    reb_set = set(reb_ticks)
    end_set = set(day_end.tolist())
    v_prev = [0.0] * S
    days = {}
    n_checks = 0
    for k in stops:
        for s in range(S):
            advance(s, k, True)
        if k in reb_set:
            n_checks += 1
            v = [st[s]["Q"] * float(close[s, start_bar + k]) for s in range(S)]
            total = 0.0
            for x in v:
                total += x
            total += usdc_balance
            actions = []
            for s in range(S):
                alloc = v[s] / total if total > 0 else 0.0
                t = float(target[s])
                dev = abs((alloc - t) / t) * 100 if t > 0 else 0.0
                if dev > iv.max_deviation_pct and v[s] < total * t:
                    actions.append((s, total * t - v[s]))
            for s, b in actions:
                buy(s, k, 2, b)
                st[s]["n_reb"] += 1
        for s in range(S):
            if st[s]["kd"] == k:
                dip_buy(s, k)
        if k in end_set:
            acc = 0.0
            for s in range(S):
                val = st[s]["Q"] * float(close[s, start_bar + k]) - st[s]["I"]
                st[s]["min_day"] = min(st[s]["min_day"], val)
                acc = acc + (val - v_prev[s])
                v_prev[s] = val
            days[int(dayv[k])] = acc
    stats = []
    for s in range(S):
        L = st[s]
        cv = L["Q"] * float(close[s, N - 1])
        I = L["I"]
        pl = cv - I if I > 0 else 0.0
        stats.append({
            "total_invested": I, "total_quantity": L["Q"], "average_price": I / L["Q"] if L["Q"] > 0 else 0.0,
            "current_value": cv, "profit_loss": pl, "profit_loss_pct": (pl / I) * 100 if I > 0 else 0.0,
            "n_scheduled": L["n_sched"], "n_dip": L["n_dip"], "n_rebalance": L["n_reb"], "order_usdc": L["order"],
            "last_purchase_price": L["last_price"], "last_purchase_tick": L["last_tick"], "next_scheduled_us": L["next_us"],
            "last_dip_tick": L["last_dip"], "n_zero_quantity": L["n_zero"], "n_rebalance_checks": n_checks,
            "min_day_profit_loss": L["min_day"], "purchase_hash": L["hash"], "n_ticks": T, "reserved": 0.0,
        })
    return {"stats": stats, "service": service_of(stats), "purchases": purchases, "day": days}
