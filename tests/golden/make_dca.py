"""Generate the DCA fixture by EXECUTING the reference's own service loop.

Run where a copy of the reference tree exists (as for make_golden.py):

    python tests/golden/make_dca.py

Writes tests/golden/dca_reference.json.  services/dca_strategy.py is imported with `binance`, `binance.exceptions` and
`redis` replaced by stubs, and DCAStrategy.run() (:140-239) runs unmodified, one service instance per case, in simulation
mode:
  - a fake clock: datetime.now() and time.time() read the current tick's time (t0 + k bar lengths), asyncio.sleep()
    advances one tick and raises CancelledError after the last one, which run() catches;
  - the ticker serves the tick's bar close of the symbol; get_historical_klines(1d, "7 days ago UTC") serves the day highs
    of the UTC days whose start is >= now - 7 days, each the max high of its bars with start <= now; get_exchange_info
    serves a LOT_SIZE step per symbol (or no filter); get_account serves the case's USDC balance;
  - the Redis stub serves market_regime_history as [{"regime": <label of the tick's bar>}] (or nothing) and nothing else,
    and keeps the last dca_performance write;
  - config.json is written to a temporary working directory.
Prices and highs are float32 values on a 1/16 price tick, stored as integer ticks (closes as differences, highs as offsets
above the close) so that the file stays small; labels are stored as runs.
"""
from __future__ import annotations

import asyncio
import json
import os
import sys
import tempfile
import types
from datetime import datetime, timedelta
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
OUT = Path(__file__).resolve().parent / "dca_reference.json"
MINUTE0 = 28_401_120          # 2024-01-01 00:00 UTC (a Monday) in minutes, the first bar of every case but one
LABELS = ("bull", "bear", "ranging", "volatile", "unknown")
EPOCH = datetime(1970, 1, 1)


class _Clock:
    now_s = 0.0


class FakeDateTime(datetime):
    @classmethod
    def now(cls, tz=None):
        t = EPOCH + timedelta(seconds=_Clock.now_s)
        return cls(t.year, t.month, t.day, t.hour, t.minute, t.second, t.microsecond)


def _load():
    from oracle import ref_runner
    ref_runner._prepare()
    for name in ("binance", "binance.client", "binance.exceptions", "redis"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["binance.client"].Client = type("Client", (), {})
    sys.modules["binance.exceptions"].BinanceAPIException = type("BinanceAPIException", (Exception,), {})
    import importlib
    return importlib.import_module("services.dca_strategy")


def day_highs(high, minute0, bar_minutes, b):
    now = minute0 + b * bar_minutes
    lo = now - 7 * 1440
    out = []
    for d in range(-(-lo // 1440), now // 1440 + 1):
        first = max(0, -(-(d * 1440 - minute0) // bar_minutes))
        bars = [j for j in range(first, b + 1) if minute0 + j * bar_minutes < (d + 1) * 1440]
        if bars:
            out.append(max(high[j] for j in bars))
    return out


def run_case(mod, case):
    symbols, bm, start = case["symbols"], case["bar_minutes"], case["start_bar"]
    m0 = case.get("minute0", MINUTE0)
    closes, highs = case["closes"], case["highs"]
    N = len(closes[0])
    T = N - start
    t0_s = (m0 + start * bm) * 60
    tick = {"k": 0}
    labels = case.get("labels")
    perf = {}

    def set_clock():
        _Clock.now_s = t0_s + tick["k"] * bm * 60

    class Redis:
        def __init__(self, *a, **k):
            pass

        def set(self, key, value):
            if key == "dca_performance":
                perf["last"] = json.loads(value)

        def get(self, key):
            if key == "market_regime_history" and labels is not None:
                return json.dumps([{"regime": LABELS[labels[start + tick["k"]]]}])
            return None

        def hget(self, *a):
            return None

        def publish(self, *a, **k):
            return 0

        def lpush(self, *a):
            return 0

        def ltrim(self, *a):
            return True

    steps = case.get("steps") or [None] * len(symbols)

    class Client:
        KLINE_INTERVAL_1DAY = "1d"

        def __init__(self, *a, **k):
            pass

        def get_symbol_ticker(self, symbol):
            return {"symbol": symbol, "price": repr(closes[symbols.index(symbol)][start + tick["k"]])}

        def get_exchange_info(self):
            return {"symbols": [{"symbol": sym, "filters": [] if st is None else
                                 [{"filterType": "LOT_SIZE", "stepSize": st}]} for sym, st in zip(symbols, steps)]}

        def get_historical_klines(self, symbol, interval, start_str):
            assert start_str == "7 days ago UTC" and interval == "1d"
            h = highs[symbols.index(symbol)]
            return [[0, "0", repr(x), "0", "0"] for x in day_highs(h, m0, bm, start + tick["k"])]

        def get_account(self):
            return {"balances": [{"asset": "BTC", "free": "1.0"}, {"asset": "USDC", "free": repr(case["usdc"])}]}

    async def sleep(_):
        tick["k"] += 1
        if tick["k"] >= T:
            raise asyncio.CancelledError()
        set_clock()

    mod.redis = types.SimpleNamespace(Redis=Redis)
    mod.Client = Client
    mod.datetime = FakeDateTime
    mod.time = types.SimpleNamespace(time=lambda: _Clock.now_s)
    mod.asyncio = types.SimpleNamespace(sleep=sleep, CancelledError=asyncio.CancelledError)
    cfg = {"dca_strategy": dict(case["config"], enabled=True, simulation_mode=True, symbols=symbols)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        Path("config.json").write_text(json.dumps(cfg))
        set_clock()
        svc = mod.DCAStrategy()
        asyncio.run(svc.run())
        os.chdir(cwd)
    t0 = EPOCH + timedelta(seconds=t0_s)
    tick_of = lambda iso: int((datetime.fromisoformat(iso) - t0) / timedelta(minutes=bm))
    positions = {}
    for sym in symbols:
        p = svc.dca_positions[sym]
        positions[sym] = {k: v for k, v in p.items() if k not in ("purchases", "last_purchase_time", "symbol")}
        positions[sym]["last_purchase_tick"] = tick_of(p["last_purchase_time"]) if p["last_purchase_time"] else -1
        positions[sym]["purchases"] = [[tick_of(q["timestamp"]), q["type"], q["price"], q["quantity"], q["amount_usdc"]]
                                       for q in p["purchases"]]
    last = perf["last"]
    return {
        "name": case["name"], "symbols": symbols, "bar_minutes": bm, "minute0": m0, "start_bar": start,
        "closes": closes, "highs": highs, "labels": labels, "config": case["config"], "steps": case.get("steps"),
        "usdc": case["usdc"], "positions": positions,
        "next_scheduled_us": {sym: (svc.next_scheduled_buys[sym] - t0) // timedelta(microseconds=1) for sym in symbols},
        "last_dip_tick": {sym: tick_of(svc.dip_purchases[sym].isoformat()) if sym in svc.dip_purchases else -1
                          for sym in symbols},
        "service": {k: last[k] for k in ("total_purchases", "total_invested", "total_value", "total_profit",
                                         "total_profit_pct")},
        "service_total_invested": svc.total_invested,
    }


def f16(x):
    return [float(v) for v in np.asarray(np.round(np.asarray(x) * 16) / 16, dtype=np.float32)]


def ohlc(rng, n, p0, vol, drift=0.0):
    c = f16(p0 * np.exp(np.cumsum(drift + vol * rng.standard_normal(n))))
    h = f16(np.asarray(c) * (1 + np.abs(rng.normal(0, vol / 3, n))))
    return c, [max(a, b) for a, b in zip(c, h)]


def cases(rng):
    none = {"adaptive_scheduling": False, "price_dip_detection": False, "periodic_rebalancing": {"enabled": False},
            "interval_hours": 2.5, "base_order_size_usdc": 100, "min_order_size_usdc": 20, "max_order_size_usdc": 500}
    out = []
    c, h = ohlc(rng, 1440 + 17, 2000.0, 0.0005)
    out.append({"name": "fixed schedule", "bar_minutes": 1, "start_bar": 0, "bars": [(c, h)], "symbols": ["BTCUSDC"],
                "usdc": 0.0, "config": dict(none)})
    # every label; bear intervals and orders; crab never fires (the labeller says ranging)
    c, h = ohlc(rng, 6 * 96, 2000.0, 0.003)
    lab = [int(v) for v in np.repeat(rng.integers(0, 5, 6 * 24 + 1), 4)[:len(c)]]
    out.append({"name": "regime intervals", "bar_minutes": 15, "start_bar": 3, "bars": [(c, h)], "labels": lab,
                "symbols": ["ETHUSDC"], "usdc": 0.0,
                "config": dict(none, adaptive_scheduling=True, interval_hours=5,
                               scheduling_strategies={"market_regime_based": {
                                   "bull_interval_hours": 9, "bear_interval_hours": 2.5, "crab_interval_hours": 1,
                                   "volatile_interval_hours": 1.25}},
                               market_condition_rules={"increase_in_bear_market": True, "bear_market_adjustment": 1.7})})
    # weekend factor from a Thursday: 7.3 h * (1 + 0.2 * 0.37) has a sub-minute (and sub-second) remainder
    c, h = ohlc(rng, 5 * 96, 150.0, 0.004)
    out.append({"name": "weekend factor", "minute0": MINUTE0 + 3 * 1440, "bar_minutes": 15, "start_bar": 7,
                "bars": [(c, h)], "symbols": ["SOLUSDC"], "usdc": 0.0,
                "config": dict(none, adaptive_scheduling=True, interval_hours=7.3,
                               scheduling_strategies={"weighted_scheduling": {
                                   "enabled": True, "weight_factors": {"day_of_week": 0.37, "market_volatility": 0.4}}})})
    # dips: a saw-tooth whose troughs reach exactly 6.25 % below the 7-day high (1024 -> 960), from the first bar (< 2
    # klines on day one); cooldowns 0, 1 and 7 days
    n = 12 * 96
    base = 1024 - 64 * (0.5 + 0.5 * np.sin(np.arange(n) * 2 * np.pi / 113.0))
    c = f16(np.maximum(base + rng.normal(0, 1.5, n), 900))
    c = [960.0 if (j % 113 == 85) else v for j, v in enumerate(c)]
    h = [max(v, 1024.0 if j % 96 == 3 else v) for j, v in enumerate(c)]
    for cd in (0, 1, 7):
        out.append({"name": f"dips, cooldown {cd}", "bar_minutes": 15, "start_bar": 0, "bars": [(c, h)],
                    "symbols": ["BNBUSDC"], "usdc": 0.0,
                    "config": dict(none, interval_hours=24, price_dip_detection=True, dip_threshold_pct=6.25,
                                   additional_dip_allocation=0.75, max_dip_frequency_days=cd)})
    # clamps at both bounds, precision 0 through a 1e-05 step and precision 3
    out.append({"name": "clamps and precision", "bar_minutes": 60, "start_bar": 48,
                "bars": [ohlc(rng, 96, 3000.0, 0.01), ohlc(rng, 96, 12.0, 0.01)], "symbols": ["BTCUSDC", "LINKUSDC"],
                "steps": ["0.00001000", "0.00100000"], "usdc": 0.0,
                "config": dict(none, interval_hours=3, base_order_size_usdc=10, price_dip_detection=True,
                               dip_threshold_pct=1.0, additional_dip_allocation=60.0, max_dip_frequency_days=1)})
    # a 3-symbol service with symbol_settings (only the last keeps them) and rebalancing from a USDC balance
    bars = [ohlc(rng, 5 * 288, p0, 0.0025, d) for p0, d in ((4000.0, 0.0004), (250.0, -0.0004), (30.0, 0.0))]
    full = {"adaptive_scheduling": True, "interval_hours": 24, "base_order_size_usdc": 100, "min_order_size_usdc": 20,
            "max_order_size_usdc": 500, "price_dip_detection": True, "dip_threshold_pct": 3.0,
            "additional_dip_allocation": 0.5, "max_dip_frequency_days": 1,
            "scheduling_strategies": {"market_regime_based": {"bull_interval_hours": 18, "bear_interval_hours": 6,
                                                              "crab_interval_hours": 24, "volatile_interval_hours": 3},
                                      "weighted_scheduling": {"enabled": True, "weight_factors": {
                                          "day_of_week": 0.3, "market_volatility": 0.4, "social_sentiment": 0.3}}},
            "symbol_settings": [{"symbol": "BTCUSDC", "allocation": 0.6, "interval_hours": 24, "base_order_size_usdc": 150},
                                {"symbol": "ETHUSDC", "allocation": 0.3, "interval_hours": 48, "base_order_size_usdc": 80},
                                {"symbol": "BNBUSDC", "allocation": 0.1, "interval_hours": 72, "base_order_size_usdc": 50}],
            "periodic_rebalancing": {"enabled": True, "rebalance_interval_days": 2, "max_deviation_pct": 40.0},
            "market_condition_rules": {"increase_in_bear_market": True, "bear_market_adjustment": 1.5}}
    lab5 = [int(v) for v in np.repeat(rng.integers(0, 5, 5 * 288 // 36 + 1), 36)[:5 * 288]]
    out.append({"name": "3 symbols, rebalancing, 5-minute clock", "bar_minutes": 5, "start_bar": 288 + 5, "bars": bars,
                "labels": lab5, "symbols": ["BTCUSDC", "ETHUSDC", "BNBUSDC"], "usdc": 2000.0, "config": full})
    out.append({"name": "3 symbols, rebalancing every day", "bar_minutes": 5, "start_bar": 0, "bars": bars,
                "symbols": ["BTCUSDC", "ETHUSDC", "BNBUSDC"], "usdc": 750.5,
                "config": dict(full, periodic_rebalancing={"enabled": True, "rebalance_interval_days": 1,
                                                           "max_deviation_pct": 5.0})})
    for case in out:
        case["closes"] = [c for c, _ in case["bars"]]
        case["highs"] = [h for _, h in case["bars"]]
    return out


def encode(close, high):
    """A symbol's bars in 1/16 price ticks: the closes as first value and differences, the highs as offsets above them."""
    c = [int(round(v * 16)) for v in close]
    return {"close": c[:1] + [b - a for a, b in zip(c, c[1:])], "high": [int(round(h * 16)) - x for h, x in zip(high, c)]}


def main():
    mod = _load()
    import logging
    logging.disable(logging.CRITICAL)
    rng = np.random.default_rng(17)
    results = [run_case(mod, c) for c in cases(rng)]
    series, labels = {}, {}
    for r in results:                      # each distinct bar / label series is stored once
        names = []
        for c, h in zip(r.pop("closes"), r.pop("highs")):
            enc = encode(c, h)
            name = next((k for k, v in series.items() if v == enc), f"bars{len(series)}")
            series[name] = enc
            names.append(name)
        r["bars"] = names
        if r["labels"] is not None:
            name = next((k for k, v in labels.items() if v == r["labels"]), f"labels{len(labels)}")
            labels[name] = r["labels"]
            r["labels"] = name
    for name, lab in labels.items():       # labels as runs [label, length]
        runs = []
        for v in lab:
            if runs and runs[-1][0] == v:
                runs[-1][1] += 1
            else:
                runs.append([v, 1])
        labels[name] = runs
    block = lambda d: "{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}"
                                          for k, v in d.items()) + "\n}"
    OUT.write_text('{"series": ' + block(series) + ',\n"label_runs": ' + block(labels) + ',\n"cases": [\n' +
                   ",\n".join(json.dumps(r, separators=(',', ':')) for r in results) + "\n]}\n")
    for r in results:
        kinds = {}
        for p in r["positions"].values():
            for q in p["purchases"]:
                kinds[q[1]] = kinds.get(q[1], 0) + 1
        print(f"{r['name']}: {kinds}, total_profit_pct {r['service']['total_profit_pct']:.4f}")


if __name__ == "__main__":
    main()
