"""Generate the grid-trading fixture by EXECUTING the reference's own service loop.

Run where a copy of the reference tree exists (as for make_golden.py):

    python tests/golden/make_grid.py

Writes tests/golden/grid_reference.json.  services/grid_trading_strategy.py is imported with `binance`,
`binance.exceptions` and `redis` replaced by stubs, and GridTradingStrategy.run() (:122-233) runs unmodified, one service
instance per case with one symbol, in simulation mode:
  - a fake clock: datetime.now() and time.time() read the current tick's time (t0 + k bar lengths), asyncio.sleep()
    advances one tick and raises CancelledError after the last one, which run() catches;
  - the ticker serves the tick's bar close; get_historical_klines(1d, "<n> days ago UTC") serves the daily closes of
    the UTC days whose start is >= t0 - n days, each closed by its last bar at or before t0;
  - the Redis stub serves market_regime_history as [{"regime": <label of the tick's bar>}] (or nothing), and records
    every grid_config (initial grid and regenerations), every grid_profit and grid_performance write;
  - config.json is written to a temporary working directory.
Prices are float32 values (the engine's closes) on a price tick of 1/16 or 1/4, written as Python floats, so the file
stays small; only the first and the last grid of each case keep their levels.
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
OUT = Path(__file__).resolve().parent / "grid_reference.json"
MINUTE0 = 28_401_120          # 2024-01-01 00:00 UTC in minutes
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
    sys.modules["binance.exceptions"].BinanceAPIException = type("BinanceAPIException", (Exception,), {})
    import importlib
    return importlib.import_module("services.grid_trading_strategy")


def daily_closes(closes, minute0, bar_minutes, start_bar, lookback):
    t0 = minute0 + start_bar * bar_minutes
    lo = t0 - lookback * 1440
    out = []
    for d in range(-(-lo // 1440), t0 // 1440 + 1):
        b = (min(t0, (d + 1) * 1440 - 1) - minute0) // bar_minutes
        if b >= 0 and minute0 + b * bar_minutes >= d * 1440:
            out.append(closes[b])
    return out


def run_case(mod, case):
    closes, bm, start = case["closes"], case["bar_minutes"], case["start_bar"]
    T = len(closes) - start
    t0_s = (MINUTE0 + start * bm) * 60
    tick = {"k": 0}
    store, log = {}, {"configs": [], "profits": [], "performance": []}
    labels = case.get("labels")

    def set_clock():
        _Clock.now_s = t0_s + tick["k"] * bm * 60

    class Redis:
        def __init__(self, *a, **k):
            pass

        def set(self, key, value):
            store[key] = value
            if key.startswith("grid_config:"):
                g = json.loads(value)
                log["configs"].append({"tick": tick["k"], "lower": g["lower_boundary"], "upper": g["upper_boundary"],
                                       "levels": g["grid_levels"]})
            elif key.startswith("grid_profit:"):
                log["profits"].append((tick["k"], json.loads(value)))
            elif key == "grid_performance":
                log["performance"].append((tick["k"], json.loads(value)))

        def get(self, key):
            if key == "market_regime_history" and labels is not None:
                return json.dumps([{"regime": LABELS[labels[start + tick["k"]]]}])
            return None

        def publish(self, *a, **k):
            return 0

    class Client:
        KLINE_INTERVAL_1DAY = "1d"

        def __init__(self, *a, **k):
            pass

        def get_symbol_ticker(self, symbol):
            return {"symbol": symbol, "price": repr(closes[start + tick["k"]])}

        def get_exchange_info(self):
            return {"symbols": [{"symbol": case["symbol"], "filters": []}]}

        def get_historical_klines(self, symbol, interval, start_str):
            n = int(start_str.split()[0])
            return [[0, "0", "0", "0", repr(c)] for c in daily_closes(closes, MINUTE0, bm, start, n)]

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
    cfg = {"grid_trading": dict(case["config"], enabled=True, simulation_mode=True, symbols=[case["symbol"]],
                                notify_on_trade=True)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        Path("config.json").write_text(json.dumps(cfg))
        set_clock()
        svc = mod.GridTradingStrategy()
        asyncio.run(svc.run())
        os.chdir(cwd)
    days = [(MINUTE0 + (start + k) * bm) // 1440 for k in range(T)]
    snaps = []
    for k, gp in log["profits"]:
        if k == T - 1 or days[k + 1] != days[k]:
            snaps.append({"day": days[k], "tick": k, "total_trades": gp["total_trades"],
                          "profitable_trades": gp["profitable_trades"], "total_profit": gp["total_profit"]})
    perf = log["performance"][-1][1]
    return {
        "name": case["name"], "symbol": case["symbol"], "bar_minutes": bm, "minute0": MINUTE0, "start_bar": start,
        "closes": closes, "labels": labels, "config": case["config"],
        "regenerations": [dict({"tick": c["tick"], "lower": c["lower"], "upper": c["upper"], "n": len(c["levels"]) - 1},
                               **({"levels": c["levels"]} if j in (0, len(log["configs"]) - 1) else {}))
                          for j, c in enumerate(log["configs"])],
        "grid_profits": {k: v for k, v in svc.grid_profits[case["symbol"]].items() if k != "start_time"},
        "performance": {k: perf[k] for k in ("total_trades", "profitable_trades", "win_rate", "total_profit",
                                             "profit_per_day", "running_time_hours")},
        "final": {"num_grids": svc.num_grids, "lower_boundary_pct": svc.lower_boundary_pct,
                  "upper_boundary_pct": svc.upper_boundary_pct, "lower": svc.active_grids[case["symbol"]]["lower_boundary"],
                  "upper": svc.active_grids[case["symbol"]]["upper_boundary"]},
        "snapshots": snaps,
    }


def f32(x):
    return [float(v) for v in np.asarray(x, dtype=np.float32)]


def walk(rng, n, p0, vol, drift=0.0, tick=1 / 16):
    return f32(np.round(p0 * np.exp(np.cumsum(drift + vol * rng.standard_normal(n))) / tick) * tick)


def cases(rng):
    fixed = {"auto_boundaries": False, "lower_boundary_pct": 25.0, "upper_boundary_pct": 25.0, "num_grids": 8,
             "grid_type": "arithmetic", "rebalance_frequency": 3600, "auto_adjust_period": 86400,
             "adapt_to_market_regime": False, "quantity_per_grid": 0.5}
    out = []
    # exact levels: P0 = 1024, pct 25, n = 8 -> 768 .. 1280 step 64; hits, flat stretches, gaps of many levels
    path = [1024.0] * 5 + [1088.0, 1088.0, 1152.0, 1000.0, 768.0, 1280.0, 1280.0, 1216.0, 1024.0, 1024.0, 896.0, 1100.0]
    path += [float(v) for v in (1024 + 64 * np.round(rng.uniform(-3, 3, 400)) / 2)]
    out.append({"name": "arithmetic exact levels", "bar_minutes": 1, "start_bar": 0, "closes": f32(path),
                "config": dict(fixed)})
    # geometric exact levels: n = 2, pcts 50 / 100 -> 512, 1024, 2048
    gpath = [1024.0, 1024.0, 2048.0, 512.0, 1024.0, 1500.0, 700.0, 2048.0, 2100.0, 1024.0] * 8
    out.append({"name": "geometric exact levels", "bar_minutes": 1, "start_bar": 0, "closes": f32(gpath),
                "config": dict(fixed, grid_type="geometric", num_grids=2, lower_boundary_pct=50.0,
                               upper_boundary_pct=100.0, auto_adjust_period=100000000)})
    # random walks over a lookback: auto boundaries, both types, adjustment on / off, regimes
    N = 2 * 1440 + 2537
    base = walk(rng, N, 30000.0, 0.0012, tick=1 / 4)
    lab = [int(v) for v in np.repeat(rng.integers(0, 5, N // 240 + 1), 240)[:N]]
    cfg = dict(fixed, auto_boundaries=True, volatility_lookback=2, rebalance_frequency=3600, auto_adjust_period=7200,
               adapt_to_market_regime=True, num_grids=10, ranging_num_grids=15, volatile_num_grids=12,
               quantity_per_grid=0.01)
    out.append({"name": "auto arithmetic, regimes", "bar_minutes": 1, "start_bar": 2 * 1440 + 37, "closes": base,
                "labels": lab, "config": dict(cfg)})
    out.append({"name": "auto geometric, regimes", "bar_minutes": 1, "start_bar": 2 * 1440 + 37, "closes": base,
                "labels": lab, "config": dict(cfg, grid_type="geometric")})
    out.append({"name": "fixed, adjustment off", "bar_minutes": 1, "start_bar": 2 * 1440, "closes": base,
                "config": dict(cfg, auto_boundaries=False, lower_boundary_pct=2.0, upper_boundary_pct=3.0,
                               auto_adjust_period=10 ** 9, rebalance_frequency=1800.5)})
    # win rates: an up-trend (profitable crossings) and a down-trend (crossings without profit)
    upt = walk(rng, 2000, 100.0, 0.0008, 0.0004)
    dnt = walk(rng, 2000, 100.0, 0.0008, -0.0004)
    wr = dict(fixed, lower_boundary_pct=4.0, upper_boundary_pct=4.0, num_grids=12, auto_adjust_period=3600,
              rebalance_frequency=1500)
    out.append({"name": "win rate above 0.7", "bar_minutes": 1, "start_bar": 0, "closes": upt, "config": dict(wr)})
    out.append({"name": "win rate below 0.4", "bar_minutes": 1, "start_bar": 0, "closes": dnt,
                "config": dict(wr, grid_type="geometric")})
    # a 5-minute clock with a start after a 3-day lookback
    five = walk(rng, 3 * 288 + 1200, 2500.0, 0.003, tick=1 / 4)
    out.append({"name": "5-minute clock", "bar_minutes": 5, "start_bar": 3 * 288 + 11, "closes": five,
                "labels": [int(v) for v in np.repeat(rng.integers(0, 5, 200), 12)[:len(five)]],
                "config": dict(cfg, volatility_lookback=3, rebalance_frequency=3599, auto_adjust_period=14400)})
    for c in out:
        c["symbol"] = "BTCUSDC"
    return out


def main():
    mod = _load()
    import logging
    logging.disable(logging.CRITICAL)
    rng = np.random.default_rng(7)
    results = [run_case(mod, c) for c in cases(rng)]
    series, labels = {}, {}
    for r in results:                      # each distinct close / label series is stored once
        for key, table in (("closes", series), ("labels", labels)):
            if r[key] is not None:
                name = next((k for k, v in table.items() if v == r[key]), f"{key}{len(table)}")
                table[name] = r[key]
                r[key] = name
    for name, lab in labels.items():       # labels as runs [label, length]
        runs = []
        for v in lab:
            if runs and runs[-1][0] == v:
                runs[-1][1] += 1
            else:
                runs.append([v, 1])
        labels[name] = runs
    block = lambda d: "{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in d.items()) + "\n}"
    OUT.write_text('{"series": ' + block(series) + ',\n"label_runs": ' + block(labels) + ',\n"cases": [\n' +
                   ",\n".join(json.dumps(r) for r in results) + "\n]}\n")          # one series / case per line
    for r in results:
        print(f"{r['name']}: {r['grid_profits']['total_trades']} trades, {len(r['regenerations']) - 1} regenerations, "
              f"final num_grids {r['final']['num_grids']}")


if __name__ == "__main__":
    main()
