"""Generate the multi-symbol grid service fixture by EXECUTING the reference's own service loop.

Run where a copy of the reference tree exists (as for make_grid.py):

    python tests/golden/make_grid_service.py

Writes tests/golden/grid_service_reference.json.  As make_grid.py (whose stubs, fake clock and daily-close rule this
imports), but ONE GridTradingStrategy instance runs all of a case's symbols (config grid_trading.symbols), so num_grids and
the pcts are shared and every symbol's _adjust_grid_parameters mutates them.  The Redis stub records every grid_config write
as (tick, n) per symbol, the last one's boundaries, the service's (num_grids, lower_pct, upper_pct) at the writes where
they changed, and the last grid_profit of each symbol and grid_performance.  Closes are integer 1/16 price ticks (the
float32 closes are ticks / 16, exactly), stored as the first tick and then the differences.
"""
from __future__ import annotations

import asyncio
import json
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_grid  # noqa: E402

OUT = Path(__file__).resolve().parent / "grid_service_reference.json"
MINUTE0 = make_grid.MINUTE0
LABELS = make_grid.LABELS


def run_case(mod, case):
    syms, bm, start = case["symbols"], case["bar_minutes"], case["start_bar"]
    closes = {s: [t / 16 for t in case["ticks"][j]] for j, s in enumerate(syms)}
    T = len(closes[syms[0]]) - start
    t0_s = (MINUTE0 + start * bm) * 60
    tick = {"k": 0}
    log = {"regens": {}, "final_grid": {}, "service": [], "performance": None}
    labels = case.get("labels")
    holder = {}

    def set_clock():
        make_grid._Clock.now_s = t0_s + tick["k"] * bm * 60

    class Redis:
        def __init__(self, *a, **k):
            pass

        def set(self, key, value):
            if key.startswith("grid_config:"):
                g, svc, sym = json.loads(value), holder["svc"], key.split(":", 1)[1]
                log["regens"].setdefault(sym, []).append([tick["k"], len(g["grid_levels"]) - 1])
                log["final_grid"][sym] = [g["lower_boundary"], g["upper_boundary"]]
                values = [svc.num_grids, svc.lower_boundary_pct, svc.upper_boundary_pct]
                if not log["service"] or log["service"][-1][1:] != values:
                    log["service"].append([tick["k"]] + values)
            elif key == "grid_performance":
                log["performance"] = json.loads(value)

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
            return {"symbol": symbol, "price": repr(closes[symbol][start + tick["k"]])}

        def get_exchange_info(self):
            return {"symbols": [{"symbol": s, "filters": []} for s in syms]}

        def get_historical_klines(self, symbol, interval, start_str):
            n = int(start_str.split()[0])
            return [[0, "0", "0", "0", repr(c)] for c in make_grid.daily_closes(closes[symbol], MINUTE0, bm, start, n)]

    async def sleep(_):
        tick["k"] += 1
        if tick["k"] >= T:
            raise asyncio.CancelledError()
        set_clock()

    mod.redis = types.SimpleNamespace(Redis=Redis)
    mod.Client = Client
    mod.datetime = make_grid.FakeDateTime
    mod.time = types.SimpleNamespace(time=lambda: make_grid._Clock.now_s)
    mod.asyncio = types.SimpleNamespace(sleep=sleep, CancelledError=asyncio.CancelledError)
    cfg = {"grid_trading": dict(case["config"], enabled=True, simulation_mode=True, symbols=syms, notify_on_trade=True)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        Path("config.json").write_text(json.dumps(cfg))
        set_clock()
        svc = mod.GridTradingStrategy()
        holder["svc"] = svc
        asyncio.run(svc.run())
        os.chdir(cwd)
    perf = log["performance"]
    return {
        "name": case["name"], "symbols": syms, "bar_minutes": bm, "minute0": MINUTE0, "start_bar": start,
        "closes": case["ticks"], "labels": labels, "config": case["config"], "regenerations": log["regens"],
        "final_grid": log["final_grid"], "service": log["service"],
        "grid_profits": {s: {k: v for k, v in svc.grid_profits[s].items() if k in ("total_profit", "total_trades",
                                                                                   "profitable_trades")} for s in syms},
        "performance": {k: perf[k] for k in ("total_trades", "profitable_trades", "win_rate", "total_profit")},
        "final": {"num_grids": svc.num_grids, "lower_boundary_pct": svc.lower_boundary_pct,
                  "upper_boundary_pct": svc.upper_boundary_pct},
    }


def ticks(rng, n, p0, vol, drift=0.0):
    """A log-normal walk on the 1/16 price tick, as integer ticks."""
    return [int(v) for v in np.round(p0 * np.exp(np.cumsum(drift + vol * rng.standard_normal(n))) * 16)]


def cases(rng):
    from oracle import ref_runner
    block = json.loads((ref_runner.REFERENCE_ROOT / "config.json").read_text())["grid_trading"]
    block = {k: v for k, v in block.items() if k not in ("enabled", "simulation_mode", "symbols")}
    out = []
    # the config.json grid block as shipped on its three symbols: 60-minute bars after its 14-day lookback, regimes
    n60 = 14 * 24 + 96
    lab60 = [int(v) for v in np.repeat(rng.integers(0, 5, n60 // 12 + 1), 12)[:n60]]
    out.append({"name": "config.json as shipped, 60-minute clock", "symbols": ["BTCUSDC", "ETHUSDC", "BNBUSDC"],
                "bar_minutes": 60, "start_bar": 14 * 24 + 1, "labels": lab60, "config": block,
                "ticks": [ticks(rng, n60, 900, 0.006), ticks(rng, n60, 300, 0.008), ticks(rng, n60, 60, 0.007)]})
    fixed = {"auto_boundaries": False, "lower_boundary_pct": 1.0, "upper_boundary_pct": 1.0, "num_grids": 9,
             "grid_type": "arithmetic", "rebalance_frequency": 900, "auto_adjust_period": 1800,
             "adapt_to_market_regime": True, "quantity_per_grid": 0.1}
    # 1-minute series: rising, falling, driftless, and a flat one (<= 10 trades)
    n1 = 600
    up1, up2 = ticks(rng, n1, 100, 0.0008, 0.0004), ticks(rng, n1, 50, 0.0008, 0.0005)
    dn1, dn2 = ticks(rng, n1, 100, 0.0008, -0.0004), ticks(rng, n1, 80, 0.0008, -0.0004)
    mid, flat = ticks(rng, n1, 60, 0.001), [16 * 50] * n1
    flat[300:303] = [16 * 51, 16 * 52, 16 * 50]
    lab1 = [int(v) for v in np.repeat(rng.integers(0, 5, n1 // 60 + 1), 60)[:n1]]
    # the regime rule fires (ranging / volatile runs) and the last symbol's win rate decides; 5 symbols
    out.append({"name": "regime rule, last symbol decides", "symbols": ["BTCUSDC", "ETHUSDC", "BNBUSDC", "SOLUSDC",
                                                                        "XRPUSDC"],
                "bar_minutes": 1, "start_bar": 0, "labels": lab1, "config": dict(fixed),
                "ticks": [up1, dn1, mid, flat, up2]})
    # no regime source: the +-2 steps of the symbols add up to the clamps (rising pair -> 20, falling pair -> 5)
    out.append({"name": "no regime source, steps add up to 20", "symbols": ["BTCUSDC", "ETHUSDC"], "bar_minutes": 1,
                "start_bar": 0, "labels": None, "config": dict(fixed, num_grids=6), "ticks": [up1, up2]})
    out.append({"name": "no regime source, steps add down to 5", "symbols": ["BTCUSDC", "ETHUSDC"], "bar_minutes": 1,
                "start_bar": 0, "labels": None, "config": dict(fixed, num_grids=16), "ticks": [dn1, dn2]})
    # geometric grids with auto_boundaries after a 1-day lookback, 5-minute clock
    n5 = 288 + 360
    lab5 = [int(v) for v in np.repeat(rng.integers(0, 5, n5 // 24 + 1), 24)[:n5]]
    g5 = [ticks(rng, n5, 900, 0.003, 0.0003), ticks(rng, n5, 200, 0.004, -0.0003), ticks(rng, n5, 30, 0.003)]
    auto = dict(fixed, auto_boundaries=True, volatility_lookback=1, grid_type="geometric", rebalance_frequency=3600,
                auto_adjust_period=7200, num_grids=10)
    out.append({"name": "geometric, auto boundaries, 5-minute clock", "symbols": ["BTCUSDC", "ETHUSDC", "BNBUSDC"],
                "bar_minutes": 5, "start_bar": 288 + 7, "labels": lab5, "config": auto, "ticks": g5})
    # an adjust period shorter than the rebalance period, arithmetic auto boundaries, 5-minute clock
    out.append({"name": "adjust shorter than rebalance, 5-minute clock", "symbols": ["BTCUSDC", "ETHUSDC"],
                "bar_minutes": 5, "start_bar": 288 + 3, "labels": lab5,
                "config": dict(auto, grid_type="arithmetic", rebalance_frequency=5400, auto_adjust_period=1200),
                "ticks": g5[:2]})
    return out


def main():
    mod = make_grid._load()
    import logging
    logging.disable(logging.CRITICAL)
    rng = np.random.default_rng(11)
    results = [run_case(mod, c) for c in cases(rng)]
    series, labels = {}, {}
    for r in results:                      # each distinct tick / label series is stored once
        names = []
        for row in r["closes"]:
            name = next((k for k, v in series.items() if v == row), f"ticks{len(series)}")
            series[name] = row
            names.append(name)
        r["closes"] = names
        if r["labels"] is not None:
            name = next((k for k, v in labels.items() if v == r["labels"]), f"labels{len(labels)}")
            labels[name] = r["labels"]
            r["labels"] = name
    for name, row in series.items():       # ticks as the first one and the differences
        series[name] = row[:1] + [b - a for a, b in zip(row, row[1:])]
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
                   ",\n".join(json.dumps(r) for r in results) + "\n]}\n")
    for r in results:
        print(f"{r['name']}: {r['performance']['total_trades']} trades, "
              f"{sum(len(v) for v in r['regenerations'].values())} grid_config writes, "
              f"final num_grids {r['final']['num_grids']}")


if __name__ == "__main__":
    main()
