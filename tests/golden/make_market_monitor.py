"""Generate the market-monitor fixture by EXECUTING the reference's own code.

Run where a copy of the reference tree exists (as for make_volume_profile.py):

    python tests/golden/make_market_monitor.py

Writes tests/golden/market_monitor_reference.json.  services/market_monitor_service.py is loaded unmodified from its file
with binance / redis / websockets / metrics / circuit-breaker stubs and oracle/ref_runner.py's `ta` shim, in a temporary
working directory holding logs/ (ref_runner._prepare).  Then:

* MarketMonitorService.calculate_technical_indicators(None, data) runs on frames cut from seeded 1-minute series:
  float32-exact integer ticks (1/16), resampled with origin="epoch" and cut by the completed-kline rule (the last W
  klines completed by the close of bar t on each clock).  Cases: W in {1, 13, 14, 15, 26, 27, 50, 100}, flat stretches,
  a rise without down moves, a series start off the 15-minute grid, and every trend class.
* services/utils/indicator_combinations.py's calculate_indicator_combinations runs on those updates and on crafted
  dicts: every branch boundary, NaN / +-inf / -0.0 in each field, avg_volume 0, present volume / ema_12 / ema_26
  (ema_26 = 0 included), a missing price_change_3m and missing required fields, and for every rounded output whose
  value is not confined to a few constants, inputs whose unrounded value makes Python's and NumPy's round(x, 4) disagree.
Stored compactly: the bars as close steps and high / low offsets (open is the previous close), the crafted dicts as
changes to BASE, and the combination results (updates first, then the crafted dicts) as the error dict, or per
combination None or its values in order.
"""
from __future__ import annotations

import json
import math
import sys
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
OUT = Path(__file__).resolve().parent / "market_monitor_reference.json"
TICK = 16
# outputs whose value is confined to a few constants (no midpoint can exist), or is np.tanh's own value (the kernel's
# tanh is CUDA's, so a midpoint there would test tanh, not the rounding route)
BASE = dict(rsi=55.0, rsi_3m=52.0, rsi_5m=51.0, stoch_k=60.0, macd=0.0002, macd_3m=0.0001, macd_5m=0.0001,
            williams_r=-40.0, bb_position=0.6, trend='uptrend', trend_strength=0.4, price_change_1m=0.3,
            price_change_3m=0.5, price_change_5m=0.7, price_change_15m=1.1, current_price=100.0, avg_volume=1e6)
NO_MIDPOINT = {"osc_agreement": "0, 2/3 or 1", "tsi_confidence": "0.5, 0.8 or 1.0",
               "reversal_probability": "sums of 0.25, 0.2, 0.15 capped at 0.95", "vwpm": "np.tanh's own value"}


def _series(rng, N, kind):
    """(open, high, low, close) ticks of N one-minute bars."""
    step = rng.integers(-30, 31, N)
    if kind == "up":
        step = np.abs(step) + 1
    elif kind == "down":
        step = -np.abs(step) - 1
    close = 40_000 + np.cumsum(step)
    if kind == "flat":
        close[:] = 40_000
    open_ = np.concatenate([[close[0]], close[:-1]])
    high = np.maximum(open_, close) + (0 if kind == "flat" else rng.integers(0, 20, N))
    low = np.minimum(open_, close) - (0 if kind == "flat" else rng.integers(0, 20, N))
    return open_, high, low, close


def series_cases():
    rng = np.random.default_rng(2025)
    cases = []
    for W in (1, 13, 14, 15, 26, 27, 50, 100):
        cases.append(dict(name=f"walk_{W}", W=W, minute0=28_401_120, kind="walk"))
    cases += [dict(name="up_30", W=30, minute0=28_401_120, kind="up"),
              dict(name="down_30", W=30, minute0=28_401_120, kind="down"),
              dict(name="flat_30", W=30, minute0=28_401_120, kind="flat"),
              dict(name="off_grid_27", W=27, minute0=28_401_127, kind="walk")]
    for c in cases:
        N = 5 * c["W"] + 20
        c["bars"] = _series(rng, N, c["kind"])
        first = next(t for t in range(N) if _valid(t, c["minute0"], c["W"]))
        c["picks"] = sorted({first - 1, first, first + 1, N - 1} - {-1})
    return cases


def _valid(t, minute0, W):
    from market_monitor_ref import completed_kline
    return t - W + 1 >= 0 and all(completed_kline(t, minute0, k) - W + 1 >= 0 for k in (3, 5)) and \
        completed_kline(t, minute0, 15) >= 0


def frames(bars, minute0, t, W):
    """The reference's data dict: DataFrames of the last W klines completed by the close of bar t on each clock."""
    import pandas as pd
    o, h, l, c = (np.asarray(x, dtype=np.float64)[:t + 1] / TICK for x in bars)
    idx = pd.to_datetime((minute0 + np.arange(t + 1)) * 60, unit="s")
    df = pd.DataFrame({"open": o, "high": h, "low": l, "close": c, "volume": 1.0}, index=idx)
    out = {}
    for k in (1, 3, 5, 15):
        r = df.resample(f"{k}min", origin="epoch", label="left", closed="left").agg(
            {"open": "first", "high": "max", "low": "min", "close": "last", "volume": "sum"}).dropna()
        end = pd.Timestamp((minute0 + t + 1) * 60, unit="s")
        r = r[r.index + pd.Timedelta(minutes=k) <= end]          # completed klines only
        out[f"data_{k}m"] = r.iloc[-W:].reset_index(names="timestamp")
    return out


def crafted():
    """Crafted market_update-like dicts."""
    base = BASE
    out = []
    fields = ('rsi', 'macd', 'stoch_k', 'williams_r', 'bb_position', 'price_change_1m', 'price_change_3m',
              'price_change_5m', 'trend_strength', 'rsi_3m', 'rsi_5m', 'avg_volume')
    bounds = dict(rsi=(30, 40, 50, 60, 70), williams_r=(-20, -50, -80), stoch_k=(20, 50, 80),
                  bb_position=(0.1, 0.2, 0.5, 0.8, 0.9), price_change_1m=(0.1, -0.1, 0.0),
                  price_change_5m=(1.0, -1.0, 0.0, 2.0), trend_strength=(0.3, 0.6, 1.0, 2.0),
                  price_change_3m=(2.0, 6.0), rsi_5m=(30, 50, 70), avg_volume=(0.0,), macd=(0.0, 0.0005, -0.0005, 0.001))
    trends = ('uptrend', 'downtrend', 'sideways')
    for trend in trends:                     # sideways reads rsi, bb_position and macd only through the same branches
        for f, vals in bounds.items():
            if trend != 'sideways' or f in ('rsi', 'bb_position', 'macd'):
                out += [dict(base, trend=trend, **{f: float(v)}) for v in vals]
    for i, f in enumerate(fields):
        out += [dict(base, trend=trends[(i + j) % 3], **{f: v}) for j, v in enumerate((math.nan, math.inf, -math.inf, -0.0))]
    for trend in ('uptrend', 'downtrend'):
        for rsi, will, stoch, bb, pc5 in ((80, -10, 90, 0.95, 1.5), (20, -90, 10, 0.05, -1.5), (75, -15, 70, 0.85, 2.0),
                                          (25, -85, 30, 0.15, -2.0), (45, -60, 40, 0.5, 0.5), (55, -40, 60, 0.5, -0.5)):
            for macd in (-0.002, 0.0001):
                out.append(dict(base, trend=trend, rsi=float(rsi), williams_r=float(will), stoch_k=float(stoch),
                                bb_position=bb, price_change_5m=pc5, price_change_1m=pc5 / 2, macd=macd,
                                price_change_3m=3 * pc5))
    for vol, avg in ((2e6, 1e6), (1.1e6, 1e6), (0.5e6, 1e6), (1e6, 0.0), (math.nan, 1e6), (1e6, math.inf)):
        for pc1 in (0.5, -0.5, 0.05):
            out.append(dict(base, volume=vol, avg_volume=avg, price_change_1m=pc1))
    d = dict(base)
    del d['avg_volume']
    out += [d, dict(d, volume=3.0)]
    for e12, e26 in ((101.0, 100.0), (99.0, 100.0), (110.0, 100.0), (90.0, 100.0), (100.0, 100.0), (1.0, 0.0),
                     (-1.0, 0.0), (0.0, 0.0), (None, 100.0), (100.0, None)):
        out.append(dict(base, ema_12=e12, ema_26=e26))
    d = dict(base)
    del d['price_change_3m']
    out.append(d)
    d = dict(base)
    del d['rsi_5m']
    out += [d, {k: v for k, v in d.items() if k != 'rsi_3m'}]
    for f in ('rsi', 'trend', 'price_change_5m', 'trend_strength'):
        out.append({k: v for k, v in base.items() if k != f})
    out += midpoints(base)
    return out


def _nudged(x, n):
    for _ in range(abs(n)):
        x = math.nextafter(x, math.inf if n > 0 else -math.inf)
    return x


def midpoints(base):
    """Dicts whose unrounded value of one output is a place where Python's and NumPy's round(x, 4) disagree."""
    from market_monitor_ref import combinations, roundings_disagree
    # (output, base dict, input varied, its value as a function of the target unrounded value v)
    up = dict(base, trend='uptrend', macd=0.0)
    plans = [
        ("trend_confirmation", dict(up), "trend_strength", lambda v: v / 0.6),
        ("momentum_trend_alignment", dict(up, rsi=60.0, macd=0.001, williams_r=-30.0), "trend_strength", lambda v: v),
        ("tma_score", dict(up), "trend_strength", lambda v: 2 * (v - 0.5)),
        ("volatility_adjusted_momentum", dict(up, price_change_1m=0.0, price_change_3m=0.0, price_change_5m=0.0,
                                              williams_r=-50.0), "rsi", lambda v: 50 + 50 * v * 3 / (0.5 + 0.5 / 3.0)),
        ("volatility_trend_score", dict(up, bb_position=0.5), "trend_strength", lambda v: v / 0.3),
        ("osc_strength", dict(up, williams_r=-10.0, stoch_k=50.0), "rsi", lambda v: 50 + 30 * (2 * v - 1)),
        ("stoch_rsi", dict(up), "rsi", lambda v: 30 + 40 * (v - 0.33) / 0.34),
        ("drsi_divergence", dict(up, rsi_5m=50.0), "rsi", lambda v: 50 + v),
        ("vpc_strength", dict(up, price_change_1m=0.5, avg_volume=1e6), "volume", lambda v: 1e6 * (0.8 + 0.4 * v)),
        ("tsi_strength", dict(up, rsi=50.0, bb_position=0.0), "trend_strength", lambda v: v / 0.4),
        ("regime_confidence", dict(up), "trend_strength", lambda v: v / 1.1),
        ("breakout_confirmation", dict(up, price_change_5m=1.5, bb_position=0.9), "rsi", lambda v: 50 + 30 * (2 * v - 1)),
        ("divergence_strength", dict(up, price_change_5m=0.5, macd=0.0), "rsi", lambda v: 50 * (1 - (2 * v - 1))),
    ]
    out = []
    rng = np.random.default_rng(7)
    for name, d0, field, inv in plans:
        found = 0
        for _ in range(4000):
            k = int(rng.integers(1000, 9000))
            v = (k + 0.5) / 1e4
            x0 = inv(v)
            for n in range(-6, 7):
                d = dict(d0, **{field: _nudged(x0, n)})
                raw = combinations(d, unrounded=True)
                if name in raw and roundings_disagree(raw[name]):
                    out.append(d)
                    found += 1
                    break
            if found:
                break
        assert found, f"no rounding-midpoint case found for {name}"
    return out


def coverage(dicts):
    """Every rounded output not in NO_MIDPOINT has a case whose unrounded value the two roundings disagree on."""
    from market_monitor_ref import combinations, roundings_disagree
    seen = set()
    for d in dicts:
        raw = combinations(d, unrounded=True)
        if 'error' in raw:
            continue
        seen |= {k for k, v in raw.items() if roundings_disagree(v)}
    names = set(combinations(crafted()[0], unrounded=True))
    missing = names - seen - set(NO_MIDPOINT)
    assert not missing, f"no rounding-midpoint case for {sorted(missing)}"
    return sorted(seen)


def leaves(result):
    """A combinations dict stored compactly: the error dict as it is, else per combination None or its values in order."""
    if 'error' in result:
        return result
    return [None if v is None else list(v.values()) if isinstance(v, dict) else [v] for v in result.values()]


def _load_monitor():
    from oracle import ref_runner
    ref_runner._prepare()
    ref_runner._install_ta_shim()
    import importlib.util
    import logging
    for name in ("websockets", "services.utils.metrics", "services.utils.circuit_breaker",
                 "services.utils.volume_profile_analyzer"):
        sys.modules[name] = types.ModuleType(name)
    m = sys.modules
    m["services.utils.metrics"].get_metrics = lambda *a, **k: None
    m["services.utils.metrics"].is_metrics_enabled = lambda: False
    cb = m["services.utils.circuit_breaker"]
    cb.circuit_breaker = cb.with_retry = cb.CircuitBreakerConfig = cb.get_circuit_breaker = lambda *a, **k: None
    cb.CircuitBreakerOpenException = Exception
    m["services.utils.volume_profile_analyzer"].VolumeProfileAnalyzer = object
    # indicator_combinations from its file (the services.utils package's __init__ imports the ML detectors)
    path = ref_runner.REFERENCE_ROOT / "services" / "utils" / "indicator_combinations.py"
    spec = importlib.util.spec_from_file_location("services.utils.indicator_combinations", path)
    ic = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ic)
    m["services.utils.indicator_combinations"] = ic
    if "services.utils" not in m:
        pkg = types.ModuleType("services.utils")
        pkg.__path__ = []
        m["services.utils"] = pkg
    path = ref_runner.REFERENCE_ROOT / "services" / "market_monitor_service.py"
    spec = importlib.util.spec_from_file_location("market_monitor_service", path)
    mms = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mms)
    logging.getLogger().setLevel(logging.CRITICAL)
    return mms.MarketMonitorService, ic.calculate_indicator_combinations


def _diff(d):
    """A crafted dict stored against BASE: the keys it sets to another value, and the BASE keys it lacks."""
    same = lambda a, b: a is b or (type(a) is type(b) and a == b and (not isinstance(a, float) or
                                                                     math.copysign(1, a) == math.copysign(1, b)))
    return {"set": {k: v for k, v in d.items() if k not in BASE or not same(v, BASE[k])},
            "drop": [k for k in BASE if k not in d]}


def main():
    svc, combine = _load_monitor()
    series = []
    updates = []
    for c in series_cases():
        o, h, l, close = (np.asarray(x, dtype=np.int64) for x in c["bars"])
        rec = dict(name=c["name"], W=c["W"], minute0=c["minute0"], close_steps=np.diff(close, prepend=0).tolist(),
                   high_over=(h - np.maximum(o, close)).tolist(), low_under=(np.minimum(o, close) - l).tolist(),
                   picks=c["picks"], snapshots=[])
        for t in c["picks"]:
            snap = None
            if _valid(t, c["minute0"], c["W"]):
                snap = svc.calculate_technical_indicators(None, frames(c["bars"], c["minute0"], t, c["W"]))
                assert snap is not None, (c["name"], t)
                updates.append(dict(snap, current_price=1.0, avg_volume=1e6))
            rec["snapshots"].append(snap)
        series.append(rec)
    trends = {u["trend"] for u in updates}
    assert trends == {"uptrend", "downtrend", "sideways"}, trends
    dicts = crafted()
    seen = coverage(updates + dicts)
    results = [leaves(combine(dict(d))) for d in updates + dicts]
    OUT.write_text(json.dumps({"tick": TICK, "series": series, "base": BASE, "crafted": [_diff(d) for d in dicts],
                               "combined": results, "no_midpoint": NO_MIDPOINT}, separators=(",", ":")) + "\n")
    print(f"wrote {OUT}: {len(series)} series ({len(updates)} updates), {len(dicts)} crafted dicts, midpoint cases "
          f"for {len(seen)} outputs")


if __name__ == "__main__":
    main()
