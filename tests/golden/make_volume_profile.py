"""Generate the volume-profile fixture by EXECUTING the reference's own VolumeProfileAnalyzer.

Run where a copy of the reference tree exists (as for make_golden.py):

    python tests/golden/make_volume_profile.py

Writes tests/golden/volume_profile_reference.json.  services/utils/volume_profile_analyzer.py is loaded unmodified from
its file (without the services.utils package) with matplotlib stubbed, in a temporary working directory holding logs/
(oracle/ref_runner.py), and analyze_volume_profile, analyze_volume_delta and detect_volume_anomalies run on a fresh copy of each case's DataFrame (five-minute klines with a
datetime timestamp column, as the monitor's df_5m).  The dicts are stored without their timestamp and histogram.

Inputs are seeded and float32-exact: prices and volumes are integers of a 1/16 tick, stored as such.  `tie_at_cut` marks
the cases where the value area's last bin has the volume of a bin left out of it, so that the reference's (unstable,
platform-dependent) argsort decides value_area_low / value_area_high there.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
OUT = Path(__file__).resolve().parent / "volume_profile_reference.json"
TICK = 16
T0 = "2024-01-01 00:00:00"


def _walk(rng, W, spike=False):
    """(open, high, low, close, volume) in ticks: a random walk around 40 000 ticks (2 500), volume 1/16 .. ~100."""
    close = 40_000 + np.cumsum(rng.integers(-40, 41, W))
    open_ = np.concatenate([[close[0] - rng.integers(-20, 21)], close[:-1]])
    high = np.maximum(open_, close) + rng.integers(0, 30, W)
    low = np.minimum(open_, close) - rng.integers(0, 30, W)
    vol = rng.integers(1, 1600, W)
    if spike:
        vol[rng.random(W) < 0.08] *= 12
    return open_, high, low, close, vol


def cases():
    rng = np.random.default_rng(2024)
    out = []
    for W in (1, 5, 19, 20, 39, 40, 100, 300):
        for k, B in enumerate((20, 7)):
            out.append(dict(name=f"walk_{W}_{B}", num_bins=B, bars=_walk(rng, W, spike=True)))
    flat = np.full(20, 40_000)
    out.append(dict(name="flat", num_bins=20, bars=(flat, flat, flat, flat, rng.integers(1, 1600, 20))))
    o, h, l, c, v = _walk(rng, 20)
    h[7], l[7] = h.max() + 50, l.min() - 50                       # one candle spans every bin
    out.append(dict(name="one_candle_spans_all", num_bins=20, bars=(o, h, l, c, v)))
    o, h, l, c, v = _walk(rng, 100)
    v[:] = 800                                                    # constant volume: no anomalies, tied bins
    out.append(dict(name="constant_volume", num_bins=20, bars=(o, h, l, c, v)))
    o, h, l, c, v = _walk(rng, 60, spike=True)
    v[20:45] = 320                                                # a constant run inside the frame
    out.append(dict(name="constant_run", num_bins=20, bars=(o, h, l, c, v)))
    o, h, l, c, v = _walk(rng, 40)
    out.append(dict(name="sell_only", num_bins=20, bars=(c + 5, np.maximum(h, c + 5), l, c, v)))
    out.append(dict(name="zero_volume", num_bins=20, bars=(o, h, l, c, np.zeros(40, dtype=np.int64))))
    # a single-bin value area whose midpoint is the close: 0 / 0 in the relative position
    lo_, hi_ = np.array([1600, 1768, 1768, 1768, 1768]), np.array([1920, 1768, 1768, 1768, 1768])
    out.append(dict(name="close_on_single_bin_midpoint", num_bins=20,
                    bars=(lo_ * 0 + 1768, hi_, lo_, lo_ * 0 + 1768, np.array([1, 256, 256, 256, 256]))))
    # value-area cuts inside a group of equal bins: ten one-bin candles of equal volume
    for W, B in ((10, 20), (13, 16), (30, 20)):
        base = 40_000 + 64 * (np.arange(W) % 10)
        out.append(dict(name=f"tie_group_{W}_{B}", num_bins=B,
                        bars=(base, base + 1, base - 1, base, np.full(W, 160))))
    return out


def _frame(bars):
    import pandas as pd
    o, h, l, c, v = (np.asarray(x, dtype=np.float64) / TICK for x in bars)
    ts = pd.date_range(T0, periods=len(c), freq="5min")
    return pd.DataFrame({"timestamp": ts, "open": o, "high": h, "low": l, "close": c, "volume": v})


def _strip(d):
    return {k: v for k, v in d.items() if k not in ("timestamp", "histogram_base64")}


def tie_at_cut(volumes, pct):
    """The last bin the value area takes has the volume of a bin it leaves out."""
    v = np.asarray(volumes)
    order = np.argsort(v, kind="stable")[::-1]
    thr, cum = v.sum() * pct, 0.0
    for k, i in enumerate(order):
        cum += v[i]
        if cum >= thr:
            return bool(np.any(v[order[k + 1:]] == v[i]))
    return False


def main():
    from oracle import ref_runner
    ref_runner._prepare()
    import importlib.util
    import logging
    # loaded from its file: the services.utils package's __init__ imports the ML detectors, which this module does not use
    path = ref_runner.REFERENCE_ROOT / "services" / "utils" / "volume_profile_analyzer.py"
    spec = importlib.util.spec_from_file_location("volume_profile_analyzer", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    logging.getLogger().setLevel(logging.CRITICAL)
    out = []
    for case in cases():
        an = mod.VolumeProfileAnalyzer(num_bins=case["num_bins"])
        prof = _strip(an.analyze_volume_profile(_frame(case["bars"])))
        rec = dict(name=case["name"], num_bins=case["num_bins"], start=T0,
                   bars=[np.asarray(x, dtype=np.int64).tolist() for x in case["bars"]],
                   profile=prof, delta=_strip(an.analyze_volume_delta(_frame(case["bars"]))),
                   anomalies=_strip(an.detect_volume_anomalies(_frame(case["bars"]))),
                   tie_at_cut="volumes" in prof and tie_at_cut(prof["volumes"], 0.7))
        out.append(rec)
    OUT.write_text(json.dumps({"tick": TICK, "cases": out}, separators=(",", ":")) + "\n")
    print(f"wrote {OUT} ({len(out)} cases, {sum(c['tie_at_cut'] for c in out)} with a tie at the cut)")


if __name__ == "__main__":
    main()
