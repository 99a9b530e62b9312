"""ctypes wrapper + build recipe for oracle/sim_oracle.c.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
import subprocess
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
BUILD_DIR = _HERE / "_build"
LIB = BUILD_DIR / "libsim_oracle.so"


class Params(C.Structure):
    _fields_ = [("rsi_oversold", C.c_double), ("rsi_overbought", C.c_double), ("take_profit", C.c_double),
                ("stop_loss", C.c_double), ("position_size", C.c_double)]


class Config(C.Structure):
    _fields_ = [("initial_capital", C.c_double), ("minute0", C.c_int64), ("bar_minutes", C.c_int32),
                ("primary", C.c_int32), ("secondary_mask", C.c_int32), ("reserved", C.c_int32),
                ("gap_bar", C.c_int32), ("gap_minutes", C.c_int32)]


STATS_FIELDS = ("n_records", "n_wins", "n_losses", "total_profit", "total_loss", "net_profit", "max_drawdown",
                "sharpe_ratio", "n_days", "largest_profit", "largest_loss", "sum_duration_bars", "score",
                "win_rate", "profit_factor", "sortino_ratio", "n_negative_days", "downside_deviation", "mean_daily_pnl",
                "trade_hash")
STATS_DTYPE = np.dtype([(n, "<f8") for n in STATS_FIELDS[:-1]] + [("trade_hash", "<u8")])


def build(force: bool = False) -> Path:
    src = _HERE / "sim_oracle.c"
    if LIB.exists() and not force and LIB.stat().st_mtime >= src.stat().st_mtime:
        return LIB
    BUILD_DIR.mkdir(exist_ok=True)
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-o", str(LIB), str(src), "-lm"])
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.oracle_lane.restype = C.c_int
        _lib.oracle_lane.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(Params), C.POINTER(Config),
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        _lib.oracle_lanes.restype = C.c_int
        _lib.oracle_lanes.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.POINTER(Config),
                                      C.c_void_p]
    return _lib


def params_of(p: dict) -> Params:
    """Same float64 expressions as strategy_evaluation.py:762-774."""
    return Params(float(p.get("rsi_oversold", 30)), float(p.get("rsi_overbought", 70)),
                  p.get("take_profit", 3) / 100, p.get("stop_loss", 2) / 100,
                  10000 * (min(p.get("max_position_size", 5), 20) / 100))


_PRIMARY = {"sharpe_ratio": 0, "return_pct": 1, "profit_factor": 2, "win_rate": 3, "net_profit": 4, "total_trades": 5,
            "max_drawdown": 6, "total_profit": 7, "total_loss": 8, "largest_profit": 9, "largest_loss": 10,
            "average_profit": 11, "average_loss": 12}
_PRIMARY_ADV = {"sortino_ratio": 13, "expectancy": 14, "calmar_ratio": 15, "profit_per_day": 16, "recovery_factor": 17}


def config_of(minute0: int, bar_minutes: int = 1, goals: dict | None = None, initial_capital: float = 10000.0,
              gap_bar: int = 0, gap_minutes: int = 0, advanced: bool = False) -> Config:
    """`advanced`: score on calculate_advanced_metrics' dict (strategy_evaluation.py:545-557) instead of the plain one."""
    goals = goals or {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"]}
    table = dict(_PRIMARY, **_PRIMARY_ADV) if advanced else _PRIMARY
    prim = table.get(goals.get("primary", "sharpe_ratio"), 99)          # metrics.get(primary, 0)
    secs = {"max_drawdown": 1, "win_rate": 2, "profit_factor": 4}
    if advanced:
        secs["expectancy"] = 8
    sec = 0
    for m in goals.get("secondary", []):
        sec |= secs.get(m, 0)
    return Config(float(initial_capital), int(minute0), int(bar_minutes), prim, sec, 0, int(gap_bar), int(gap_minutes))


def lane(price32: np.ndarray, rsi32: np.ndarray, p: dict, cfg: Config, event_cap: int = 0):
    """-> (stats record, events uint32[<=cap] or None, pnl float64[<=cap] or None)."""
    price32 = np.ascontiguousarray(price32, dtype=np.float32)
    rsi32 = np.ascontiguousarray(rsi32, dtype=np.float32)
    assert price32.shape == rsi32.shape and price32.ndim == 1
    out = np.zeros(1, dtype=STATS_DTYPE)
    ev = np.zeros(event_cap, dtype=np.uint32) if event_cap else None
    pn = np.zeros(event_cap, dtype=np.float64) if event_cap else None
    prm = params_of(p)
    lib().oracle_lane(price32.ctypes.data, rsi32.ctypes.data, len(price32), C.byref(prm), C.byref(cfg),
                      out.ctypes.data, ev.ctypes.data if event_cap else None,
                      pn.ctypes.data if event_cap else None, event_cap)
    n = int(out["n_records"][0])
    if event_cap:
        ev, pn = ev[:min(n, event_cap)], pn[:min(n, event_cap)]
    return out[0], ev, pn


def lanes(price32: np.ndarray, rsi32: np.ndarray, plist: list, cfg: Config) -> np.ndarray:
    price32 = np.ascontiguousarray(price32, dtype=np.float32)
    rsi32 = np.ascontiguousarray(rsi32, dtype=np.float32)
    arr = (Params * len(plist))(*[params_of(p) for p in plist])
    out = np.zeros(len(plist), dtype=STATS_DTYPE)
    lib().oracle_lanes(price32.ctypes.data, rsi32.ctypes.data, len(price32), arr, len(plist), C.byref(cfg),
                       out.ctypes.data)
    return out


def population(close: np.ndarray, bank: np.ndarray, row_of, population: list, cfg: Config, event_cap: int = 0,
               workers: int | None = None):
    """`lane` on every (individual, symbol) of `population`, on the host fp32 rows a sweep reads: close [S][N], RSI bank
    [S][R][N].  `row_of`: {rsi_period: bank row} (an individual without the gene reads period 14) or a callable
    individual -> bank row.
    -> (stats STATS_DTYPE [pop][S], events, pnl): with event_cap > 0 events[i][s] / pnl[i][s] are the lane's first
    min(n_records, event_cap) event words / record pnl, else both are None.  `workers` > 1 runs the individuals in that
    many threads (ctypes releases the GIL); the results do not depend on it."""
    row = row_of if callable(row_of) else (lambda p: row_of[int(p.get("rsi_period", 14))])

    def one(p):
        r = row(p)
        # copies: a lane's slices would keep its whole event_cap buffers alive
        return [(st, np.array(ev), np.array(pn)) if event_cap else (st, None, None)
                for st, ev, pn in (lane(close[s], bank[s][r], p, cfg, event_cap) for s in range(len(close)))]

    if workers is not None and workers > 1:
        with ThreadPoolExecutor(max_workers=workers) as ex:
            out = list(ex.map(one, population))
    else:
        out = [one(p) for p in population]
    stats = np.zeros((len(population), len(close)), dtype=STATS_DTYPE)
    for i, lanes_i in enumerate(out):
        stats[i] = [st for st, _, _ in lanes_i]
    if not event_cap:
        return stats, None, None
    return stats, [[ev for _, ev, _ in lanes_i] for lanes_i in out], [[pn for _, _, pn in lanes_i] for lanes_i in out]


# The sweep-against-oracle check (DESIGN.md section 5): counts, days, durations and the trade hash exact, every float
# statistic to max(rtol |want|, atol).
EXACT_FIELDS = ("n_records", "n_wins", "n_losses", "n_days", "sum_duration_bars", "n_negative_days", "trade_hash")
CLOSE_FIELDS = tuple(f for f in STATS_FIELDS if f not in EXACT_FIELDS)


def _column(x, f: str) -> np.ndarray:
    """Field `f` of a STATS_DTYPE array, a mapping field -> array, or a sequence of dicts; trade_hash as uint64."""
    if isinstance(x, np.ndarray) or hasattr(x, "keys"):
        col = x[f]
    else:
        col = [d[f] for d in x]
    return np.asarray(col, dtype=np.uint64 if f == "trade_hash" else np.float64)


def assert_lanes(got, want, where: str, exact=EXACT_FIELDS, close=CLOSE_FIELDS, rtol: float = 1e-9,
                 atol: float = 1e-11) -> None:
    """Fields `exact` equal and fields `close` within max(rtol |want|, atol) (NaN equals NaN, an infinity must match in
    sign) between two sets of lanes or books: STATS_DTYPE arrays, mappings field -> array (lane_stats(),
    book_stats()) or sequences of dicts (tests/book_ref.book), of the same shape."""
    for f in exact + close:
        g, w = _column(got, f), _column(want, f)
        assert g.shape == w.shape, f"{where}: {f} has shape {g.shape}, want {w.shape}"
        if f in exact:
            bad = g != w
        else:
            with np.errstate(invalid="ignore"):
                near = np.isfinite(w) & (np.abs(g - w) <= np.maximum(rtol * np.abs(w), atol))
                bad = ~((g == w) | (np.isnan(g) & np.isnan(w)) | near)
        if bad.any():
            k = tuple(int(j) for j in np.argwhere(bad)[0])
            raise AssertionError(f"{where}: {f} differs in {int(bad.sum())} of {bad.size} lanes, first at {k}: "
                                 f"got {g[k]!r}, want {w[k]!r}")


def assert_events(events, want_events, where: str) -> None:
    """The first n_records event words of every lane: `events` [pop][S][cap] (PopulationSweep.events()) against the
    ragged want_events[i][s] of `population`."""
    for i, lanes_i in enumerate(want_events):
        for s, ev in enumerate(lanes_i):
            np.testing.assert_array_equal(events[i][s][:len(ev)], ev, err_msg=f"{where}: events of lane {(i, s)}")
