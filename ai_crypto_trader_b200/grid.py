"""Grid trading on the GPU engine: backtest a population of grid parameter sets over a market's bars, and evolve them.

Reference: services/grid_trading_strategy.py (GridTradingStrategy).  The reference evaluates a grid only in
"simulation mode": its live loop run() (:122-233) against the exchange ticker, once per update_interval, for as long as
one waits.  Here one (individual, symbol) lane is one symbol's service instance run over history by b200bt_grid_sweep
(csrc/grid.cu; the rule restated in include/b200bt.h and DESIGN.md section 3.13): a tick per bar, the bar's close as the
ticker price, the rebalance and adjustment checks on the ticks the reference's clock arithmetic gives them.  With
service=True one individual is instead ONE service instance trading all of the market's symbols, as the reference runs
one instance for its configured symbols (b200bt_grid_service_sweep): num_grids and the pcts are the instance's, and every
symbol's adjustment mutates them in symbol order.

    grid_param_ranges()      genes of the config keys the service reads (grid type as an index, booleans as 0 / 1)
    GridSweep                population fitness / stats / objectives / per-day profit rows on the device
    GridTradingStrategy      one parameter set on one symbol, in the reference's result shape

The initial boundaries are computed here on the host (the same NumPy expressions as _initialize_grid :266-289): fixed
pcts, or with auto_boundaries the volatility np.std(closes) / np.mean(closes) * 100 of the daily closes the reference
fetches with get_historical_klines(1d, "<lookback> days ago UTC"): the UTC days whose start is >= t0 - lookback days, each
closed by its last bar at or before t0 (the current day is partial).  "volatility_based" grids draw np.random and are
refused.
"""
from __future__ import annotations

import ctypes as C
import logging
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .population import StrategySweep, iso_minute

logger = logging.getLogger("b200bt.grid")

FIELDS = _lib.GRID_STATS_FIELDS
OBJECTIVE_FIELDS = FIELDS[:-1]          # near_ties describes the arithmetic, not the strategy
SERVICE_FIELDS = _lib.GRID_SERVICE_FIELDS
GRID_TYPES = _lib.GRID_TYPES
MAX_TICKS = (1 << 31) - 1

# GridTradingStrategy.__init__ defaults (:64-106)
DEFAULTS = {
    "grid_type": "arithmetic", "num_grids": 10, "auto_boundaries": True, "lower_boundary_pct": 5.0,
    "upper_boundary_pct": 5.0, "quantity_per_grid": 0.01, "volatility_lookback": 14, "auto_adjust_period": 86400,
    "adapt_to_market_regime": True, "rebalance_frequency": 3600,
}
# the per-regime keys of _adjust_grid_parameters (:861-880) and their defaults; "trending" is never a label here
REGIME_KEYS = {"ranging": (15, 3.0, 3.0), "trending": (8, 8.0, 8.0), "volatile": (12, 6.0, 6.0)}


def grid_param_ranges() -> Dict[str, Tuple]:
    """GA genes of the grid service's parameters (integer ranges where the reference's value is an integer or a flag):
    grid_type 0 = arithmetic, 1 = geometric; auto_boundaries / adapt_to_market_regime 0 / 1; periods in seconds."""
    return {
        "num_grids": (5, 30),
        "grid_type": (0, 1),
        "lower_boundary_pct": (1.0, 15.0),
        "upper_boundary_pct": (1.0, 15.0),
        "auto_boundaries": (0, 1),
        "volatility_lookback": (3, 30),
        "rebalance_frequency": (300, 86400),
        "auto_adjust_period": (3600, 7 * 86400),
        "adapt_to_market_regime": (0, 1),
    }


def grid_block(config: Optional[Dict]) -> Dict:
    """The grid_trading block of a config (a whole config.json dict, or the block itself)."""
    config = config or {}
    return config.get("grid_trading", config) if isinstance(config, dict) else {}


def period_ticks(seconds: float, bar_minutes: int) -> int:
    """Ticks between two runs of a check `(now - last) > seconds` that resets `last` whenever it runs: the smallest k >= 1
    with k * bar_seconds > seconds (floor(seconds / bar_seconds) + 1), capped at 2^31 - 1 (never, within a series)."""
    seconds = float(seconds)
    if not seconds >= 0.0:
        raise ValueError(f"a check period must be >= 0 seconds ({seconds})")
    bar = 60.0 * int(bar_minutes)
    if seconds >= bar * MAX_TICKS:
        return MAX_TICKS
    k = int(math.floor(seconds / bar)) + 1
    while (k - 1) >= 1 and (k - 1) * bar > seconds:
        k -= 1
    while k * bar <= seconds:
        k += 1
    return k


def _grid_type(value) -> int:
    if isinstance(value, str):
        if value == "volatility_based":
            raise ValueError("grid_type 'volatility_based' draws np.random levels (:363-377) and cannot be backtested")
        if value not in GRID_TYPES:
            raise ValueError(f"unknown grid_type {value!r} (one of {', '.join(GRID_TYPES)})")
        return GRID_TYPES.index(value)
    k = int(value)
    if k == 2:
        raise ValueError("grid_type 2 ('volatility_based') draws np.random levels (:363-377) and cannot be backtested")
    if k not in (0, 1):
        raise ValueError(f"grid_type index {value!r} must be 0 (arithmetic) or 1 (geometric)")
    return k


def decode_individual(params: Dict, defaults: Dict, bar_minutes: int) -> Dict:
    """One parameter dict (genes or config keys; missing keys from `defaults`) -> the kernel's fields plus the host's
    boundary rule: {num_grids, grid_type, rebalance_ticks, adjust_ticks, flags, lower_pct, upper_pct, auto, lookback}."""
    get = lambda k: params.get(k, defaults.get(k, DEFAULTS[k]))
    n = int(get("num_grids"))
    if not 1 <= n <= _lib.GRID_MAX_GRIDS:
        raise ValueError(f"num_grids = {n} outside 1 .. {_lib.GRID_MAX_GRIDS}")
    lo, up = float(get("lower_boundary_pct")), float(get("upper_boundary_pct"))
    if not (0.0 < lo < 100.0 and 0.0 < up < math.inf):
        raise ValueError(f"boundary pcts must satisfy 0 < lower < 100 and upper > 0 ({lo}, {up})")
    auto, adapt = bool(int(get("auto_boundaries"))), bool(int(get("adapt_to_market_regime")))
    lookback = int(get("volatility_lookback"))
    if auto and lookback < 1:
        raise ValueError(f"volatility_lookback = {lookback} days, need >= 1")
    return {"num_grids": n, "grid_type": _grid_type(get("grid_type")),
            "rebalance_ticks": period_ticks(get("rebalance_frequency"), bar_minutes),
            "adjust_ticks": period_ticks(get("auto_adjust_period"), bar_minutes),
            "flags": (_lib.GRID_ADAPT_REGIME if adapt else 0) | (_lib.GRID_AUTO_BOUNDARIES if auto else 0),
            "lower_pct": lo, "upper_pct": up, "auto": auto, "lookback": lookback if auto else 0}


def daily_closes(close_row: np.ndarray, minute0: int, bar_minutes: int, start_bar: int, lookback_days: int) -> List[float]:
    """The daily closes get_historical_klines(1d, "<lookback> days ago UTC") returns at t0 = the start bar's minute: one
    per UTC day whose start is >= t0 - lookback days, closed by the day's last bar at or before t0."""
    t0 = minute0 + start_bar * bar_minutes
    lo = t0 - lookback_days * 1440
    if lo < minute0:
        raise ValueError(f"start_bar = {start_bar} leaves no room for a {lookback_days}-day lookback (the series starts "
                         f"{(t0 - minute0) / 1440:.3f} days before it)")
    out = []
    for d in range(-(-lo // 1440), t0 // 1440 + 1):
        b = (min(t0, (d + 1) * 1440 - 1) - minute0) // bar_minutes
        if minute0 + b * bar_minutes >= d * 1440:
            out.append(float(close_row[b]))
    return out


def initial_bounds(p0: float, lower_pct: float, upper_pct: float, closes: Optional[List[float]] = None) -> Tuple[float, float]:
    """(lower, upper) of _initialize_grid (:266-289): from the volatility of `closes` when given, else from the pcts."""
    if closes is not None:
        volatility = np.std(closes) / np.mean(closes) * 100
        return float(p0 * (1 - volatility / 100)), float(p0 * (1 + volatility / 100))
    return p0 * (1 - lower_pct / 100), p0 * (1 + upper_pct / 100)


def regime_table(block: Dict) -> "C.Array":
    """b200bt_grid_regime_rule[5] of the config's per-regime keys, indexed by B200BT_REGIME_* (bull, bear, ranging,
    volatile, unknown): ranging and volatile set (num_grids, lower, upper) as :861-880 do; the labeller emits no
    "trending", so that branch never fires."""
    table = (_lib.GridRegimeRule * 5)()
    for label, name in ((2, "ranging"), (3, "volatile")):
        n, lo, up = REGIME_KEYS[name]
        table[label] = _lib.GridRegimeRule(1, int(block.get(f"{name}_num_grids", n)),
                                           float(block.get(f"{name}_lower_boundary_pct", lo)),
                                           float(block.get(f"{name}_upper_boundary_pct", up)))
    return table


def symbol_quantity(block: Dict, symbol: str) -> float:
    """_calculate_grid_quantity (:387-400): symbol_settings' quantity_per_grid, else the global one."""
    for s in block.get("symbol_settings", []) or []:
        if s.get("symbol") == symbol and "quantity_per_grid" in s:
            return float(s["quantity_per_grid"])
    return float(block.get("quantity_per_grid", DEFAULTS["quantity_per_grid"]))


class GridSweep(StrategySweep):
    """b200bt_grid_sweep for populations of grid parameter dicts on one market.

    market      MarketData (device closes, bar clock)
    quantity    qty per grid level: a number, one per symbol, or None = the config's symbol_settings / quantity_per_grid
    start_bar   tick 0 (default: the first bar that leaves room for the longest lookback of grid_param_ranges(), 30 days)
    regime      None (no regime source: the regime rule changes nothing), a device uint8 label tensor [S or 1][N]
                (B200BT_REGIME_*), or True for regime.regime_labels(market)
    config      config.json dict or its grid_trading block: defaults of the keys an individual does not set, the
                per-regime keys and the quantities
    objective   the stats field evaluate() averages over the symbols (default total_profit)
    service     False: one service per (individual, symbol) lane (b200bt_grid_sweep).  True: one service instance per
                individual trading all symbols, num_grids and pcts coupled across them (b200bt_grid_service_sweep); the
                regime source is then one label row: regime=True labels the market by PRIMARY_TRADING_SYMBOL (environment,
                default BTCUSDC), which must be one of the market's symbols, and per-symbol label rows are refused.

    Individuals that decode alike (same kernel fields and initial boundaries) are evaluated once."""

    FIELDS, OBJECTIVE_FIELDS, SERVICE_FIELDS = FIELDS, OBJECTIVE_FIELDS, SERVICE_FIELDS

    def __init__(self, market, quantity: Union[None, float, Sequence[float]] = None, start_bar: Optional[int] = None,
                 regime=None, config: Optional[Dict] = None, objective: str = "total_profit", service: bool = False):
        self.market = market
        self.service = bool(service)
        self.block = grid_block(config)
        self.defaults = {k: self.block.get(k, v) for k, v in DEFAULTS.items()}
        S, N = market.S, market.N
        if quantity is None:
            qty = [symbol_quantity(self.block, sym) for sym in market.symbols]
        elif np.ndim(quantity) == 0:
            qty = [float(quantity)] * S
        else:
            qty = [float(q) for q in quantity]
        if len(qty) != S or not all(np.isfinite(qty)):
            raise ValueError(f"quantity: {S} finite values needed")
        self.quantity = np.array(qty, dtype=np.float64)
        self._qty = torch.from_numpy(self.quantity).to(market.device)
        if start_bar is None:
            start_bar = min(N - 1, -(-30 * 1440 // market.bar_minutes))
        if not 0 <= int(start_bar) < N:
            raise ValueError(f"start_bar = {start_bar} outside [0, {N})")
        self.start_bar = int(start_bar)
        from .regime import label_rows, regime_labels
        if regime is True:
            if self.service:
                primary = os.getenv("PRIMARY_TRADING_SYMBOL", "BTCUSDC")
                if primary not in market.symbols:
                    raise ValueError(f"regime=True in service mode labels the market by PRIMARY_TRADING_SYMBOL = "
                                     f"{primary!r}, which is not one of the market's symbols {market.symbols}")
                regime = regime_labels(market, primary=primary)[0]
            else:
                regime = regime_labels(market)[0]
        self.labels, self.ld_labels = None, 0
        if regime is not None:
            self.labels, self.ld_labels = label_rows(regime, S, N)
            if self.service and self.ld_labels:
                raise ValueError("service mode reads one regime label row (market_regime_history): pass [1][N] labels")
        self.table = regime_table(self.block)
        self.objective = objective
        self._column(objective)
        self._closes = None                      # host closes up to the start bar (auto boundaries)
        self._vol_cache: Dict[Tuple[int, int], List[float]] = {}

    # -- host decoding --------------------------------------------------------------------------------------------
    def _history(self, s: int, lookback: int) -> List[float]:
        if self._closes is None:
            self._closes = self.market.close[:, :self.start_bar + 1].cpu().numpy()
        key = (s, lookback)
        if key not in self._vol_cache:
            self._vol_cache[key] = daily_closes(self._closes[s], self.market.minute0, self.market.bar_minutes,
                                                self.start_bar, lookback)
        return self._vol_cache[key]

    def decode(self, population: List[Dict]) -> Tuple[np.ndarray, np.ndarray]:
        """(individuals: GridIndividual bytes [pop], init_bounds float64 [pop][S][2])."""
        m = self.market
        if self._closes is None:
            self._closes = m.close[:, :self.start_bar + 1].cpu().numpy()
        p0 = [float(self._closes[s, self.start_bar]) for s in range(m.S)]
        rows = (_lib.GridIndividual * len(population))()
        bounds = np.empty((len(population), m.S, 2), dtype=np.float64)
        for i, params in enumerate(population):
            d = decode_individual(params, self.defaults, m.bar_minutes)
            rows[i] = _lib.GridIndividual(d["num_grids"], d["grid_type"], d["rebalance_ticks"], d["adjust_ticks"],
                                          d["flags"], 0, d["lower_pct"], d["upper_pct"])
            for s in range(m.S):
                closes = self._history(s, d["lookback"]) if d["auto"] else None
                if d["auto"] and not closes:
                    raise ValueError("auto_boundaries: no daily closes before the start bar")
                lo, up = initial_bounds(p0[s], d["lower_pct"], d["upper_pct"], closes)
                if d["grid_type"] == 1 and not lo > 0.0:
                    raise ValueError(f"a geometric grid needs a positive lower boundary ({lo})")
                bounds[i, s] = (lo, up)
        packed = np.frombuffer(bytes(rows), dtype=np.uint8).reshape(len(population), C.sizeof(_lib.GridIndividual))
        return packed, bounds

    def _inputs(self, population: List[Dict]):
        return list(self.decode(population)), {}

    def launch(self, indiv: torch.Tensor, bounds: torch.Tensor, stats: torch.Tensor,
               service: Optional[torch.Tensor] = None, rows: Optional[torch.Tensor] = None) -> None:
        """One launch on the current stream for the decoded individuals `indiv` (GridIndividual bytes [U]) and their
        initial boundaries `bounds` [U][S][2], writing `stats` [U][S][20] and, when given, the per-day rows `rows` [U][D]:
        b200bt_grid_service_sweep when `service` [U][12] is given, else b200bt_grid_sweep."""
        m = self.market
        table = self.table if self.labels is not None else None
        args = [m.close.data_ptr(), _lib.ld(m.close), m.S, m.N, self.start_bar, m.bar_minutes, m.minute0, indiv.data_ptr(),
                indiv.shape[0], self._qty.data_ptr(), bounds.data_ptr(), _lib.ptr(self.labels), self.ld_labels, table,
                stats.data_ptr()]
        if service is not None:
            args.append(service.data_ptr())
        _lib.call("b200bt_grid_service_sweep" if service is not None else "b200bt_grid_sweep", *args, _lib.ptr(rows),
                  0 if rows is None else rows.shape[1], _lib.current_stream())

    grid_stats = StrategySweep.stats_dict

    def day_profit(self, population: List[Dict]) -> Tuple[torch.Tensor, int]:
        """(rows float64 [pop][D] on the device, first_day): row i, column d = individual i's realised grid profit on
        calendar day first_day + d, summed over its symbols -- the row shape b200bt_cscv takes."""
        return self.day_rows(population)


class GridTradingStrategy:
    """The grid service's evaluation on the GPU engine, one parameter set at a time.  config: config.json dict (or its
    grid_trading block), as the reference reads it."""

    def __init__(self, config: Optional[Dict] = None):
        self.config = config or {}
        self.grid_config = grid_block(self.config)

    def backtest(self, symbol: str, market, params: Optional[Dict] = None, start_bar: Optional[int] = None,
                 regime=None) -> Optional[Dict]:
        """Run the service for `symbol` (one of market.symbols) over the market's bars from start_bar with `params`
        (keys of the grid_trading block; the config's values fill the rest).  Returns {"grid_profits": the reference's
        grid_profits[symbol] (without last_trade_profit, which the kernel does not keep), "performance": the
        _update_performance_metrics dict (:941-958) at the last tick, "grid": the final num_grids / boundaries, "stats":
        every b200bt_grid_stats field}.  Errors are logged and give None (the reference's convention)."""
        try:
            s = market.symbols.index(symbol)
            sweep = GridSweep(market, start_bar=start_bar, regime=regime, config=self.grid_config)
            st = sweep.grid_stats([dict(params or {})])
            v = {k: float(a[0, s]) for k, a in st.items()}
            t0 = market.minute0 + sweep.start_bar * market.bar_minutes
            t1 = market.minute0 + (market.N - 1) * market.bar_minutes
            trades, prof = int(v["total_trades"]), int(v["profitable_trades"])
            return {
                "grid_profits": {"total_profit": v["total_profit"], "total_trades": trades, "profitable_trades": prof,
                                 "start_time": iso_minute(t0)},
                "performance": {"timestamp": iso_minute(t1), "start_time": iso_minute(t0),
                                "running_time_hours": (t1 - t0) * 60 / 3600,
                                "total_trades": trades, "profitable_trades": prof, "win_rate": v["win_rate"],
                                "total_profit": v["total_profit"], "profit_per_day": v["profit_per_day"],
                                "symbols": [symbol], "simulation_mode": True, "symbol_profits": {symbol: v["total_profit"]}},
                "grid": {"num_grids": int(v["num_grids"]), "lower_boundary": v["lower"], "upper_boundary": v["upper"]},
                "stats": v,
            }
        except Exception as e:
            logger.error("Error backtesting grid for %s: %s", symbol, e)
            return None

    def backtest_service(self, market, params: Optional[Dict] = None, start_bar: Optional[int] = None,
                         regime=None) -> Optional[Dict]:
        """Run ONE service instance on all of the market's symbols (the reference's multi-symbol service, num_grids and
        pcts shared) with `params` over the market's bars from start_bar.  Returns {"grid_profits": {symbol: the
        reference's grid_profits[symbol] without last_trade_profit}, "performance": grid_performance (:941-958) at the
        last tick, "service": the final num_grids / pcts and the adjustment counts, "grid": {symbol: the final grid},
        "stats": {symbol: every b200bt_grid_stats field}}.  Errors are logged and give None."""
        try:
            sweep = GridSweep(market, start_bar=start_bar, regime=regime, config=self.grid_config, service=True)
            st = sweep.grid_stats([dict(params or {})])
            sv = {k: float(a[0]) for k, a in sweep.service_stats().items()}
            t0 = market.minute0 + sweep.start_bar * market.bar_minutes
            t1 = market.minute0 + (market.N - 1) * market.bar_minutes
            lanes = {sym: {k: float(a[0, s]) for k, a in st.items()} for s, sym in enumerate(market.symbols)}
            return {
                "grid_profits": {sym: {"total_profit": v["total_profit"], "total_trades": int(v["total_trades"]),
                                       "profitable_trades": int(v["profitable_trades"]), "start_time": iso_minute(t0)}
                                 for sym, v in lanes.items()},
                "performance": {"timestamp": iso_minute(t1), "start_time": iso_minute(t0),
                                "running_time_hours": (t1 - t0) * 60 / 3600,
                                "total_trades": int(sv["total_trades"]), "profitable_trades": int(sv["profitable_trades"]),
                                "win_rate": sv["win_rate"], "total_profit": sv["total_profit"],
                                "profit_per_day": sv["profit_per_day"], "symbols": list(market.symbols),
                                "simulation_mode": True,
                                "symbol_profits": {sym: v["total_profit"] for sym, v in lanes.items()}},
                "service": {"num_grids": int(sv["num_grids"]), "lower_boundary_pct": sv["lower_pct"],
                            "upper_boundary_pct": sv["upper_pct"], "n_adjustments": int(sv["n_adjustments"]),
                            "n_num_grids_changes": int(sv["n_num_grids_changes"]),
                            "min_num_grids": int(sv["min_num_grids"]), "max_num_grids": int(sv["max_num_grids"])},
                "grid": {sym: {"num_grids": int(v["num_grids"]), "lower_boundary": v["lower"],
                               "upper_boundary": v["upper"]} for sym, v in lanes.items()},
                "stats": lanes,
            }
        except Exception as e:
            logger.error("Error backtesting the grid service: %s", e)
            return None
