"""Market monitor on the GPU engine: the monitor's market_update replayed over a market's history (one update per
1-minute bar, with its fifteen combined indicators), per-bar labels of the combinations' categorical outputs for
PopulationSweep.class_stats, and services/utils/indicator_combinations.py as a drop-in.

Reference: services/market_monitor_service.py :219-301 (snapshot), :432-485 (market_update, combined_indicators),
:487-524 (volume_profile block, volume_profile.monitor_summary), :561-562 (trading opportunity); and
services/utils/indicator_combinations.py :56-694.  b200bt_market_monitor / b200bt_indicator_combinations compute every
number; the host only assembles the dicts.  The deliberate differences are listed in DESIGN.md section 3.17.
"""
from __future__ import annotations

import ctypes as C
import logging
from dataclasses import dataclass
from datetime import datetime, timedelta, timezone
from typing import Dict, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib

ROW_DTYPE = np.dtype(_lib.MONITOR_ROW_DTYPE)
_ROW_WORDS = ROW_DTYPE.itemsize // 8
LABEL_FIELDS = tuple(name for name, _ in _lib.MM_LABEL_FIELDS)
REQUIRED_FIELDS = ('rsi', 'macd', 'stoch_k', 'williams_r', 'bb_position', 'price_change_1m', 'price_change_5m', 'trend',
                   'trend_strength')
_DICT_INPUTS = ("rsi", "rsi_3m", "rsi_5m", "stoch_k", "macd", "williams_r", "bb_position", "trend_strength",
                "price_change_1m", "price_change_3m", "price_change_5m", "volume", "avg_volume", "ema_12", "ema_26")
_NONE_IS_ABSENT = ("rsi_5m", "ema_12", "ema_26")       # read with data.get(key, None) and tested against None
DEFAULT_TRADING_PARAMS = {"min_price_change_pct": 0.5, "min_volume_usdc": 50000}


def monitor_params(frame_bars: int = 100, label_field: int = 0, min_price_change_pct: float = 0.5,
                   min_volume_usdc: float = 50000.0) -> _lib.MonitorParams:
    return _lib.MonitorParams(frame_bars=int(frame_bars), label_field=int(label_field),
                              min_price_change_pct=float(min_price_change_pct), min_volume_usdc=float(min_volume_usdc))


def _run(market, params: _lib.MonitorParams, rows: bool, labels: bool):
    """b200bt_market_monitor on a MarketData with a 1-minute clock: (rows float64 [S][N][44] or None, labels uint8 [S][N]
    or None).  The 3-, 5- and 15-minute klines are made on the device by b200bt_resample."""
    from . import indicators as ind
    if market.bar_minutes != 1:
        raise ValueError(f"the market monitor replays a 1-minute clock (bar_minutes = {market.bar_minutes})")
    S, N = market.S, market.N
    k3, k5, k15 = (ind.resample(market, k) for k in (3, 5, 15))
    out_rows = torch.empty((S, N, _ROW_WORDS), dtype=torch.float64, device=market.device) if rows else None
    out_labels = torch.empty((S, N), dtype=torch.uint8, device=market.device) if labels else None
    with torch.cuda.device(market.device):
        _lib.call("b200bt_market_monitor", market.ohlcv.data_ptr(), S, N, market.minute0, market.bar_minutes,
                  k3.ohlcv.data_ptr(), k3.N, k5.ohlcv.data_ptr(), k5.N, k15.ohlcv.data_ptr(), k15.N, C.byref(params),
                  _lib.ptr(out_rows), _lib.ptr(out_labels), _lib.current_stream())
    return out_rows, out_labels


def rows_table(rows: torch.Tensor) -> np.ndarray:
    """Structured host view (_lib.MONITOR_ROW_DTYPE) of device rows [..][44]."""
    return rows.cpu().numpy().view(ROW_DTYPE)[..., 0]


def combine_rows(table: np.ndarray, device=None) -> np.ndarray:
    """b200bt_indicator_combinations on a structured array of rows whose snapshot half is filled: the rows with their
    combination half, as a new host array."""
    flat = np.ascontiguousarray(table.reshape(-1))
    dev = torch.from_numpy(flat.view(np.float64).copy()).to(device or torch.device("cuda", torch.cuda.current_device()))
    with torch.cuda.device(dev.device):
        _lib.call("b200bt_indicator_combinations", dev.data_ptr(), flat.size, _lib.current_stream())
    return dev.cpu().numpy().view(ROW_DTYPE).reshape(table.shape)


def combined_dict(row) -> Dict:
    """calculate_combined_indicators' dict from a row's combination half: None where the reference's combination
    failed, ints where the reference returns ints."""
    done = int(row["computed"])
    f = lambda name: float(row[name])
    builders = (
        lambda: f("trend_confirmation"),
        lambda: f("momentum_trend_alignment"),
        lambda: {"score": f("tma_score"), "state": _lib.MM_TMA_STATES[int(row["tma_state"])]},
        lambda: f("volatility_adjusted_momentum"),
        lambda: f("volatility_trend_score"),
        lambda: {"signal": _lib.MM_OSC_SIGNALS[int(row["osc_signal"])], "strength": f("osc_strength"),
                 "agreement": f("osc_agreement")},
        lambda: f("stoch_rsi"),
        lambda: {"signal": _lib.MM_DRSI_SIGNALS[int(row["drsi_signal"])], "divergence": f("drsi_divergence")},
        lambda: f("vwpm"),
        lambda: {"confirmation": _lib.MM_VPC_CONFIRMATIONS[int(row["vpc_confirmation"])],
                 "strength": 0 if _lib.MM_VPC_CONFIRMATIONS[int(row["vpc_confirmation"])] == "neutral"
                 else f("vpc_strength")},
        lambda: {"direction": _lib.MM_TSI_DIRECTIONS[int(row["tsi_direction"])], "strength": f("tsi_strength"),
                 "confidence": f("tsi_confidence")},
        lambda: {"regime": _lib.MM_REGIMES[int(row["regime"])], "confidence": f("regime_confidence")},
        lambda: {"probability": f("reversal_probability"),
                 "signals": [n for i, n in enumerate(_lib.MM_REVERSAL_SIGNALS) if int(row["reversal_signals"]) >> i & 1]},
        lambda: {"direction": int(row["breakout_direction"]), "confirmation": f("breakout_confirmation"),
                 "status": _lib.MM_BREAKOUT_STATUSES[int(row["breakout_status"])]},
        lambda: {"divergence": _lib.MM_DIVERGENCES[int(row["divergence"])], "strength": f("divergence_strength")},
    )
    return {name: (build() if done >> i & 1 else None) for i, (name, build) in enumerate(zip(_lib.MM_COMBINATIONS,
                                                                                              builders))}


def snapshot_row(market_data: Dict) -> np.ndarray:
    """One structured row whose snapshot half holds a market_update-like dict (every value through float(); trend as
    the reference compares it; absent keys cleared in `present`)."""
    row = np.zeros((), dtype=ROW_DTYPE)
    row["valid"] = 1
    t = market_data["trend"]
    row["trend"] = 0 if t == "uptrend" else 1 if t == "downtrend" else 2
    present = 0
    for key in _DICT_INPUTS:
        value = market_data.get(key)
        if key not in market_data or (value is None and key in _NONE_IS_ABSENT):
            row[key] = np.nan
            continue
        row[key] = float(value)
        present |= _lib.MM_HAS.get(key, 0)
    row["present"] = present
    return row


class IndicatorCombinations:
    """services/utils/indicator_combinations.py's IndicatorCombinations on the GPU: the reference's dicts, computed by
    b200bt_indicator_combinations."""

    def __init__(self):
        self.logger = logging.getLogger(__name__)
        self.combinations = _lib.MM_COMBINATIONS

    def calculate_combined_indicators(self, market_data: Dict) -> Dict:
        try:
            for field in REQUIRED_FIELDS:
                if field not in market_data:
                    self.logger.warning(f"Missing required field: {field}")
                    return {'error': f"Missing required field: {field}"}
            return combined_dict(combine_rows(snapshot_row(market_data)[None])[0])
        except Exception as e:
            self.logger.error(f"Error calculating combined indicators: {str(e)}")
            return {'error': str(e)}


def calculate_indicator_combinations(market_data: Dict) -> Dict:
    """Drop-in for services/utils/indicator_combinations.calculate_indicator_combinations."""
    return IndicatorCombinations().calculate_combined_indicators(market_data)


@dataclass
class MarketUpdateHistory:
    """One market update per 1-minute bar of `market`: rows (device float64 [S][N][44], one b200bt_monitor_row per bar
    close; None when not asked for) and labels (device uint8 [S][N] of label field 0, the trend, when rows were not
    asked for; else None)."""
    market: object
    frame_bars: int
    rows: Optional[torch.Tensor]
    labels: Optional[torch.Tensor]

    def table(self) -> np.ndarray:
        """The rows as a structured host array [S][N] of _lib.MONITOR_ROW_DTYPE."""
        if self.rows is None:
            raise ValueError("this history was computed without rows")
        return rows_table(self.rows)


def market_update_history(market, frame_bars: int = 100, config: Optional[Dict] = None,
                          rows: bool = True) -> MarketUpdateHistory:
    """The monitor's market update at the close of every bar of `market` (a MarketData on a 1-minute clock), from
    frames of `frame_bars` completed klines on each clock.  The trading-opportunity thresholds are
    config["trading_params"]'s min_price_change_pct (0.5 when absent) and min_volume_usdc, as the monitor reads them;
    without a config the reference's defaults (0.5 %, 50 000 USDC)."""
    tp = (config or {"trading_params": DEFAULT_TRADING_PARAMS})["trading_params"]
    pct, vol = float(tp.get("min_price_change_pct", 0.5)), float(tp["min_volume_usdc"])
    out_rows, labels = _run(market, monitor_params(frame_bars, 0, pct, vol), rows, not rows)
    return MarketUpdateHistory(market, int(frame_bars), out_rows, labels)


def _close_time(market, t: int) -> str:
    return (datetime(1970, 1, 1, tzinfo=timezone.utc) + timedelta(minutes=market.minute0 + t + 1)).isoformat()


def market_update(history: MarketUpdateHistory, s: int, t: int, volume_profile=None,
                  table: Optional[np.ndarray] = None) -> Optional[Dict]:
    """The monitor's market_update dict (:445-465) at the close of bar t of symbol s, with combined_indicators
    (:474-485) and, given a volume_profile.volume_profile_history of the market's 5-minute klines, the volume_profile
    block of the frame ending at the last 5-minute kline completed by then (:487-524).  timestamp is bar t's close time
    (UTC).  None where the monitor publishes no update: the frames are not full yet.  `table`: history.table(), when
    many updates are read."""
    rows = history.table() if table is None else table
    row = rows[s, t]
    if not row["valid"]:
        return None
    m = history.market
    out = {"symbol": m.symbols[s], "current_price": float(row["current_price"]), "avg_volume": float(row["avg_volume"]),
           "timestamp": _close_time(m, t)}
    for name in _lib.MM_SNAPSHOT_FIELDS[2:]:
        out[name] = float(row[name])
        if name == "bb_position":
            out["trend"] = _lib.MM_TRENDS[int(row["trend"])]
    out["combined_indicators"] = combined_dict(row)
    if volume_profile is not None:
        from . import volume_profile as vp
        minute = m.minute0 + t
        j = minute // 5 - m.minute0 // 5 - (0 if (minute + 1) // 5 != minute // 5 else 1)
        if j >= 0:
            summary = vp.monitor_summary(volume_profile.table(), s, j)
            if summary is not None:
                out["volume_profile"] = summary
    return out


def monitor_labels(market, field: Union[int, str], frame_bars: int = 100) -> Tuple[torch.Tensor, tuple]:
    """(labels uint8 [S][N], names): the code of one categorical field of every bar's market update (an index into
    names; 255 before the first full frames, so those bars belong to no class).  field: a name of LABEL_FIELDS or its
    index.  PopulationSweep.class_stats(population, labels, len(names)) then gives trade metrics per value."""
    f = LABEL_FIELDS.index(field) if isinstance(field, str) else int(field)     # ValueError: an unknown name
    _, labels = _run(market, monitor_params(frame_bars, f), False, True)
    return labels, _lib.MM_LABEL_FIELDS[f][1]
