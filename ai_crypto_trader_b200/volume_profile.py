"""Volume profile on the GPU engine: the reference's VolumeProfileAnalyzer as a drop-in, and its analysis replayed over a
market's history (one frame per bar) with per-bar zone labels for PopulationSweep.class_stats.

Reference: services/utils/volume_profile_analyzer.py
  analyze_volume_profile    :43-84    (_calculate_volume_profile :86-173, _generate_signals :232-316,
                                       _create_summary :318-394)
  detect_volume_anomalies   :487-562
  analyze_volume_delta      :564-684
and services/market_monitor_service.py, which analyses its df_5m frame, the last 100 five-minute klines (:170, :328),
and publishes the volume_profile block of a market update (:487-524).  b200bt_volume_profile computes every number; the
host only assembles the dicts and strings.

Differences, by design:
* Inputs go through float32, the project-wide market contract: prices and volumes that are not exact in float32 are
  rounded before the analysis.
* Equal bin volumes enter the value area in descending bin index (np.argsort(v, kind="stable")[::-1]).  The reference's
  unstable argsort leaves that order to the platform.
* The rolling volume mean / std of the anomaly pass are the sequential sum / window and the two-pass sample variance.
  pandas' rolling algorithm can differ from them in the last bits.
* histogram_base64 is None (no plotting); the analyzer does not add its work columns (delta, volume_ma, ...) to the
  caller's DataFrame; analyze_volume_by_time is not ported (the monitor never calls it).
* History frames are completed bars; the monitor's live frame also holds the kline in progress.
"""
from __future__ import annotations

import ctypes as C
import logging
from dataclasses import dataclass
from datetime import datetime
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib

logger = logging.getLogger("b200bt.volume_profile")

SIGNALS = _lib.VP_SIGNALS
ROW_DTYPE = np.dtype(_lib.VP_ROW_DTYPE)
_ROW_WORDS = ROW_DTYPE.itemsize // 8
_FLAT_FRAME_ERROR = "cannot convert float NaN to integer"      # the reference's int(NaN) on a frame with max == min
_EMPTY_FRAME_ERROR = "single positional indexer is out-of-bounds"


def vp_params(frame_bars: int, num_bins: int = 20, value_area_pct: float = 0.7, anomaly_window: int = 20,
              std_threshold: float = 2.0) -> _lib.VpParams:
    return _lib.VpParams(num_bins=int(num_bins), frame_bars=int(frame_bars), anomaly_window=int(anomaly_window),
                         reserved=0, value_area_pct=float(value_area_pct), std_threshold=float(std_threshold))


def _run(ohlcv: torch.Tensor, params: _lib.VpParams, rows: bool, bins: bool, device):
    """b200bt_volume_profile on device float32 [5][S][N]: (rows float64 [S][N][48] or None, bins [S][N][B] or None,
    labels uint8 [S][N])."""
    _, S, N = ohlcv.shape
    out_rows = torch.empty((S, N, _ROW_WORDS), dtype=torch.float64, device=device) if rows else None
    out_bins = torch.empty((S, N, params.num_bins), dtype=torch.float64, device=device) if bins else None
    labels = torch.empty((S, N), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.call("b200bt_volume_profile", ohlcv.data_ptr(), N, S, N, C.byref(params), _lib.ptr(out_rows),
                  _lib.ptr(out_bins), labels.data_ptr(), N, _lib.current_stream())
    return out_rows, out_bins, labels


def rows_table(rows: torch.Tensor) -> np.ndarray:
    """Structured host view (_lib.VP_ROW_DTYPE) [S][N] of device rows."""
    return rows.cpu().numpy().view(ROW_DTYPE)[..., 0]


def _price(x: float) -> str:
    return f"{x:.8f}" if x < 1 else f"{x:.2f}"


def _summary(row) -> str:
    """_create_summary (:318-394) from a row."""
    c, poc, vah, val = float(row["close"]), float(row["poc"]), float(row["value_area_high"]), float(row["value_area_low"])
    position = "inside" if val <= c <= vah else "above" if c > vah else "below"
    poc_position = "at" if abs(c - poc) / c < 0.005 else "above" if c > poc else "below"
    text = (f"Current price {_price(c)} is {position} the value area ({_price(val)} - {_price(vah)}) and {poc_position} "
            f"the point of control ({_price(poc)}). ")
    n_hvn = int(row["hvn_count"])
    if n_hvn > 0:
        if n_hvn <= 3:
            prices = ", ".join(_price(float(p)) for p in row["hvn_price"][:n_hvn])
            text += f"High volume nodes (potential support/resistance) at: {prices}. "
        else:
            text += f"Multiple high volume nodes identified ({n_hvn}). "
    if int(row["lvn_count"]) > 0:
        lvn = float(row["closest_lvn"])
        if abs(lvn - c) / c * 100 < 1.0:
            text += f"Price is near a low volume node at {_price(lvn)} (potential breakout zone). "
    text += {
        0: "Volume profile suggests potential resistance at current level.",
        1: "Volume profile suggests potential support at current level.",
        2: "Current price is in a low volume area, suggesting a potential breakout zone.",
        3: "Price is above the value area, potentially overbought based on volume profile.",
        4: "Price is below the value area, potentially oversold based on volume profile.",
    }.get(int(row["signal"]), "")
    return text


def _signals(row) -> Dict:
    s = {"poc": _lib.VP_POC_CODES[int(row["poc_code"])],
         "value_area": _lib.VP_VALUE_AREA_CODES[int(row["value_area_code"])]}
    if row["at_low_volume_node"]:
        s["low_volume_node"] = "at_low_volume_node"
    if row["at_high_volume_node"]:
        s["high_volume_node"] = "at_high_volume_node"
    s["overall"] = SIGNALS[int(row["signal"])]
    return s


def monitor_summary(rows: np.ndarray, s: int, t: int) -> Optional[Dict]:
    """The monitor's volume_profile block of a market update (market_monitor_service.py:492-512) for the frame ending
    at bar t of symbol s (rows: the structured table of volume_profile_history).  None where the monitor publishes no
    block: no frame, or a flat frame (the analyzer fails).  volume_pressure is absent where analyze_volume_delta fails
    (no buying volume: its insight divides by the ratio 0), volume_divergence is present when there is a divergence,
    volume_anomalies / recent_anomaly_percentage when anomalies were detected, as the monitor adds them."""
    row = rows[s, t]
    if not row["n_bars"] or not row["valid"]:
        return None
    out = {"poc": float(row["poc"]), "value_area_high": float(row["value_area_high"]),
           "value_area_low": float(row["value_area_low"]), "signal": SIGNALS[int(row["signal"])],
           "summary": _summary(row)}
    if row["buy_sell_ratio"] != 0:
        out["volume_pressure"] = _lib.VP_PRESSURES[int(row["pressure"])]
        if _lib.VP_DIVERGENCES[int(row["divergence"])] != "no_divergence":
            out["volume_divergence"] = _lib.VP_DIVERGENCES[int(row["divergence"])]
    if row["anomaly_status"] and row["total_anomalies"] > 0:
        out["volume_anomalies"] = True
        out["recent_anomaly_percentage"] = float(row["recent_anomaly_pct"])
    return out


@dataclass
class VolumeProfileHistory:
    """One frame per bar of `market` (the frame clock): rows (device float64 [S][N][48], one b200bt_vp_row per frame end;
    None when not asked for) and labels (device uint8 [S][N]: the overall signal, an index into SIGNALS, or 255)."""
    market: object
    rows: Optional[torch.Tensor]
    labels: torch.Tensor

    def table(self) -> np.ndarray:
        """The rows as a structured host array [S][N] of _lib.VP_ROW_DTYPE."""
        if self.rows is None:
            raise ValueError("this history was computed without rows")
        return rows_table(self.rows)


def _frame_market(market, timeframe_minutes: int):
    from . import indicators as ind
    k = int(timeframe_minutes)
    if k < market.bar_minutes or k % market.bar_minutes:
        raise ValueError(f"volume profile frames need {k}-minute bars derived from the market's clock (bar_minutes = "
                         f"{market.bar_minutes} does not divide {k})")
    return market if k == market.bar_minutes else ind.resample(market, k)


def volume_profile_history(market, timeframe_minutes: int = 5, frame_bars: int = 100, num_bins: int = 20,
                           value_area_pct: float = 0.7, rows: bool = True) -> VolumeProfileHistory:
    """The monitor's volume analysis (profile, delta, anomalies with window 20 and threshold 2) of every frame of
    `frame_bars` consecutive `timeframe_minutes` bars of `market` (a MarketData), resampled on the device when the
    timeframe is longer than the market's clock.  Frame ends before frame_bars - 1 have no frame."""
    fm = _frame_market(market, timeframe_minutes)
    out_rows, _, labels = _run(fm.ohlcv, vp_params(frame_bars, num_bins, value_area_pct), rows, False, fm.device)
    return VolumeProfileHistory(fm, out_rows, labels)


def volume_profile_labels(market, timeframe_minutes: int = 5, frame_bars: int = 100, num_bins: int = 20,
                          value_area_pct: float = 0.7) -> torch.Tensor:
    """Overall-signal labels uint8 [S][N] on the market's own clock: bar t carries the label of the frame ending at the
    last timeframe bar completed by the end of bar t (indicators.align_to_base), 255 where there is none (before the
    first full frame, or a flat frame), so those bars belong to no class of PopulationSweep.class_stats(population,
    labels, 6)."""
    from . import indicators as ind
    h = volume_profile_history(market, timeframe_minutes, frame_bars, num_bins, value_area_pct, rows=False)
    aligned = ind.align_to_base(h.labels.float(), market, int(timeframe_minutes))
    return torch.nan_to_num(aligned, nan=float(_lib.VP_NO_LABEL)).to(torch.uint8)


def profile_result(row, volumes: np.ndarray) -> Dict:
    """analyze_volume_profile's dict (:64-78) from a frame's row and bin volumes."""
    edges = np.linspace(float(row["price_min"]), float(row["price_max"]), len(volumes) + 1)
    levels = (edges[:-1] + edges[1:]) / 2
    max_volume = volumes.max() if volumes.max() > 0 else 1
    return {
        "timestamp": datetime.now().isoformat(),
        "price_levels": levels.tolist(),
        "volumes": volumes.tolist(),
        "normalized_volumes": (volumes / max_volume).tolist(),
        "poc": float(row["poc"]),
        "value_area_high": float(row["value_area_high"]),
        "value_area_low": float(row["value_area_low"]),
        "high_volume_nodes": [float(x) for x in levels[volumes >= 0.7 * max_volume]],
        "low_volume_nodes": [float(x) for x in levels[volumes <= 0.3 * max_volume]],
        "histogram_base64": None,
        "signals": _signals(row),
        "summary": _summary(row),
    }


def delta_result(row) -> Dict:
    """analyze_volume_delta's dict (:591-678) from a frame's row."""
    ratio = float(row["buy_sell_ratio"])
    result = {
        "timestamp": datetime.now().isoformat(),
        "current_cumulative_delta": float(row["cumulative_delta"]),
        "net_period_delta": float(row["net_period_delta"]),
        "buying_volume": float(row["buying_volume"]),
        "selling_volume": float(row["selling_volume"]),
        "buy_sell_ratio": ratio,
        "recent_delta": float(row["recent_delta"]),
    }
    if row["has_momentum"]:
        m = float(row["delta_momentum"])
        result["delta_momentum"] = m
        result["delta_momentum_direction"] = "accelerating_buying" if m > 0 else "accelerating_selling"
    signals = {"overall_pressure": _lib.VP_PRESSURES[int(row["pressure"])],
               "recent_pressure": _lib.VP_RECENT_PRESSURES[int(row["recent_pressure"])],
               "divergence": _lib.VP_DIVERGENCES[int(row["divergence"])]}
    result["signals"] = signals
    insights = []
    if signals["overall_pressure"] in ("strong_buying", "moderate_buying"):
        insights.append(f"Overall buying pressure exceeds selling ({ratio:.2f}x)")
    elif signals["overall_pressure"] in ("strong_selling", "moderate_selling"):
        insights.append(f"Overall selling pressure exceeds buying ({1 / ratio:.2f}x)")
    if "delta_momentum" in result and abs(result["delta_momentum"]) > 0:
        insights.append("Buying pressure is accelerating" if result["delta_momentum"] > 0
                        else "Selling pressure is accelerating")
    if signals["divergence"] == "bullish_divergence":
        insights.append("Bullish divergence: price down, but buying volume increasing")
    elif signals["divergence"] == "bearish_divergence":
        insights.append("Bearish divergence: price up, but selling volume increasing")
    result["insights"] = insights
    return result


def anomaly_result(row, data) -> Dict:
    """detect_volume_anomalies' dict (:520-558) from a frame's row (None: no anomalies) and the DataFrame (the timestamps
    of recent_anomalies; without a timestamp column the reference fails there, and so does this)."""
    import pandas as pd
    if row is None or row["total_anomalies"] == 0:
        return {"timestamp": datetime.now().isoformat(), "anomalies_detected": False,
                "message": "No volume anomalies detected"}
    n = int(row["n_recent"])
    recent = data.iloc[row["recent_offset"][:n]][["timestamp", "volume"]].copy()
    if pd.api.types.is_datetime64_dtype(recent["timestamp"]):
        recent["timestamp"] = recent["timestamp"].dt.strftime("%Y-%m-%d %H:%M:%S")
    records = [{"timestamp": ts, "volume": float(np.float32(v)), "volume_ma": float(ma), "anomaly_significance": float(sig)}
               for ts, v, ma, sig in zip(recent["timestamp"].tolist(), recent["volume"].tolist(), row["recent_ma"][:n],
                                         row["recent_significance"][:n])]
    result = {
        "timestamp": datetime.now().isoformat(),
        "anomalies_detected": True,
        "total_anomalies": int(row["total_anomalies"]),
        "recent_anomalies": records,
        "strongest_anomaly": {"significance": float(row["strongest_significance"]),
                              "volume": float(row["strongest_volume"]), "normal_volume": float(row["strongest_ma"])},
        "recent_anomaly_percentage": float(row["recent_anomaly_pct"]),
    }
    if result["recent_anomaly_percentage"] > 15:
        result["message"] = "There is elevated trading volume activity recently"
    return result


class VolumeProfileAnalyzer:
    """services/utils/volume_profile_analyzer.py's VolumeProfileAnalyzer on the GPU: each call analyses the DataFrame as
    one frame and returns the reference's dict, or {'error': ...} where the reference fails."""

    def __init__(self, num_bins: int = 20, value_area_pct: float = 0.7):
        self.num_bins = num_bins
        self.value_area_pct = value_area_pct
        self.logger = logging.getLogger(__name__)

    def _frame(self, data, window: int = 20, std_threshold: float = 2.0):
        """(row, bins) of `data` analysed as one frame; missing columns (not read by the calling method) are filled."""
        W = len(data)
        cols = []
        for name in ("open", "high", "low", "close", "volume"):
            src = name if name in data.columns else "close" if "close" in data.columns else None
            cols.append(data[src].to_numpy(dtype=np.float32) if src else np.ones(W, dtype=np.float32))
        ohlcv = torch.from_numpy(np.stack(cols)[:, None, :]).cuda()
        params = vp_params(W, self.num_bins, self.value_area_pct, max(int(window), 2), std_threshold)
        rows, bins, _ = _run(ohlcv, params, True, True, ohlcv.device)
        return rows_table(rows)[0, W - 1], bins[0, W - 1].cpu().numpy()

    def analyze_volume_profile(self, data) -> Dict:
        try:
            for col in ("high", "low", "close", "volume"):
                if col not in data.columns:
                    self.logger.warning(f"Missing required column: {col}")
                    return {"error": f"Missing required column: {col}"}
            if len(data) == 0:
                raise IndexError(_EMPTY_FRAME_ERROR)
            row, volumes = self._frame(data)
            if not row["valid"]:
                raise ValueError(_FLAT_FRAME_ERROR)
            return profile_result(row, volumes)
        except Exception as e:
            self.logger.error(f"Error analyzing volume profile: {str(e)}")
            return {"error": str(e)}

    def detect_volume_anomalies(self, data, window: int = 20, std_threshold: float = 2.0) -> Dict:
        try:
            if "volume" not in data.columns:
                return {"error": "Missing required column: volume"}
            if len(data) < window:
                return {"error": f"Insufficient data for window size {window}"}
            if window < 0:
                raise ValueError("window must be an integer 0 or greater")
            if window < 2:                       # pandas' std of fewer than 2 values is NaN: nothing exceeds it
                return anomaly_result(None, data)
            row, _ = self._frame(data, window, std_threshold)
            return anomaly_result(row, data)
        except Exception as e:
            self.logger.error(f"Error detecting volume anomalies: {str(e)}")
            return {"error": str(e)}

    def analyze_volume_delta(self, data) -> Dict:
        try:
            for col in ("open", "close", "volume"):
                if col not in data.columns:
                    return {"error": f"Missing required column: {col}"}
            if len(data) == 0:
                raise IndexError(_EMPTY_FRAME_ERROR)
            row, _ = self._frame(data)
            return delta_result(row)
        except Exception as e:
            self.logger.error(f"Error analyzing volume delta: {str(e)}")
            return {"error": str(e)}


def analyze_volume_profile(df, num_bins: int = 20, value_area_pct: float = 0.7) -> Dict:
    return VolumeProfileAnalyzer(num_bins=num_bins, value_area_pct=value_area_pct).analyze_volume_profile(df)


def detect_volume_anomalies(df, window: int = 20, std_threshold: float = 2.0) -> Dict:
    return VolumeProfileAnalyzer().detect_volume_anomalies(df, window, std_threshold)


def analyze_volume_delta(df) -> Dict:
    return VolumeProfileAnalyzer().analyze_volume_delta(df)
