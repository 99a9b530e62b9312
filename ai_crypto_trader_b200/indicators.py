"""Rolling indicators on the GPU (host side of Family 1, include/b200bt.h).

Each function takes fp32 CUDA tensors shaped [S][N] (one row per symbol) and returns fp32
tensors; arithmetic is fp64 inside the kernels.  `fill=True` applies the reference's
TechnicalAnalyzer._handle_nan_values policy (binance_ml_strategy.py:28-38: ffill, bfill, 0);
`fill=False` leaves `ta`'s leading NaNs in place.  TechnicalAnalyzer below mirrors the
reference class of the same name (binance_ml_strategy.py:14-249) for a whole batch of symbols.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib
from .sweep import rsi_bank  # noqa: F401  (re-export: RSI lives with the sweep that consumes it)


def _rows(*ts):
    """-> (S, N, ld, inputs): fp32 CUDA [S][N] inputs with unit time stride, and the one row stride `ld` every kernel reads
    all of a call's inputs with.  Inputs whose row strides differ (a slice of a padded buffer next to a dense tensor) are
    copied to contiguous rows first."""
    S, N = ts[0].shape
    for t in ts:
        if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and tuple(t.shape) == (S, N) and t.stride(1) == 1):
            raise ValueError(f"inputs must be device float32 tensors [{S}][{N}] with unit stride along the bars")
    if len({_lib.ld(t) for t in ts}) > 1:
        ts = tuple(t.contiguous() for t in ts)
    return S, N, _lib.ld(ts[0]), ts


def _ints(v: Sequence[int]):
    return (C.c_int * len(v))(*[int(x) for x in v])


def nanfill_(x: torch.Tensor) -> torch.Tensor:
    """In-place ffill -> bfill -> 0 along the last axis of a contiguous fp32 CUDA tensor."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()):
        raise ValueError("x must be a contiguous device float32 tensor")
    N = x.shape[-1]
    rows = x.numel() // N
    ws = torch.empty(int(_lib.load().b200bt_nanfill_workspace_floats(rows, N)), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.call("b200bt_nanfill", x.data_ptr(), rows, N, ws.data_ptr(), _lib.current_stream())
    return x


def _bank(fn: str, x: torch.Tensor, windows: Sequence[int], fill: bool, extra=()):
    S, N, ld, (x,) = _rows(x)
    out = torch.empty((S, len(windows), N), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.call(fn, *extra, x.data_ptr(), S, N, ld, _ints(windows), len(windows), out.data_ptr(),
                  _lib.current_stream())
    return nanfill_(out) if fill else out


def ema_bank(close: torch.Tensor, spans: Sequence[int], fill: bool = True) -> torch.Tensor:
    return _bank("b200bt_ema_bank", close, spans, fill)


def sma_bank(close: torch.Tensor, windows: Sequence[int], fill: bool = True) -> torch.Tensor:
    return _bank("b200bt_sma_bank", close, windows, fill)


def atr_bank(high, low, close, windows: Sequence[int]) -> torch.Tensor:
    S, N, ld, (high, low, close) = _rows(high, low, close)
    out = torch.empty((S, len(windows), N), dtype=torch.float32, device=close.device)
    with torch.cuda.device(close.device):
        _lib.call("b200bt_atr_bank", high.data_ptr(), low.data_ptr(), close.data_ptr(), S, N, ld,
                  _ints(windows), len(windows), out.data_ptr(), _lib.current_stream())
    return out


def _outs(n, like):
    return [torch.empty_like(like) for _ in range(n)]


def _maybe_fill(ts, fill):
    if fill:
        for t in ts:
            nanfill_(t)
    return ts


def macd(close, fast: int = 12, slow: int = 26, sign: int = 9, fill: bool = True):
    S, N, ld, (close,) = _rows(close)
    line, signal, diff = _outs(3, close.contiguous())
    with torch.cuda.device(close.device):
        _lib.call("b200bt_macd", close.data_ptr(), S, N, ld, fast, slow, sign, line.data_ptr(),
                  signal.data_ptr(), diff.data_ptr(), _lib.current_stream())
    return tuple(_maybe_fill([line, signal, diff], fill))


def bollinger(close, window: int = 20, dev: float = 2.0, fill: bool = True):
    """-> (high, mid, low, width, position)."""
    S, N, ld, (close,) = _rows(close)
    outs = _outs(5, close.contiguous())
    with torch.cuda.device(close.device):
        _lib.call("b200bt_bollinger", close.data_ptr(), S, N, ld, window, float(dev),
                  *[o.data_ptr() for o in outs], _lib.current_stream())
    return tuple(_maybe_fill(outs, fill))


def stochastic(high, low, close, window: int = 14, smooth: int = 3, fill: bool = True):
    S, N, ld, (high, low, close) = _rows(high, low, close)
    k, d = _outs(2, close.contiguous())
    with torch.cuda.device(close.device):
        _lib.call("b200bt_stochastic", high.data_ptr(), low.data_ptr(), close.data_ptr(), S, N, ld,
                  window, smooth, k.data_ptr(), d.data_ptr(), _lib.current_stream())
    return tuple(_maybe_fill([k, d], fill))


def williams_r(high, low, close, lbp: int = 14, fill: bool = True):
    S, N, ld, (high, low, close) = _rows(high, low, close)
    (out,) = _outs(1, close.contiguous())
    with torch.cuda.device(close.device):
        _lib.call("b200bt_williams_r", high.data_ptr(), low.data_ptr(), close.data_ptr(), S, N, ld, lbp,
                  out.data_ptr(), _lib.current_stream())
    return _maybe_fill([out], fill)[0]


def ichimoku(high, low, w1: int = 9, w2: int = 26, w3: int = 52, fill: bool = True):
    S, N, ld, (high, low) = _rows(high, low)
    a, b = _outs(2, high.contiguous())
    with torch.cuda.device(high.device):
        _lib.call("b200bt_ichimoku", high.data_ptr(), low.data_ptr(), S, N, ld, w1, w2, w3, a.data_ptr(),
                  b.data_ptr(), _lib.current_stream())
    return tuple(_maybe_fill([a, b], fill))


def vwap(high, low, close, volume, window: int = 14, fill: bool = True):
    S, N, ld, (high, low, close, volume) = _rows(high, low, close, volume)
    (out,) = _outs(1, close.contiguous())
    with torch.cuda.device(close.device):
        _lib.call("b200bt_vwap", high.data_ptr(), low.data_ptr(), close.data_ptr(), volume.data_ptr(), S, N,
                  ld, window, out.data_ptr(), _lib.current_stream())
    return _maybe_fill([out], fill)[0]


class TechnicalAnalyzer:
    """binance_ml_strategy.py:14-249 for S symbols at once: the 18 indicator columns as device
    tensors in `self.data`, and the last-bar scalars `get_all_indicators(symbol_index)` reads."""

    COLUMNS = ("sma_20", "sma_50", "sma_200", "ema_12", "ema_26", "macd", "macd_signal", "macd_diff", "ichimoku_a",
               "ichimoku_b", "rsi", "stoch_k", "stoch_d", "williams_r", "bb_high", "bb_mid", "bb_low", "bb_width",
               "bb_position", "atr", "vwap")

    def __init__(self, market):
        from .sweep import MarketData
        assert isinstance(market, MarketData)
        self.market = market
        o, h, l, c, v = market.open, market.high, market.low, market.close, market.volume
        S, N, ld, (h, l, c, v) = _rows(h, l, c, v)
        # all 21 columns of _calculate_all_indicators (:40-182) + _handle_nan_values in three fused launches and one batched
        # NaN-policy call (b200bt_analyzer): one [21][S][N] allocation, self.data[name] = its [S][N] block
        lib = _lib.load()
        cols = torch.empty((len(_lib.ANALYZER_COLUMNS), S, N), dtype=torch.float32, device=c.device)
        ws = torch.empty(int(lib.b200bt_analyzer_workspace_floats(S, N)), dtype=torch.float32, device=c.device)
        with torch.cuda.device(c.device):
            _lib.call("b200bt_analyzer", h.data_ptr(), l.data_ptr(), c.data_ptr(), v.data_ptr(), S, N, ld, cols.data_ptr(),
                      ws.data_ptr(), _lib.current_stream())
        d: Dict[str, torch.Tensor] = {name: cols[i] for i, name in enumerate(_lib.ANALYZER_COLUMNS)}
        self.data = d
        last = torch.stack([d[k][:, -1] for k in self.COLUMNS] + [c[:, -1], h[:, -1], l[:, -1]], dim=1)
        self._last = last.double().cpu().numpy()                           # [S][len(COLUMNS)+3]

    def _get(self, s: int, name: str) -> float:
        extra = {"close": len(self.COLUMNS), "high": len(self.COLUMNS) + 1, "low": len(self.COLUMNS) + 2}
        idx = extra[name] if name in extra else self.COLUMNS.index(name)
        return float(self._last[s, idx])

    def get_trend(self, s: int = 0) -> Tuple[str, float]:
        last_close, sma20, sma50 = self._get(s, "close"), self._get(s, "sma_20"), self._get(s, "sma_50")
        strength = ((last_close - sma20) / sma20 * 100 + (last_close - sma50) / sma50 * 100) / 2      # :191-192
        if last_close > sma20 and sma20 > sma50:
            return "uptrend", abs(strength)
        if last_close < sma20 and sma20 < sma50:
            return "downtrend", abs(strength)
        return "sideways", abs(strength)

    def get_volatility(self, s: int = 0) -> float:
        return self._get(s, "atr") / self._get(s, "close")                 # :208

    def get_support_resistance(self, s: int = 0) -> Dict[str, float]:
        h, l, c = self._get(s, "high"), self._get(s, "low"), self._get(s, "close")
        pivot = (h + l + c) / 3
        return {"support1": 2 * pivot - h, "support2": pivot - (h - l), "resistance1": 2 * pivot - l,
                "resistance2": pivot + (h - l)}

    def get_all_indicators(self, s: int = 0) -> Dict:
        trend, strength = self.get_trend(s)
        return {"rsi": self._get(s, "rsi"), "stoch_k": self._get(s, "stoch_k"), "stoch_d": self._get(s, "stoch_d"),
                "macd": self._get(s, "macd"), "macd_signal": self._get(s, "macd_signal"),
                "williams_r": self._get(s, "williams_r"), "bb_position": self._get(s, "bb_position"),
                "volatility": self.get_volatility(s), "trend": trend, "trend_strength": strength}


# ---------------------------------------------------------------------------------------
# Multi-timeframe (BASELINE configs[3]); recipe: services/market_monitor_service.py:219-301
# ---------------------------------------------------------------------------------------
def resample(market, k: int):
    """Clock-aligned k-minute bars derived on the device from `market` (a MarketData)."""
    from .sweep import MarketData
    M = int(_lib.load().b200bt_resample_bars(market.N, market.minute0, market.bar_minutes, k))
    out = torch.empty((5, market.S, M), dtype=torch.float32, device=market.device)
    with torch.cuda.device(market.device):
        _lib.call("b200bt_resample", market.ohlcv.data_ptr(), market.S, market.N, market.minute0, market.bar_minutes, k,
                  out.data_ptr(), M, _lib.current_stream())
    first_bucket_minute = (market.minute0 // k) * k
    return MarketData(out, symbols=market.symbols, minute0=first_bucket_minute, bar_minutes=k, device=market.device)


def align_to_base(series: torch.Tensor, base, k: int) -> torch.Tensor:
    """Higher-timeframe series [S][M] -> base clock [S][N]: value of the last COMPLETED k-minute bar."""
    S, M = series.shape
    out = torch.empty((S, base.N), dtype=torch.float32, device=series.device)
    series = series.contiguous()
    with torch.cuda.device(series.device):
        _lib.call("b200bt_align", series.data_ptr(), S, M, base.N, base.minute0, base.bar_minutes, k, out.data_ptr(),
                  _lib.current_stream())
    return out


def multi_timeframe_indicators(market, s: int = 0) -> Dict:
    """calculate_technical_indicators (market_monitor_service.py:219-301) for symbol `s`: RSI/MACD on
    1m, 3m, 5m; stochastic, Williams, Bollinger position, SMA20/50 on 1m; SMA20 on 5m; trend from 1m;
    trend_strength = |0.6*s_1m + 0.4*s_5m|; price changes against the open of each timeframe's last bar."""
    tf = {1: market, 3: resample(market, 3), 5: resample(market, 5), 15: resample(market, 15)}
    last = lambda t: float(t[s, -1].item())
    out = {}
    for k, name in ((1, ""), (3, "_3m"), (5, "_5m")):
        m = tf[k]
        out["rsi" + name] = last(rsi_bank(m.close, [14], fill=False)[:, 0])
        out["macd" + name] = last(macd(m.close, fill=False)[0])
    m1 = tf[1]
    out["stoch_k"] = last(stochastic(m1.high, m1.low, m1.close, fill=False)[0])
    out["williams_r"] = last(williams_r(m1.high, m1.low, m1.close, fill=False))
    out["bb_position"] = last(bollinger(m1.close, fill=False)[4])
    sma1 = sma_bank(m1.close, [20, 50], fill=False)
    sma20_1m, sma50_1m = last(sma1[:, 0]), last(sma1[:, 1])
    sma20_5m = last(sma_bank(tf[5].close, [20], fill=False)[:, 0])
    last_close = last(m1.close)
    strength_1m = (last_close - sma20_1m) / sma20_1m * 100
    strength_5m = (last_close - sma20_5m) / sma20_5m * 100
    out["trend_strength"] = abs(strength_1m * 0.6 + strength_5m * 0.4)
    if last_close > sma20_1m and sma20_1m > sma50_1m:
        out["trend"] = "uptrend"
    elif last_close < sma20_1m and sma20_1m < sma50_1m:
        out["trend"] = "downtrend"
    else:
        out["trend"] = "sideways"
    for k in (1, 3, 5, 15):
        o = last(tf[k].open)
        out[f"price_change_{k}m"] = ((last_close - o) / o) * 100
    return out
