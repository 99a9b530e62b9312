"""NumPy float64 restatement of b200bt_volume_profile (csrc/volume_profile.cu): the row, the bins and the label of one
frame, and of every frame of a market.

It follows services/utils/volume_profile_analyzer.py expression for expression, with the kernel's two fixed choices:
equal bin volumes enter the value area in descending bin index (np.argsort(v, kind="stable")[::-1]), and the rolling
volume mean / std are the sequential sum / w and the two-pass sample variance (pandas' rolling algorithm is not
restated).  Sums the reference takes with np.sum or Series.sum go through `pairwise_sum`, numpy's own order."""
from __future__ import annotations

import math

import numpy as np

from ai_crypto_trader_b200 import _lib

ROW = np.dtype(_lib.VP_ROW_DTYPE)
RECENT = 5


def pairwise_sum(values) -> float:
    """numpy's pairwise summation of float64 values (np.add.reduce): sequential from 0.0 below 8 values, 8 interleaved
    accumulators up to 128, halves split at a multiple of 8 above."""
    a = [float(x) for x in values]

    def rec(lo, n):
        if n < 8:
            r = 0.0
            for i in range(n):
                r += a[lo + i]
            return r
        if n <= 128:
            r = a[lo:lo + 8]
            i = 8
            while i < n - n % 8:
                for j in range(8):
                    r[j] += a[lo + i + j]
                i += 8
            s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            while i < n:
                s += a[lo + i]
                i += 1
            return s
        n2 = n // 2
        n2 -= n2 % 8
        return rec(lo, n2) + rec(lo + n2, n - n2)

    return rec(0, len(a))


def price_levels(pmin: float, pmax: float, B: int) -> np.ndarray:
    """np.linspace(pmin, pmax, B + 1) midpoints, as the reference computes them."""
    edges = np.linspace(pmin, pmax, B + 1)
    return (edges[:-1] + edges[1:]) / 2


def rolling_stats(vol: np.ndarray, g: int, w: int):
    s = 0.0
    for x in vol[g - w + 1:g + 1]:
        s += float(x)
    ma = s / w
    ss = 0.0
    for x in vol[g - w + 1:g + 1]:
        d = float(x) - ma
        ss += d * d
    return ma, math.sqrt(ss / (w - 1))


def _dist_pct(a, c):
    return abs(c - a) / c * 100


def empty_row() -> np.ndarray:
    row = np.zeros((), dtype=ROW)
    for name in ROW.names:
        if ROW[name].base.kind == "f":
            row[name] = np.nan
    for name in ("poc_code", "value_area_code", "poc_bin", "value_area_low_bin", "value_area_high_bin",
                 "closest_lvn_bin", "pressure", "recent_pressure", "divergence", "strongest_offset"):
        row[name] = -1
    row["recent_offset"] = -1
    row["signal"] = _lib.VP_NO_LABEL
    return row


def frame(o, h, l, c, v, num_bins=20, value_area_pct=0.7, window=20, std_threshold=2.0):
    """(row, bins) of one frame: float64 arrays of its bars in order."""
    o, h, l, c, v = (np.asarray(x, dtype=np.float64) for x in (o, h, l, c, v))
    W, B = len(c), num_bins
    row = empty_row()
    bins = np.zeros(B)
    row["n_bars"] = W
    pmin, pmax, close = float(l.min()), float(h.max()), float(c[-1])
    row["price_min"], row["price_max"], row["close"] = pmin, pmax, close
    row["valid"] = int(pmax > pmin)
    if row["valid"]:
        bin_size = (pmax - pmin) / B
        for i in range(W):
            lb = max(0, int((float(l[i]) - pmin) / bin_size))
            hb = min(B - 1, int((float(h[i]) - pmin) / bin_size))
            if hb >= lb:
                bins[lb:hb + 1] += float(v[i]) / (hb - lb + 1)
        levels = price_levels(pmin, pmax, B)
        mv = float(bins.max())
        max_volume = mv if mv > 0 else 1.0
        poc_bin = int(np.argmax(bins))
        total = pairwise_sum(bins)
        thr = total * value_area_pct
        cum, idx = 0.0, []
        for i in np.argsort(bins, kind="stable")[::-1]:
            cum += float(bins[i])
            idx.append(int(i))
            if cum >= thr:
                break
        va_lo, va_hi = min(idx), max(idx)
        poc, val, vah = float(levels[poc_bin]), float(levels[va_lo]), float(levels[va_hi])
        hvn = np.nonzero(bins >= 0.7 * max_volume)[0]
        lvn = np.nonzero(bins <= 0.3 * max_volume)[0]
        if _dist_pct(poc, close) < 0.5:
            poc_code = 0 if close < poc else 1
        else:
            poc_code = 2 if close < poc else 3
        if close > vah:
            va_code = 0 if (close - vah) / close * 100 < 0.3 else 1
        elif close < val:
            va_code = 2 if (val - close) / close * 100 < 0.3 else 3
        else:
            with np.errstate(invalid="ignore", divide="ignore"):
                rel = np.float64(close - val) / np.float64(vah - val)
            va_code = 4 if rel < 0.3 else 5 if rel > 0.7 else 6
        at_l = any(_dist_pct(float(levels[i]), close) < 0.3 for i in lvn)
        at_h = any(_dist_pct(float(levels[i]), close) < 0.3 for i in hvn)
        if va_code == 0 or poc_code == 1:
            label = 0
        elif va_code == 2 or poc_code == 0:
            label = 1
        elif at_l:
            label = 2
        elif va_code == 1:
            label = 3
        elif va_code == 3:
            label = 4
        else:
            label = 5
        closest = min(lvn, key=lambda i: abs(float(levels[i]) - close)) if len(lvn) else -1
        row["signal"], row["poc_code"], row["value_area_code"] = label, poc_code, va_code
        row["at_low_volume_node"], row["at_high_volume_node"] = int(at_l), int(at_h)
        row["poc_bin"], row["value_area_low_bin"], row["value_area_high_bin"] = poc_bin, va_lo, va_hi
        row["hvn_count"], row["lvn_count"], row["closest_lvn_bin"] = len(hvn), len(lvn), closest
        row["poc"], row["value_area_low"], row["value_area_high"] = poc, val, vah
        row["total_volume"], row["max_volume"] = total, mv
        for k, i in enumerate(hvn[:3]):
            row["hvn_price"][k] = levels[i]
        if closest >= 0:
            row["closest_lvn"] = levels[closest]
    # delta
    d = np.where(c >= o, v, -v)
    cum = float(d[0])
    for x in d[1:]:
        cum += float(x)
    periods = min(20, W)
    buy, sell = pairwise_sum(d[d > 0]), abs(pairwise_sum(d[d < 0]))
    ratio = buy / sell if sell > 0 else math.inf
    recent = pairwise_sum(d[W - periods:])
    row["cumulative_delta"], row["net_period_delta"] = cum, pairwise_sum(d)
    row["buying_volume"], row["selling_volume"], row["buy_sell_ratio"] = buy, sell, ratio
    row["recent_delta"] = recent
    row["has_momentum"] = int(W >= 40)
    if W >= 40:
        row["delta_momentum"] = recent - pairwise_sum(d[W - 40:W - 20])
    row["pressure"] = 0 if ratio > 1.5 else 1 if ratio > 1.1 else 2 if ratio < 0.67 else 3 if ratio < 0.9 else 4
    row["recent_pressure"] = 0 if recent > 0 else 1
    price_up, delta_up = float(c[-1]) - float(c[W - periods]) > 0, recent > 0
    row["divergence"] = 0 if price_up and not delta_up else 1 if not price_up and delta_up else 2
    # anomalies
    row["anomaly_status"] = int(W >= window)
    row["total_anomalies"] = row["n_recent"] = 0
    if W >= window:
        found = []                                   # (offset, ma, significance)
        for g in range(window - 1, W):
            ma, sd = rolling_stats(v, g, window)
            x = float(v[g])
            if x > ma + std_threshold * sd:
                with np.errstate(divide="ignore", invalid="ignore"):
                    found.append((g, ma, float(np.float64(x - ma) / np.float64(sd))))
        row["total_anomalies"] = len(found)
        row["recent_anomaly_pct"] = sum(1 for f in found if f[0] >= W - periods) / periods * 100
        if found:
            best = max(range(len(found)), key=lambda k: (found[k][2], -k))
            g, ma, sig = found[best]
            row["strongest_offset"], row["strongest_significance"] = g, sig
            row["strongest_volume"], row["strongest_ma"] = float(v[g]), ma
            last = found[-RECENT:]
            row["n_recent"] = len(last)
            for k, (g, ma, sig) in enumerate(last):
                row["recent_offset"][k], row["recent_ma"][k], row["recent_significance"][k] = g, ma, sig
    return row, bins


def history(ohlcv: np.ndarray, frame_bars: int, num_bins=20, value_area_pct=0.7, window=20, std_threshold=2.0):
    """rows [S][N], bins [S][N][B] and labels uint8 [S][N] of every frame of float32 OHLCV [5][S][N], with the rows of
    bars without a frame as the kernel writes them."""
    _, S, N = ohlcv.shape
    rows = np.empty((S, N), dtype=ROW)
    rows[...] = empty_row()
    rows["n_bars"] = 0
    rows["valid"] = 0
    bins = np.zeros((S, N, num_bins))
    picks = [(s, t) for s in range(S) for t in range(frame_bars - 1, N)]
    if picks:
        r, b, _ = frames_at(ohlcv, picks, frame_bars, num_bins, value_area_pct, window, std_threshold)
        s_idx, t_idx = np.array(picks).T
        rows[s_idx, t_idx], bins[s_idx, t_idx] = r, b
    labels = np.where(rows["n_bars"] > 0, rows["signal"], _lib.VP_NO_LABEL).astype(np.uint8)
    return rows, bins, labels


def frames_at(ohlcv: np.ndarray, picks, frame_bars: int, num_bins=20, value_area_pct=0.7, window=20, std_threshold=2.0):
    """rows [K], bins [K][B] and labels [K] of the frames ending at the (s, t) pairs `picks` of float32 OHLCV [5][S][N]
    (t < frame_bars - 1: the row of a bar without a frame)."""
    rows = np.empty(len(picks), dtype=ROW)
    bins = np.zeros((len(picks), num_bins))
    for k, (s, t) in enumerate(picks):
        if t < frame_bars - 1:
            row = empty_row()
            row["n_bars"] = row["valid"] = 0
        else:
            sl = slice(t - frame_bars + 1, t + 1)
            row, bins[k] = frame(*(ohlcv[f, s, sl].astype(np.float64) for f in range(5)), num_bins, value_area_pct,
                                 window, std_threshold)
        rows[k] = row
    return rows, bins, rows["signal"].astype(np.uint8)


def base_labels(frame_labels: np.ndarray, base_minute0: int, base_minutes: int, N: int, frame_minute0: int, k: int):
    """Labels of the frame clock (k-minute bars from frame_minute0) on the base clock: bar t carries the label of the
    last k-minute bar completed by the end of bar t (255 before the first)."""
    S, M = frame_labels.shape
    out = np.full((S, N), _lib.VP_NO_LABEL, dtype=np.uint8)
    for t in range(N):
        end = base_minute0 + (t + 1) * base_minutes          # minute at which bar t ends
        j = (end - frame_minute0) // k - 1                   # last k-minute bar ending at or before it
        if 0 <= j < M:
            out[:, t] = frame_labels[:, j]
    return out
