"""Plain Python / NumPy restatement of b200bt_market_monitor and b200bt_indicator_combinations (csrc/market_monitor.cu):
the market monitor's snapshot on completed-kline frames and services/utils/indicator_combinations.py's fifteen
combinations, written as the reference's expressions on Python floats (np.float64 where the reference's value is a
numpy float64), with the kernel's fixed summation orders.  Used by the CPU tests against the reference's fixture and by
the GPU tests against the kernel."""
from __future__ import annotations

import math

import numpy as np

from ai_crypto_trader_b200 import _lib

DAY_BARS = 1440


# ---- rounding ----------------------------------------------------------------------------------------------------
def round_py(x: float) -> float:
    """round(x, 4) of a Python float (correctly rounded decimal); an int stays an int."""
    return round(x, 4) if isinstance(x, int) else round(float(x), 4)


def round_np(x) -> float:
    """round(x, 4) of a numpy float64: rint(x * 1e4) / 1e4."""
    return float(round(np.float64(x), 4))


def roundings_disagree(x: float) -> bool:
    a, b = round_py(x), round_np(x)
    return not (a == b and math.copysign(1, a) == math.copysign(1, b)) and not (math.isnan(a) and math.isnan(b))


# ---- the combination step ------------------------------------------------------------------------------------------
def combinations(d: dict, unrounded: bool = False) -> dict:
    """calculate_combined_indicators on dict `d` of Python floats (trend a string; keys absent as in the reference).
    Returns the reference's dict; with unrounded=True, {output: value before round} instead (used to place fixture
    cases on rounding midpoints)."""
    for field in ('rsi', 'macd', 'stoch_k', 'williams_r', 'bb_position', 'price_change_1m', 'price_change_5m', 'trend',
                  'trend_strength'):
        if field not in d:
            return {'error': f"Missing required field: {field}"}
    raw = {}

    def R(name, x, numpy_value):
        raw[name] = x
        return round_np(x) if numpy_value else round_py(x)

    rsi, macd, stoch, wr, bb = d['rsi'], d['macd'], d['stoch_k'], d['williams_r'], d['bb_position']
    pc1, pc5, ts, trend = d['price_change_1m'], d['price_change_5m'], d['trend_strength'], d['trend']
    up, down = trend == 'uptrend', trend == 'downtrend'
    out = {}
    with np.errstate(all="ignore"):
        td = 1 if up else (-1 if down else 0)
        out['trend_confirmation'] = R('trend_confirmation', (0.6 * td * ts) + (0.4 * np.tanh(macd * 5)), True)

        tb = up
        agreements = sum([1 if (rsi > 50) == tb else 0, 1 if (macd > 0) == tb else 0, 1 if (wr > -50) == tb else 0])
        out['momentum_trend_alignment'] = R('momentum_trend_alignment', agreements / 3.0 * min(1.0, ts), False)

        es, em = d.get('ema_12', None), d.get('ema_26', None)
        try:
            if es is None or em is None:
                if up:
                    score, state = 0.5 + (ts / 2), 'bullish' if ts > 0.3 else 'neutral'
                elif down:
                    score, state = 0.5 - (ts / 2), 'bearish' if ts > 0.3 else 'neutral'
                else:
                    score, state = 0.5, 'neutral'
            elif es > em:
                score = min(1.0, 0.5 + ((es - em) / em * 100 * 0.1))
                state = 'bullish' if score > 0.7 else 'neutral'
            else:
                score = max(0.0, 0.5 - ((em - es) / em * 100 * 0.1))
                state = 'bearish' if score < 0.3 else 'neutral'
            out['triple_moving_average'] = {'score': R('tma_score', score, False), 'state': state}
        except ZeroDivisionError:
            out['triple_moving_average'] = None

        if 'price_change_3m' in d:
            volatility = sum([abs(pc1), abs(d['price_change_3m']), abs(pc5)]) / 3
            signals = [(rsi - 50) / 50, (wr + 50) / 50, np.tanh(macd * 10)]
            vf = min(3.0, max(0.5, volatility)) / 3.0
            adj = sum(signals) / len(signals) * (0.5 + vf)
            out['volatility_adjusted_momentum'] = R('volatility_adjusted_momentum', max(-1.0, min(1.0, adj)), True)
        else:
            out['volatility_adjusted_momentum'] = None

        out['volatility_trend_score'] = R('volatility_trend_score', (0.7 * (abs(bb - 0.5) * 2)) + (0.3 * ts), False)

        sig = [(rsi > 70, rsi < 30, min(1.0, max(0.0, abs(rsi - 50) / 30))),
               (wr > -20, wr < -80, min(1.0, max(0.0, abs(wr + 50) / 30))),
               (stoch > 80, stoch < 20, min(1.0, max(0.0, abs(stoch - 50) / 30)))]
        nob, nos = sum(1 for s in sig if s[0]), sum(1 for s in sig if s[1])
        sob = sum(s[2] for s in sig if s[0]) / nob if nob else 0
        sos = sum(s[2] for s in sig if s[1]) / nos if nos else 0
        if nob >= 2:
            signal, strength, agreement = 'overbought', sob, nob / 3.0
        elif nos >= 2:
            signal, strength, agreement = 'oversold', sos, nos / 3.0
        else:
            signal, strength, agreement = 'neutral', 0.0, 0.0
        out['oscillator_consensus'] = {'signal': signal, 'strength': R('osc_strength', strength, False),
                                       'agreement': R('osc_agreement', agreement, False)}

        if rsi <= 30:
            v = rsi / 30
        elif rsi >= 70:
            v = 0.67 + ((rsi - 70) / 30) * 0.33
        else:
            v = 0.33 + ((rsi - 30) / 40) * 0.34
        out['stoch_rsi'] = R('stoch_rsi', v, False)

        r5 = d.get('rsi_5m', None)
        if r5 is None:
            r5 = d.get('rsi_3m', rsi)
        if rsi < 30 and r5 < 30:
            s = 'strong_oversold'
        elif rsi < 30:
            s = 'oversold'
        elif rsi > 70 and r5 > 70:
            s = 'strong_overbought'
        elif rsi > 70:
            s = 'overbought'
        elif rsi > 50 and r5 > 50:
            s = 'bullish'
        elif rsi < 50 and r5 < 50:
            s = 'bearish'
        else:
            s = 'neutral'
        out['double_rsi'] = {'signal': s, 'divergence': R('drsi_divergence', rsi - r5, False)}

        pm = (0.4 * pc1) + (0.6 * pc5)
        volume = d.get('volume', 1.0)
        avg = d.get('avg_volume', volume)
        ratio = volume / avg if avg > 0 else 1.0
        out['volume_weighted_price_momentum'] = R('vwpm', np.tanh(pm * min(2.0, ratio) / 5.0), True)

        volume = d.get('volume', 0)
        avg = d.get('avg_volume', volume)
        ratio = volume / avg if avg > 0 else 1.0
        if abs(pc1) < 0.1:
            c, st = 'neutral', 0
        elif pc1 > 0 and ratio > 1.2:
            c, st = 'strong_bullish', min(1.0, ratio - 1.0)
        elif pc1 > 0:
            c, st = 'weak_bullish', max(0.0, min(0.5, (ratio - 0.8) / 0.4))
        elif pc1 < 0 and ratio > 1.2:
            c, st = 'strong_bearish', min(1.0, ratio - 1.0)
        elif pc1 < 0:
            c, st = 'weak_bearish', max(0.0, min(0.5, (ratio - 0.8) / 0.4))
        else:
            c, st = 'neutral', 0
        out['volume_price_confirmation'] = {'confirmation': c, 'strength': R('vpc_strength', st, False)}

        direction = 1 if up else (-1 if down else 0)
        if direction > 0:
            rf, bf = ((rsi - 50) / 50 if rsi > 50 else 0), bb
        elif direction < 0:
            rf, bf = ((50 - rsi) / 50 if rsi < 50 else 0), 1 - bb
        else:
            rf, bf = 1 - (abs(rsi - 50) / 25), 1 - abs(bb - 0.5) * 2
        mf = np.tanh(macd * 20)
        cs = 0.4 * ts + 0.25 * rf + 0.25 * abs(mf) + 0.1 * bf
        if direction != 0:
            ind = 1 if (rsi > 50 and macd > 0) else (-1 if (rsi < 50 and macd < 0) else 0)
            conf, conf_np = 0.5 + (0.5 * (direction == np.sign(ind))), True
        else:
            conf, conf_np = 0.5 + (0.3 * ((abs(rsi - 50) < 10) and (abs(macd) < 0.0005))), False
        out['trend_strength_index'] = {'direction': direction, 'strength': R('tsi_strength', cs, True),
                                       'confidence': R('tsi_confidence', conf, conf_np)}

        if 'price_change_3m' in d:
            if ts > 0.6:
                regime, conf = 'trending', min(1.0, ts * 1.1)
            elif volatility > 2.0:
                regime, conf = 'volatile', min(1.0, volatility / 3.0)
            else:
                regime, conf = 'ranging', min(1.0, 0.5 + (1 - ts) * (1 - abs(bb - 0.5) * 2))
            out['market_regime_indicator'] = {'regime': regime, 'confidence': R('regime_confidence', conf, False)}
        else:
            out['market_regime_indicator'] = None

        p, signals = 0.0, []
        for cond_up, cond_dn, inc, names in ((rsi > 70, rsi < 30, 0.25, ('rsi_overbought', 'rsi_oversold')),
                                             (wr > -20, wr < -80, 0.2, ('williams_overbought', 'williams_oversold')),
                                             (bb > 0.9, bb < 0.1, 0.15, ('price_near_upper_band', 'price_near_lower_band')),
                                             (rsi < 60, rsi > 40, 0.2, ('potential_bearish_divergence',
                                                                        'potential_bullish_divergence'))):
            if up and cond_up:
                p += inc
                signals.append(names[0])
            elif down and cond_dn:
                p += inc
                signals.append(names[1])
        out['reversal_probability'] = {'probability': R('reversal_probability', min(0.95, p), False), 'signals': signals}

        bd, conf = 0, 0.0
        if pc5 > 1.0 and bb > 0.8:
            bd, conf = 1, 0.5 + (0.5 * min(1.0, (rsi - 50) / 30))
        elif pc5 < -1.0 and bb < 0.2:
            bd, conf = -1, 0.5 + (0.5 * min(1.0, (50 - rsi) / 30))
        side = 'bullish' if bd > 0 else 'bearish'
        status = 'none' if bd == 0 else ('strong_' if conf > 0.8 else 'confirmed_' if conf > 0.5 else 'potential_') + side
        out['breakout_confirmation'] = {'direction': bd, 'confirmation': R('breakout_confirmation', conf, False),
                                        'status': status}

        div, strength = 'none', 0.0
        if up and pc5 > 0 and rsi < 50:
            div, strength = 'bearish_rsi', 0.5 + (0.5 * (1 - (rsi / 50)))
        elif down and pc5 < 0 and rsi > 50:
            div, strength = 'bullish_rsi', 0.5 + (0.5 * ((rsi - 50) / 50))
        ms, mdiv = 0.0, None
        if up and pc5 > 0 and macd < 0:
            mdiv, ms = 'bearish_macd', 0.6 + (0.4 * min(1.0, abs(macd) * 1000))
        elif down and pc5 < 0 and macd > 0:
            mdiv, ms = 'bullish_macd', 0.6 + (0.4 * min(1.0, abs(macd) * 1000))
        if ms > strength:
            div, strength = mdiv, ms
        out['divergence_detector'] = {'divergence': div, 'strength': R('divergence_strength', strength, False)}
    order = list(_lib.MM_COMBINATIONS)
    return raw if unrounded else {k: out[k] for k in order}


# ---- the snapshot --------------------------------------------------------------------------------------------------
def _ewm_alpha(com):
    a = 1.0 / (1.0 + com)
    return 1.0 - a, a


def _ewm(values, om, a):
    w = values[0]
    den = om + a
    for x in values[1:]:
        if w != x:
            w = (om * w + a * x) / den
    return w


def rsi_macd(close):
    """RSI(14) and the MACD line at the last of the closes (a frame), the kernel's ewm loops."""
    c = [float(x) for x in close]
    n = len(c)
    om_r, a_r = _ewm_alpha((1 - 1 / 14) / (1 / 14))
    ups, dns = [0.0], [-0.0]
    for i in range(1, n):
        dlt = c[i] - c[i - 1]
        ups.append(dlt if dlt > 0 else 0.0)
        dns.append(-(dlt if dlt < 0 else 0.0))
    up, dn = _ewm(ups, om_r, a_r), _ewm(dns, om_r, a_r)
    with np.errstate(all="ignore"):
        rsi = math.nan if n < 14 else (100.0 if dn == 0 else float(100.0 - 100.0 / (1.0 + np.float64(up) / dn)))
    fast = _ewm(c, *_ewm_alpha((12 - 1) / 2))
    slow = _ewm(c, *_ewm_alpha((26 - 1) / 2))
    return rsi, (math.nan if n < 26 else fast - slow)


def _mean(x):
    s = 0.0
    for v in x:
        s += float(v)
    return s / len(x)


def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def snapshot(f1, f3, f5, f15) -> dict:
    """calculate_technical_indicators on frames given as dicts of float arrays (open / high / low / close on the
    1-minute clock, open / close on the others; W klines on the 1-, 3- and 5-minute clocks, at least one on the
    15-minute clock), with the kernel's window orders.  The trend
    is the reference's string."""
    W = len(f1["close"])
    close = float(f1["close"][-1])
    rsi, macd = rsi_macd(f1["close"])
    rsi3, macd3 = rsi_macd(f3["close"])
    rsi5, macd5 = rsi_macd(f5["close"])
    nan = math.nan
    if W >= 14:
        lo, hi = float(np.min(f1["low"][-14:])), float(np.max(f1["high"][-14:]))
        stoch, will = _div(100.0 * (close - lo), hi - lo), _div(-100.0 * (hi - close), hi - lo)
    else:
        stoch = will = nan
    sma20 = sma50 = sma20_5 = bbp = nan
    if W >= 20:
        x = f1["close"][-20:]
        sma20 = _mean(x)
        ss = 0.0
        for v in x:
            dv = float(v) - sma20
            ss += dv * dv
        sd = math.sqrt(ss / 20)
        hb, lb = sma20 + 2.0 * sd, sma20 - 2.0 * sd
        bbp = nan if hb - lb == 0 else (close - lb) / (hb - lb)
        sma20_5 = _mean(f5["close"][-20:])
    if W >= 50:
        sma50 = _mean(f1["close"][-50:])
    pc = [_div(close - float(f["open"][-1]), float(f["open"][-1])) * 100 for f in (f1, f3, f5, f15)]
    s1 = _div(close - sma20, sma20) * 100
    s5 = _div(close - sma20_5, sma20_5) * 100
    if close > sma20 and sma20 > sma50:
        trend = 'uptrend'
    elif close < sma20 and sma20 < sma50:
        trend = 'downtrend'
    else:
        trend = 'sideways'
    return {'rsi': rsi, 'rsi_3m': rsi3, 'rsi_5m': rsi5, 'stoch_k': stoch, 'macd': macd, 'macd_3m': macd3,
            'macd_5m': macd5, 'williams_r': will, 'bb_position': bbp, 'trend': trend,
            'trend_strength': abs(s1 * 0.6 + s5 * 0.4), 'price_change_1m': pc[0], 'price_change_3m': pc[1],
            'price_change_5m': pc[2], 'price_change_15m': pc[3]}


def completed_kline(t: int, minute0: int, k: int) -> int:
    """b200bt_align's rule on a 1-minute clock: the last k-minute kline completed by the close of bar t (-1: none)."""
    m = minute0 + t
    b = m // k - minute0 // k
    return b if (m + 1) // k != m // k else b - 1


def klines(ohlcv_s: np.ndarray, minute0: int, k: int, j_lo: int, j_hi: int) -> dict:
    """open / close float64 of k-minute klines j_lo .. j_hi of one symbol's 1-minute [5][N] (b200bt_resample:
    epoch-aligned buckets clipped to the series)."""
    m_lo = (minute0 // k + np.arange(j_lo, j_hi + 1)) * k
    t_lo = np.maximum(m_lo - minute0, 0)
    t_hi = np.minimum(m_lo + k - 1 - minute0, ohlcv_s.shape[1] - 1)
    return {"open": ohlcv_s[0, t_lo].astype(np.float64), "close": ohlcv_s[3, t_hi].astype(np.float64)}


def row_at(ohlcv: np.ndarray, minute0: int, s: int, t: int, W: int, min_pct: float = 0.5,
           min_volume: float = 50000.0) -> dict:
    """The kernel's row (s, t) as a dict of the structured row's fields (snapshot and combination halves), from host
    float32 [5][S][N]."""
    x = ohlcv[:, s]
    j = {k: completed_kline(t, minute0, k) for k in (3, 5, 15)}
    if t - W + 1 < 0 or j[3] - W + 1 < 0 or j[5] - W + 1 < 0 or j[15] < 0:
        return {"valid": 0}
    f1 = {"open": x[0, t - W + 1:t + 1].astype(np.float64), "high": x[1, t - W + 1:t + 1].astype(np.float64),
          "low": x[2, t - W + 1:t + 1].astype(np.float64), "close": x[3, t - W + 1:t + 1].astype(np.float64)}
    frames = [f1] + [klines(x, minute0, k, j[k] - W + 1, j[k]) for k in (3, 5)] + [klines(x, minute0, 15, j[15], j[15])]
    snap = snapshot(*frames)
    vol = 0.0
    for v in x[4, max(0, t - DAY_BARS + 1):t + 1]:
        vol += float(v)
    close = float(x[3, t])
    d = dict(snap, current_price=close, avg_volume=vol * close)
    out = {"valid": 1, "present": _lib.MM_HAS["rsi_3m"] | _lib.MM_HAS["rsi_5m"] | _lib.MM_HAS["price_change_3m"]
           | _lib.MM_HAS["avg_volume"], "opportunity": int(abs(d["price_change_1m"]) >= min_pct and d["avg_volume"] >= min_volume)}
    out.update({k: v for k, v in d.items()})
    out["combined"] = combinations(d)
    return out
