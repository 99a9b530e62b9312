// Market monitor (sm_90a): services/market_monitor_service.py's market_update for every 1-minute bar of a market's history
// (calculate_technical_indicators :219-301 on the 1-, 3-, 5- and 15-minute frames, the ticker fields :432-433, the
// trading-opportunity test :561-562) and the fifteen combinations of services/utils/indicator_combinations.py (:96-679).
//
// monitor_kernel       one thread per (1-minute bar t, symbol): the frames' indicators straight from the klines (the
//                      frames of neighbouring threads overlap, so the reads hit L1), then combine() on the row.
// combinations_kernel  one thread per caller-filled row: combine() alone.
//
// Every operation is rounded on its own through the __d*_rn intrinsics, so no FMA contraction changes a bit.
#include <math.h>
#include "common.cuh"

namespace b200bt {

constexpr int MM_THREADS = 128;
constexpr int MM_DAY_BARS = 1440;        // the 24-hour ticker's volume window
constexpr int MM_RSI = 14, MM_FAST = 12, MM_SLOW = 26, MM_STOCH = 14, MM_BB = 20, MM_SMA_LONG = 50;
enum { MM_UP = 0, MM_DOWN = 1, MM_SIDEWAYS = 2 };
enum { TMA_BULLISH = 0, TMA_BEARISH = 1, TMA_NEUTRAL = 2 };
enum { OSC_OVERBOUGHT = 0, OSC_OVERSOLD = 1, OSC_NEUTRAL = 2 };
enum { DRSI_STRONG_OVERSOLD = 0, DRSI_OVERSOLD, DRSI_STRONG_OVERBOUGHT, DRSI_OVERBOUGHT, DRSI_BULLISH, DRSI_BEARISH,
       DRSI_NEUTRAL };
enum { VPC_STRONG_BULLISH = 0, VPC_WEAK_BULLISH, VPC_STRONG_BEARISH, VPC_WEAK_BEARISH, VPC_NEUTRAL };
enum { REGIME_TRENDING = 0, REGIME_VOLATILE, REGIME_RANGING };
enum { BO_NONE = 0, BO_STRONG_BULLISH, BO_STRONG_BEARISH, BO_CONFIRMED_BULLISH, BO_CONFIRMED_BEARISH,
       BO_POTENTIAL_BULLISH, BO_POTENTIAL_BEARISH };
enum { DIV_NONE = 0, DIV_BEARISH_RSI, DIV_BULLISH_RSI, DIV_BEARISH_MACD, DIV_BULLISH_MACD };
// combination indices (calculate_combined_indicators' dict order)
enum { C_TREND_CONFIRMATION = 0, C_MOMENTUM_TREND_ALIGNMENT, C_TRIPLE_MA, C_VOLATILITY_ADJUSTED_MOMENTUM,
       C_VOLATILITY_TREND_SCORE, C_OSCILLATOR_CONSENSUS, C_STOCH_RSI, C_DOUBLE_RSI, C_VWPM, C_VPC,
       C_TREND_STRENGTH_INDEX, C_MARKET_REGIME, C_REVERSAL, C_BREAKOUT, C_DIVERGENCE };

__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000ll); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }

// Python's min(a, b) / max(a, b): the first argument unless the second compares less / greater (so NaN loses or wins by
// position).
__device__ __forceinline__ double py_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }

// round(x, 4) of a numpy float64: np.round multiplies by 10^4, rounds half to even and divides.
__device__ __forceinline__ double round_np(double x) { return dvd(rint(mul(x, 1e4)), 1e4); }

// round(x, 4) of a Python float: the integer p nearest the EXACT x * 10^4 (ties to even), then p / 10^4 correctly rounded
// (the double nearest the decimal, as CPython's dtoa-based round gives).  y = x * 1e4 rounded and its exact residue
// r = x * 1e4 - y (one fma) place the exact product against p +- 1/2: only where y itself is a tie (rint took the even
// neighbour) can r move the result.  Exact for |x * 10^4| < 2^52; non-finite values are returned as they are.
__device__ __forceinline__ double round_py(double x) {
    if (!isfinite(x)) return x;
    const double y = mul(x, 1e4);
    const double r = fma(x, 1e4, -y);
    double p = rint(y);
    const double d = sub(y, p);                     // exact: y and p are neighbours on the integer grid
    if (d == 0.5 && r > 0.0) p = add(p, 1.0);       // the exact product lies above the tie p + 1/2
    else if (d == -0.5 && r < 0.0) p = sub(p, 1.0); // ... below the tie p - 1/2
    return dvd(p, 1e4);
}

// pandas' ewm(adjust=False).mean() step (window_aggregations.ewm): skip when the running mean equals the new value.
struct Ewm {
    double om, a, den;                              // 1 - alpha, alpha, (1 - alpha) + alpha
    __device__ explicit Ewm(double com) {
        a = dvd(1.0, add(1.0, com));
        om = sub(1.0, a);
        den = add(om, a);
    }
    __device__ __forceinline__ double step(double w, double x) const {
        if (w == x) return w;
        const double v = add(mul(om, w), mul(a, x));
        return den == 1.0 ? v : dvd(v, den);
    }
};

__device__ __forceinline__ double ewm_com_alpha(double alpha) { return dvd(sub(1.0, alpha), alpha); }
__device__ __forceinline__ double ewm_com_span(int span) { return dvd(sub((double)span, 1.0), 2.0); }

// RSI(14) and MACD(12, 26) line at the last of n closes c[0 .. n-1] (stride 1).
struct Osc { double rsi, macd; };
__device__ Osc rsi_macd(const float* __restrict__ c, int n) {
    const Ewm er(ewm_com_alpha(dvd(1.0, (double)MM_RSI)));
    const Ewm ef(ewm_com_span(MM_FAST)), es(ewm_com_span(MM_SLOW));
    double prev = (double)c[0];
    double up = 0.0, dn = -0.0;                     // diff.where(diff > 0, 0.0) / -diff.where(diff < 0, 0.0) of NaN
    double fast = prev, slow = prev;
    for (int i = 1; i < n; ++i) {
        const double x = (double)c[i];
        const double d = sub(x, prev);
        up = er.step(up, d > 0.0 ? d : 0.0);
        dn = er.step(dn, -(d < 0.0 ? d : 0.0));
        fast = ef.step(fast, x);
        slow = es.step(slow, x);
        prev = x;
    }
    Osc o;
    if (n < MM_RSI) o.rsi = qnan();
    else o.rsi = dn == 0.0 ? 100.0 : sub(100.0, dvd(100.0, add(1.0, dvd(up, dn))));
    o.macd = (n < MM_SLOW) ? qnan() : sub(fast, slow);    // n >= 26 implies n >= 12
    return o;
}

__device__ double window_mean(const float* __restrict__ c, int w) {
    double s = 0.0;
    for (int i = 0; i < w; ++i) s = add(s, (double)c[i]);
    return dvd(s, (double)w);
}

// ---------------------------------------------------------------------------------------------------------------------
// The combination step: calculate_combined_indicators on the snapshot half of r, read as Python floats.
__device__ void combine(b200bt_monitor_row& r) {
    const double rsi = r.rsi, macd = r.macd, stoch = r.stoch_k, wr = r.williams_r, bb = r.bb_position;
    const double pc1 = r.price_change_1m, pc3 = r.price_change_3m, pc5 = r.price_change_5m, ts = r.trend_strength;
    const bool up = r.trend == MM_UP, down = r.trend == MM_DOWN;
    const int P = r.present;
    int computed = (1 << B200BT_MM_COMBINATIONS) - 1;  // cleared below for the reference's None entries

    // trend_confirmation (:96-111): numpy (np.tanh)
    {
        const int td = up ? 1 : (down ? -1 : 0);
        const double v = add(mul(mul(0.6, (double)td), ts), mul(0.4, tanh(mul(macd, 5.0))));
        r.trend_confirmation = round_np(v);
    }
    // momentum_trend_alignment (:113-142)
    {
        const bool tb = up;
        const int agreements = ((rsi > 50.0) == tb) + ((macd > 0.0) == tb) + ((wr > -50.0) == tb);
        r.momentum_trend_alignment = round_py(mul(dvd((double)agreements, 3.0), py_min(1.0, ts)));
    }
    // triple_moving_average (:144-182): the trend proxy unless ema_12 and ema_26 are both present
    {
        bool ok = true;
        double score;
        int state;
        if (!(P & B200BT_MM_HAS_EMA_12) || !(P & B200BT_MM_HAS_EMA_26)) {
            if (up) {
                score = add(0.5, dvd(ts, 2.0));
                state = ts > 0.3 ? TMA_BULLISH : TMA_NEUTRAL;
            } else if (down) {
                score = sub(0.5, dvd(ts, 2.0));
                state = ts > 0.3 ? TMA_BEARISH : TMA_NEUTRAL;
            } else {
                score = 0.5;
                state = TMA_NEUTRAL;
            }
        } else {
            const double es = r.ema_12, em = r.ema_26;
            if (em == 0.0) {                        // Python float division by zero: ZeroDivisionError
                ok = false;
                score = qnan();
                state = B200BT_MM_NO_LABEL;
            } else if (es > em) {
                const double diff = mul(dvd(sub(es, em), em), 100.0);
                score = py_min(1.0, add(0.5, mul(diff, 0.1)));
                state = score > 0.7 ? TMA_BULLISH : TMA_NEUTRAL;
            } else {
                const double diff = mul(dvd(sub(em, es), em), 100.0);
                score = py_max(0.0, sub(0.5, mul(diff, 0.1)));
                state = score < 0.3 ? TMA_BEARISH : TMA_NEUTRAL;
            }
        }
        r.tma_score = ok ? round_py(score) : qnan();
        r.tma_state = state;
        if (!ok) computed &= ~(1 << C_TRIPLE_MA);
    }
    // volatility = sum([|pc1|, |pc3|, |pc5|]) / 3 (KeyError without price_change_3m)
    const bool has_pc3 = P & B200BT_MM_HAS_PRICE_CHANGE_3M;
    const double volatility = has_pc3 ? dvd(add(add(add(0.0, fabs(pc1)), fabs(pc3)), fabs(pc5)), 3.0) : qnan();
    // volatility_adjusted_momentum (:186-220): numpy (np.tanh in the sum), clamped by Python min / max
    if (has_pc3) {
        const double rn = dvd(sub(rsi, 50.0), 50.0);
        const double wn = dvd(add(wr, 50.0), 50.0);
        const double mt = tanh(mul(macd, 10.0));
        const double vf = dvd(py_min(3.0, py_max(0.5, volatility)), 3.0);
        const double comp = dvd(add(add(add(0.0, rn), wn), mt), 3.0);
        const double adj = mul(comp, add(0.5, vf));
        r.volatility_adjusted_momentum = round_np(py_max(-1.0, py_min(1.0, adj)));
    } else {
        r.volatility_adjusted_momentum = qnan();
        computed &= ~(1 << C_VOLATILITY_ADJUSTED_MOMENTUM);
    }
    // volatility_trend_score (:222-240)
    r.volatility_trend_score = round_py(add(mul(0.7, mul(fabs(sub(bb, 0.5)), 2.0)), mul(0.3, ts)));
    // oscillator_consensus (:244-311)
    {
        const bool ob[3] = {rsi > 70.0, wr > -20.0, stoch > 80.0};
        const bool os[3] = {rsi < 30.0, wr < -80.0, stoch < 20.0};
        const double st[3] = {py_min(1.0, py_max(0.0, dvd(fabs(sub(rsi, 50.0)), 30.0))),
                              py_min(1.0, py_max(0.0, dvd(fabs(add(wr, 50.0)), 30.0))),
                              py_min(1.0, py_max(0.0, dvd(fabs(sub(stoch, 50.0)), 30.0)))};
        int nob = 0, nos = 0;
        double sob = 0.0, sos = 0.0;
        for (int i = 0; i < 3; ++i) {
            if (ob[i]) { ++nob; sob = add(sob, st[i]); }
            if (os[i]) { ++nos; sos = add(sos, st[i]); }
        }
        double strength, agreement;
        if (nob >= 2) {
            r.osc_signal = OSC_OVERBOUGHT;
            strength = dvd(sob, (double)nob);
            agreement = dvd((double)nob, 3.0);
        } else if (nos >= 2) {
            r.osc_signal = OSC_OVERSOLD;
            strength = dvd(sos, (double)nos);
            agreement = dvd((double)nos, 3.0);
        } else {
            r.osc_signal = OSC_NEUTRAL;
            strength = 0.0;
            agreement = 0.0;
        }
        r.osc_strength = round_py(strength);
        r.osc_agreement = round_py(agreement);
    }
    // stoch_rsi (:313-330)
    {
        double v;
        if (rsi <= 30.0) v = dvd(rsi, 30.0);
        else if (rsi >= 70.0) v = add(0.67, mul(dvd(sub(rsi, 70.0), 30.0), 0.33));
        else v = add(0.33, mul(dvd(sub(rsi, 30.0), 40.0), 0.34));
        r.stoch_rsi = round_py(v);
    }
    // double_rsi (:332-366): rsi_5m, else rsi_3m, else rsi
    {
        const double r5 = (P & B200BT_MM_HAS_RSI_5M) ? r.rsi_5m : ((P & B200BT_MM_HAS_RSI_3M) ? r.rsi_3m : rsi);
        int sig;
        if (rsi < 30.0 && r5 < 30.0) sig = DRSI_STRONG_OVERSOLD;
        else if (rsi < 30.0) sig = DRSI_OVERSOLD;
        else if (rsi > 70.0 && r5 > 70.0) sig = DRSI_STRONG_OVERBOUGHT;
        else if (rsi > 70.0) sig = DRSI_OVERBOUGHT;
        else if (rsi > 50.0 && r5 > 50.0) sig = DRSI_BULLISH;
        else if (rsi < 50.0 && r5 < 50.0) sig = DRSI_BEARISH;
        else sig = DRSI_NEUTRAL;
        r.drsi_signal = sig;
        r.drsi_divergence = round_py(sub(rsi, r5));
    }
    const bool has_avg = P & B200BT_MM_HAS_AVG_VOLUME, has_vol = P & B200BT_MM_HAS_VOLUME;
    // volume_weighted_price_momentum (:370-399): volume defaults to 1.0, avg_volume to volume; numpy (np.tanh)
    {
        const double pm = add(mul(0.4, pc1), mul(0.6, pc5));
        const double volume = has_vol ? r.volume : 1.0;
        const double avg = has_avg ? r.avg_volume : volume;
        const double ratio = avg > 0.0 ? dvd(volume, avg) : 1.0;
        r.vwpm = round_np(tanh(dvd(mul(pm, py_min(2.0, ratio)), 5.0)));
    }
    // volume_price_confirmation (:401-437): volume defaults to 0, avg_volume to volume
    {
        const double volume = has_vol ? r.volume : 0.0;
        const double avg = has_avg ? r.avg_volume : volume;
        const double ratio = avg > 0.0 ? dvd(volume, avg) : 1.0;
        int conf;
        double strength;
        if (fabs(pc1) < 0.1) { conf = VPC_NEUTRAL; strength = 0.0; }
        else if (pc1 > 0.0 && ratio > 1.2) { conf = VPC_STRONG_BULLISH; strength = py_min(1.0, sub(ratio, 1.0)); }
        else if (pc1 > 0.0) { conf = VPC_WEAK_BULLISH; strength = py_max(0.0, py_min(0.5, dvd(sub(ratio, 0.8), 0.4))); }
        else if (pc1 < 0.0 && ratio > 1.2) { conf = VPC_STRONG_BEARISH; strength = py_min(1.0, sub(ratio, 1.0)); }
        else if (pc1 < 0.0) { conf = VPC_WEAK_BEARISH; strength = py_max(0.0, py_min(0.5, dvd(sub(ratio, 0.8), 0.4))); }
        else { conf = VPC_NEUTRAL; strength = 0.0; }
        r.vpc_confirmation = conf;
        r.vpc_strength = round_py(strength);
    }
    // trend_strength_index (:441-503): strength numpy (np.tanh); confidence numpy when trending (np.sign), else Python
    {
        const int dir = up ? 1 : (down ? -1 : 0);
        double rf, bf;
        if (dir > 0) { rf = rsi > 50.0 ? dvd(sub(rsi, 50.0), 50.0) : 0.0; bf = bb; }
        else if (dir < 0) { rf = rsi < 50.0 ? dvd(sub(50.0, rsi), 50.0) : 0.0; bf = sub(1.0, bb); }
        else { rf = sub(1.0, dvd(fabs(sub(rsi, 50.0)), 25.0)); bf = sub(1.0, mul(fabs(sub(bb, 0.5)), 2.0)); }
        const double mf = tanh(mul(macd, 20.0));
        const double cs = add(add(add(mul(0.4, ts), mul(0.25, rf)), mul(0.25, fabs(mf))), mul(0.1, bf));
        r.tsi_direction = dir + 1;
        r.tsi_strength = round_np(cs);
        if (dir != 0) {
            const int ind = (rsi > 50.0 && macd > 0.0) ? 1 : ((rsi < 50.0 && macd < 0.0) ? -1 : 0);
            r.tsi_confidence = round_np(add(0.5, mul(0.5, dir == ind ? 1.0 : 0.0)));
        } else {
            const bool neutral = fabs(sub(rsi, 50.0)) < 10.0 && fabs(macd) < 0.0005;
            r.tsi_confidence = round_py(add(0.5, mul(0.3, neutral ? 1.0 : 0.0)));
        }
    }
    // market_regime_indicator (:505-538) (KeyError without price_change_3m)
    if (has_pc3) {
        double conf;
        if (ts > 0.6) { r.regime = REGIME_TRENDING; conf = py_min(1.0, mul(ts, 1.1)); }
        else if (volatility > 2.0) { r.regime = REGIME_VOLATILE; conf = py_min(1.0, dvd(volatility, 3.0)); }
        else {
            r.regime = REGIME_RANGING;
            const double re = mul(sub(1.0, ts), sub(1.0, mul(fabs(sub(bb, 0.5)), 2.0)));
            conf = py_min(1.0, add(0.5, re));
        }
        r.regime_confidence = round_py(conf);
    } else {
        r.regime = B200BT_MM_NO_LABEL;
        r.regime_confidence = qnan();
        computed &= ~(1 << C_MARKET_REGIME);
    }
    // reversal_probability (:540-593)
    {
        double p = 0.0;
        int sig = 0;
        if (up && rsi > 70.0) { p = add(p, 0.25); sig |= 1; }
        else if (down && rsi < 30.0) { p = add(p, 0.25); sig |= 2; }
        if (up && wr > -20.0) { p = add(p, 0.2); sig |= 4; }
        else if (down && wr < -80.0) { p = add(p, 0.2); sig |= 8; }
        if (up && bb > 0.9) { p = add(p, 0.15); sig |= 16; }
        else if (down && bb < 0.1) { p = add(p, 0.15); sig |= 32; }
        if (up && rsi < 60.0) { p = add(p, 0.2); sig |= 64; }
        else if (down && rsi > 40.0) { p = add(p, 0.2); sig |= 128; }
        r.reversal_probability = round_py(py_min(0.95, p));
        r.reversal_signals = sig;
    }
    // breakout_confirmation (:595-634)
    {
        int dir = 0;
        double conf = 0.0;
        if (pc5 > 1.0 && bb > 0.8) { dir = 1; conf = add(0.5, mul(0.5, py_min(1.0, dvd(sub(rsi, 50.0), 30.0)))); }
        else if (pc5 < -1.0 && bb < 0.2) { dir = -1; conf = add(0.5, mul(0.5, py_min(1.0, dvd(sub(50.0, rsi), 30.0)))); }
        int status;
        if (dir == 0) status = BO_NONE;
        else if (conf > 0.8) status = dir > 0 ? BO_STRONG_BULLISH : BO_STRONG_BEARISH;
        else if (conf > 0.5) status = dir > 0 ? BO_CONFIRMED_BULLISH : BO_CONFIRMED_BEARISH;
        else status = dir > 0 ? BO_POTENTIAL_BULLISH : BO_POTENTIAL_BEARISH;
        r.breakout_direction = dir;
        r.breakout_status = status;
        r.breakout_confirmation = round_py(conf);
    }
    // divergence_detector (:636-679)
    {
        int div = DIV_NONE;
        double strength = 0.0;
        if (up && pc5 > 0.0 && rsi < 50.0) { div = DIV_BEARISH_RSI; strength = add(0.5, mul(0.5, sub(1.0, dvd(rsi, 50.0)))); }
        else if (down && pc5 < 0.0 && rsi > 50.0) { div = DIV_BULLISH_RSI; strength = add(0.5, mul(0.5, dvd(sub(rsi, 50.0), 50.0))); }
        double ms = 0.0;
        int mdiv = DIV_NONE;
        if (up && pc5 > 0.0 && macd < 0.0) { mdiv = DIV_BEARISH_MACD; ms = add(0.6, mul(0.4, py_min(1.0, mul(fabs(macd), 1000.0)))); }
        else if (down && pc5 < 0.0 && macd > 0.0) { mdiv = DIV_BULLISH_MACD; ms = add(0.6, mul(0.4, py_min(1.0, mul(fabs(macd), 1000.0)))); }
        if (ms > strength) { div = mdiv; strength = ms; }
        r.divergence = div;
        r.divergence_strength = round_py(strength);
    }
    r.computed = computed;
}

__device__ void invalidate(b200bt_monitor_row& r) {
    double* d = &r.current_price;
    for (int i = 0; i < 19; ++i) d[i] = qnan();
    r.valid = 0;
    r.trend = B200BT_MM_NO_LABEL;
    r.present = 0;
    r.opportunity = 0;
    r.computed = 0;
    int* c = &r.tma_state;
    for (int i = 0; i < 8; ++i) c[i] = B200BT_MM_NO_LABEL;
    r.breakout_direction = 0;
    r.reversal_signals = 0;
    r.reserved = 0;
    double* e = &r.trend_confirmation;
    for (int i = 0; i < 17; ++i) e[i] = qnan();
}

// label of a row: the code of label field f, B200BT_MM_NO_LABEL where its combination is None or the row is not valid
__device__ __forceinline__ uint8_t label_of(const b200bt_monitor_row& r, int f) {
    if (!r.valid) return B200BT_MM_NO_LABEL;
    static constexpr int owner[B200BT_MM_LABEL_FIELDS - 1] = {C_TRIPLE_MA, C_OSCILLATOR_CONSENSUS, C_DOUBLE_RSI, C_VPC,
                                                              C_TREND_STRENGTH_INDEX, C_MARKET_REGIME, C_BREAKOUT,
                                                              C_DIVERGENCE};
    if (f == 0) return (uint8_t)r.trend;
    if (!(r.computed >> owner[f - 1] & 1)) return B200BT_MM_NO_LABEL;
    return (uint8_t)((&r.tma_state)[f - 1]);
}

struct Clock {
    const float* p;        // [5][S][M]
    int64_t M;
    int k;
};

__global__ void __launch_bounds__(MM_THREADS)
monitor_kernel(const float* __restrict__ ohlcv, int S, int64_t N, int64_t minute0, Clock c3, Clock c5, Clock c15,
               b200bt_monitor_params prm, b200bt_monitor_row* __restrict__ rows, uint8_t* __restrict__ labels) {
    const int s = blockIdx.y;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    const int W = prm.frame_bars;
    const int64_t plane = (int64_t)S * N;
    const float* o1 = ohlcv + (int64_t)s * N;
    const float* h1 = o1 + plane;
    const float* l1 = h1 + plane;
    const float* c1 = l1 + plane;
    const float* v1 = c1 + plane;
    const int64_t j3 = completed_bucket(t, minute0, 1, 3), j5 = completed_bucket(t, minute0, 1, 5);
    const int64_t j15 = completed_bucket(t, minute0, 1, 15);
    b200bt_monitor_row r;
    if (t - W + 1 < 0 || j3 - W + 1 < 0 || j5 - W + 1 < 0 || j15 < 0) {
        invalidate(r);
    } else {
        r.valid = 1;
        r.present = B200BT_MM_HAS_RSI_3M | B200BT_MM_HAS_RSI_5M | B200BT_MM_HAS_PRICE_CHANGE_3M | B200BT_MM_HAS_AVG_VOLUME;
        r.reserved = 0;
        r.volume = r.ema_12 = r.ema_26 = qnan();
        const double close = (double)c1[t];
        // ticker: 24-hour base volume * price
        double vol = 0.0;
        for (int64_t i = t - MM_DAY_BARS + 1 < 0 ? 0 : t - MM_DAY_BARS + 1; i <= t; ++i) vol = add(vol, (double)v1[i]);
        r.current_price = close;
        r.avg_volume = mul(vol, close);
        // 1-minute frame: bars t - W + 1 .. t
        const int64_t f1 = t - W + 1;
        const Osc a1 = rsi_macd(c1 + f1, W);
        r.rsi = a1.rsi;
        r.macd = a1.macd;
        if (W >= MM_STOCH) {
            double lo = (double)l1[t], hi = (double)h1[t];
            for (int64_t i = t - MM_STOCH + 1; i < t; ++i) {
                lo = fmin(lo, (double)l1[i]);
                hi = fmax(hi, (double)h1[i]);
            }
            r.stoch_k = dvd(mul(100.0, sub(close, lo)), sub(hi, lo));
            r.williams_r = dvd(mul(-100.0, sub(hi, close)), sub(hi, lo));
        } else {
            r.stoch_k = r.williams_r = qnan();
        }
        double sma20 = qnan(), sma50 = qnan();
        if (W >= MM_BB) {
            const float* x = c1 + t - MM_BB + 1;
            sma20 = window_mean(x, MM_BB);
            double ss = 0.0;
            for (int i = 0; i < MM_BB; ++i) {
                const double d = sub((double)x[i], sma20);
                ss = add(ss, mul(d, d));
            }
            const double sd = __dsqrt_rn(dvd(ss, (double)MM_BB));
            const double hb = add(sma20, mul(2.0, sd)), lb = sub(sma20, mul(2.0, sd));
            const double range = sub(hb, lb);
            r.bb_position = range == 0.0 ? qnan() : dvd(sub(close, lb), range);
        } else {
            r.bb_position = qnan();
        }
        if (W >= MM_SMA_LONG) sma50 = window_mean(c1 + t - MM_SMA_LONG + 1, MM_SMA_LONG);
        // 3- and 5-minute frames
        const float* c3c = c3.p + 3 * (int64_t)S * c3.M + (int64_t)s * c3.M;
        const float* o3 = c3.p + (int64_t)s * c3.M;
        const Osc a3 = rsi_macd(c3c + j3 - W + 1, W);
        const float* c5c = c5.p + 3 * (int64_t)S * c5.M + (int64_t)s * c5.M;
        const float* o5 = c5.p + (int64_t)s * c5.M;
        const Osc a5 = rsi_macd(c5c + j5 - W + 1, W);
        r.rsi_3m = a3.rsi;
        r.macd_3m = a3.macd;
        r.rsi_5m = a5.rsi;
        r.macd_5m = a5.macd;
        const double sma20_5 = W >= MM_BB ? window_mean(c5c + j5 - MM_BB + 1, MM_BB) : qnan();
        // price changes against the open of each clock's last kline
        const double op1 = (double)o1[t], op3 = (double)o3[j3], op5 = (double)o5[j5];
        const double op15 = (double)c15.p[(int64_t)s * c15.M + j15];
        r.price_change_1m = mul(dvd(sub(close, op1), op1), 100.0);
        r.price_change_3m = mul(dvd(sub(close, op3), op3), 100.0);
        r.price_change_5m = mul(dvd(sub(close, op5), op5), 100.0);
        r.price_change_15m = mul(dvd(sub(close, op15), op15), 100.0);
        // trend (:262-280)
        const double s1 = mul(dvd(sub(close, sma20), sma20), 100.0);
        const double s5 = mul(dvd(sub(close, sma20_5), sma20_5), 100.0);
        r.trend_strength = fabs(add(mul(s1, 0.6), mul(s5, 0.4)));
        if (close > sma20 && sma20 > sma50) r.trend = MM_UP;
        else if (close < sma20 && sma20 < sma50) r.trend = MM_DOWN;
        else r.trend = MM_SIDEWAYS;
        r.opportunity = fabs(r.price_change_1m) >= prm.min_price_change_pct && r.avg_volume >= prm.min_volume_usdc;
        combine(r);
    }
    const int64_t i = (int64_t)s * N + t;
    if (rows) rows[i] = r;
    if (labels) labels[i] = label_of(r, prm.label_field);
}

__global__ void __launch_bounds__(MM_THREADS)
combinations_kernel(b200bt_monitor_row* __restrict__ rows, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    b200bt_monitor_row r = rows[i];
    if (!r.valid) return;
    combine(r);
    rows[i] = r;
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_market_monitor(const float* ohlcv, int S, int64_t N, int64_t minute0, int bar_minutes,
                                     const float* ohlcv_3m, int64_t M3, const float* ohlcv_5m, int64_t M5,
                                     const float* ohlcv_15m, int64_t M15, const b200bt_monitor_params* params,
                                     b200bt_monitor_row* rows_or_null, uint8_t* labels_or_null, b200bt_stream_t stream) {
    B200BT_REQUIRE(ohlcv && ohlcv_3m && ohlcv_5m && ohlcv_15m && params, B200BT_EINVAL, "market_monitor: null pointer");
    B200BT_REQUIRE(rows_or_null || labels_or_null, B200BT_EINVAL, "market_monitor: no output (rows and labels both null)");
    B200BT_REQUIRE(S >= 1 && N >= 1, B200BT_EINVAL, "market_monitor: S and N must be >= 1");
    B200BT_REQUIRE(bar_minutes == 1, B200BT_EINVAL, "market_monitor: the market clock must be 1 minute (bar_minutes = %d)",
                   bar_minutes);
    B200BT_REQUIRE(minute0 >= 0, B200BT_EINVAL, "market_monitor: minute0 must be >= 0");
    B200BT_REQUIRE(params->frame_bars >= 1, B200BT_EINVAL, "market_monitor: frame_bars must be >= 1");
    B200BT_REQUIRE(params->label_field >= 0 && params->label_field < B200BT_MM_LABEL_FIELDS, B200BT_EINVAL,
                   "market_monitor: label_field must be 0 .. %d", B200BT_MM_LABEL_FIELDS - 1);
    B200BT_REQUIRE(N < ((int64_t)1 << 30), B200BT_ELIMIT, "market_monitor: N must be < 2^30");
    B200BT_REQUIRE(S <= 65535, B200BT_ELIMIT, "market_monitor: S must be <= 65535");
    B200BT_REQUIRE(M3 == b200bt_resample_bars(N, minute0, 1, 3) && M5 == b200bt_resample_bars(N, minute0, 1, 5) &&
                   M15 == b200bt_resample_bars(N, minute0, 1, 15), B200BT_EINVAL,
                   "market_monitor: kline counts must be b200bt_resample_bars(N, minute0, 1, k)");
    int rc = check_device();
    if (rc) return rc;
    const dim3 grid((unsigned)((N + MM_THREADS - 1) / MM_THREADS), (unsigned)S);
    monitor_kernel<<<grid, MM_THREADS, 0, (cudaStream_t)stream>>>(ohlcv, S, N, minute0, Clock{ohlcv_3m, M3, 3},
                                                                   Clock{ohlcv_5m, M5, 5}, Clock{ohlcv_15m, M15, 15},
                                                                   *params, rows_or_null, labels_or_null);
    B200BT_LAUNCH_CHECK("market_monitor launch");
    return B200BT_OK;
}

extern "C" int b200bt_indicator_combinations(b200bt_monitor_row* rows, int64_t n, b200bt_stream_t stream) {
    B200BT_REQUIRE(rows && n >= 1, B200BT_EINVAL, "indicator_combinations: rows must be non-null and n >= 1");
    B200BT_REQUIRE(n < ((int64_t)1 << 31), B200BT_ELIMIT, "indicator_combinations: n must be < 2^31");
    int rc = check_device();
    if (rc) return rc;
    combinations_kernel<<<(unsigned)((n + MM_THREADS - 1) / MM_THREADS), MM_THREADS, 0, (cudaStream_t)stream>>>(rows, n);
    B200BT_LAUNCH_CHECK("indicator_combinations launch");
    return B200BT_OK;
}
