// Volume profile (sm_90a): the reference's VolumeProfileAnalyzer (services/utils/volume_profile_analyzer.py) on every
// frame of W consecutive bars: profile, value area and signals (analyze_volume_profile :43-394), volume delta
// (analyze_volume_delta :564-684) and volume anomalies (detect_volume_anomalies :487-562).
//
// vp_frame_kernel  one warp per (frame end t, symbol); lane j owns bins j and j + 32.  Candles are read from global memory
//                  (neighbouring warps of a CTA share most of their bars, so the reads hit L1).
//                  1. min / max of the frame's lows / highs (warp reduction; exact in any order).
//                  2. each lane turns one candle of a 32-candle chunk into (low_bin, high_bin, volume per bin); the warp
//                     then walks the chunk in bar order, broadcasting one candle per step, and every lane adds to the bins
//                     it owns, so each bin is summed in bar order as the reference's volumes[lo:hi + 1] += vpb.
//                  3. rank of every bin by counting (descending volume, equal volumes in descending index); lane 0 walks
//                     the ranks for the value area and takes numpy's pairwise sum of the bins.
//                  4. lane 0 sums the deltas: the sequential cumsum and numpy's pairwise sums (np_pairwise_sum) of the whole
//                     frame, its positive and negative subsets and its last 20 / 40..20 bars.
//                  5. the anomaly pass: every lane recomputes the rolling mean / std of its bars (w reads each); counts by
//                     ballot, the strongest by a warp arg-max, the last five in a ring held by lanes 0..4.
#include <math.h>
#include "common.cuh"

namespace b200bt {

constexpr int VP_WARPS = 8;                  // frames per CTA
constexpr int VP_LEAF = 128;                 // numpy's PW_BLOCKSIZE
constexpr int VP_RECENT_BARS = 20;           // recent_delta, recent_anomaly_percentage: the last min(20, W) bars

// numpy's pairwise summation (np.add.reduce of float64, and so np.sum and pandas' Series.sum) of the n values `next()`
// yields in order: below 8 values a sequential sum from 0.0; up to 128 eight interleaved accumulators, combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the rest in order; above 128 the halves split at a multiple of 8
// are summed so and added.  The split tree is walked in post order with an explicit stack, so the leaves read the values
// in order and `next` can be a forward cursor over a subset.
template <class Next>
__device__ double np_pairwise_leaf(Next& next, int64_t n) {
    if (n < 8) {
        double r = 0.0;
        for (int64_t i = 0; i < n; ++i) r = __dadd_rn(r, next());
        return r;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = next();
    int64_t i = 8;
    for (; i < n - n % 8; i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], next());
    }
    double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) s = __dadd_rn(s, next());
    return s;
}

template <class Next>
__device__ double np_pairwise_sum(Next& next, int64_t n) {
    if (n <= VP_LEAF) return np_pairwise_leaf(next, n);
    int64_t len[40];        // pending ranges; n < 2^31 splits at most 24 times
    int stage[40];
    double part[40];
    int sp = 1, rp = 0;
    len[0] = n;
    stage[0] = 0;
    while (sp) {
        const int64_t m = len[sp - 1];
        if (m <= VP_LEAF) {
            part[rp++] = np_pairwise_leaf(next, m);
            --sp;
            continue;
        }
        const int64_t m2 = m / 2 - (m / 2) % 8;
        if (stage[sp - 1] == 0) {
            stage[sp - 1] = 1;
            len[sp] = m2;
            stage[sp++] = 0;
        } else if (stage[sp - 1] == 1) {
            stage[sp - 1] = 2;
            len[sp] = m - m2;
            stage[sp++] = 0;
        } else {
            --rp;
            part[rp - 1] = __dadd_rn(part[rp - 1], part[rp]);
            --sp;
        }
    }
    return part[0];
}

// The deltas of bars [i, end) in order; which: 0 every delta, 1 the positive ones, 2 the negative ones.
struct DeltaCursor {
    const float *open, *close, *vol;
    int64_t i;
    int which;
    __device__ double operator()() {
        for (;;) {
            const double v = (double)vol[i];
            const double d = close[i] >= open[i] ? v : -v;
            ++i;
            if (which == 0 || (which == 1 && d > 0.0) || (which == 2 && d < 0.0)) return d;
        }
    }
};

struct SmemCursor {
    const double* v;
    int i;
    __device__ double operator()() { return v[i++]; }
};

struct VpWarp {
    double vol[B200BT_VP_MAX_BINS];
    int order[B200BT_VP_MAX_BINS];
};

struct VpArgs {
    const float *open, *high, *low, *close, *vol;     // field rows of symbol 0; symbol s at + s * ld
    int64_t ld, N, ld_rows;
    b200bt_vp_params p;
    b200bt_vp_row* rows;
    double* bins;
    uint8_t* labels;
};

// Rolling mean and std (ddof 1) of the w volumes ending at bar g, in a fixed order: the sequential sum / w, then the
// sequential sum of the squared deviations / (w - 1).
__device__ __forceinline__ void rolling_stats(const float* vol, int64_t g, int w, double& ma, double& sd) {
    double s = 0.0;
    for (int j = w - 1; j >= 0; --j) s = __dadd_rn(s, (double)vol[g - j]);
    ma = __ddiv_rn(s, (double)w);
    double ss = 0.0;
    for (int j = w - 1; j >= 0; --j) {
        const double d = __dsub_rn((double)vol[g - j], ma);
        ss = __dadd_rn(ss, __dmul_rn(d, d));
    }
    sd = __dsqrt_rn(__ddiv_rn(ss, (double)(w - 1)));
}

// |a - c| / c * 100 (the reference's distance in percent)
__device__ __forceinline__ double dist_pct(double a, double c) {
    return __dmul_rn(__ddiv_rn(fabs(__dsub_rn(c, a)), c), 100.0);
}

__global__ void __launch_bounds__(VP_WARPS * 32)
vp_frame_kernel(const VpArgs a) {
    __shared__ VpWarp shared[VP_WARPS];
    const int s = blockIdx.y, lane = threadIdx.x & 31;
    const int64_t t = (int64_t)blockIdx.x * VP_WARPS + (threadIdx.x >> 5);
    if (t >= a.N) return;
    VpWarp& sw = shared[threadIdx.x >> 5];
    const int B = a.p.num_bins, W = a.p.frame_bars, w = a.p.anomaly_window;
    const int64_t so = (int64_t)s * a.ld;
    const float *op = a.open + so, *hi = a.high + so, *lo = a.low + so, *cl = a.close + so, *vo = a.vol + so;
    const int64_t r = (int64_t)s * a.ld_rows + t;
    b200bt_vp_row* row = a.rows ? a.rows + r : nullptr;
    double* bins = a.bins ? a.bins + r * B : nullptr;
    const bool frame = t >= W - 1;
    const int64_t t0 = t - W + 1;

    // ---- 1. price range
    double pmin = INFINITY, pmax = -INFINITY;
    if (frame)
        for (int64_t i = t0 + lane; i <= t; i += 32) {
            pmin = fmin(pmin, (double)lo[i]);
            pmax = fmax(pmax, (double)hi[i]);
        }
    pmin = warp_min_d(pmin);
    pmax = warp_max_d(pmax);
    const bool valid = frame && pmax > pmin;
    const double c = frame ? (double)cl[t] : NAN;

    // ---- 2. bins, in bar order
    double v0 = 0.0, v1 = 0.0;                       // bins lane and lane + 32
    const double bin_size = __ddiv_rn(__dsub_rn(pmax, pmin), (double)B);
    if (valid) {
        for (int64_t base = t0; base <= t; base += 32) {
            const int64_t i = base + lane;
            int lb = 0, hb = -1;
            double vpb = 0.0;
            if (i <= t) {
                lb = max(0, (int)__ddiv_rn(__dsub_rn((double)lo[i], pmin), bin_size));
                hb = min(B - 1, (int)__ddiv_rn(__dsub_rn((double)hi[i], pmin), bin_size));
                if (hb >= lb) vpb = __ddiv_rn((double)vo[i], (double)(hb - lb + 1));
            }
            const int n = (int)min((int64_t)32, t - base + 1);
            for (int k = 0; k < n; ++k) {
                const int kl = __shfl_sync(FULL, lb, k), kh = __shfl_sync(FULL, hb, k);
                const double kv = shfl_d(vpb, k);
                if (lane >= kl && lane <= kh) v0 = __dadd_rn(v0, kv);
                if (lane + 32 >= kl && lane + 32 <= kh) v1 = __dadd_rn(v1, kv);
            }
        }
    }
    if (bins)
        for (int i = lane; i < B; i += 32) bins[i] = i < 32 ? v0 : v1;

    // ---- 3. profile and signals
    int label = B200BT_VP_NO_LABEL;
    if (valid) {
        const bool own1 = lane + 32 < B;
        if (lane < B) sw.vol[lane] = v0;
        if (own1) sw.vol[lane + 32] = v1;
        __syncwarp();
        // rank: larger volumes first, equal volumes in descending index
        for (int q = 0; q < 2; ++q) {
            const int i = lane + 32 * q;
            if (i >= B) break;
            const double vi = sw.vol[i];
            int rank = 0;
            for (int j = 0; j < B; ++j) {
                const double vj = sw.vol[j];
                rank += vj > vi || (vj == vi && j > i);
            }
            sw.order[rank] = i;
        }
        // the largest bin (the first on ties)
        double mv = lane < B ? v0 : -INFINITY;
        int mi = lane;
        if (own1 && v1 > mv) {
            mv = v1;
            mi = lane + 32;
        }
        for (int m = 16; m > 0; m >>= 1) {
            const double ov = shfl_xor_d(mv, m);
            const int oi = __shfl_xor_sync(FULL, mi, m);
            if (ov > mv || (ov == mv && oi < mi)) {
                mv = ov;
                mi = oi;
            }
        }
        const double max_volume = mv > 0.0 ? mv : 1.0;
        // price levels: np.linspace edges i * step + min (the last one max), midpoints (e_i + e_i+1) / 2
        auto edge = [&](int i) { return i == B ? pmax : __dadd_rn(__dmul_rn((double)i, bin_size), pmin); };
        auto level = [&](int i) { return __ddiv_rn(__dadd_rn(edge(i), edge(i + 1)), 2.0); };
        // high / low volume nodes, the closest low-volume node, the node flags
        const double hvn_thr = __dmul_rn(0.7, max_volume), lvn_thr = __dmul_rn(0.3, max_volume);
        bool hvn0 = false, hvn1 = false, lvn0 = false, lvn1 = false, at_l = false, at_h = false;
        double cd = INFINITY;
        int ci = -1;
        for (int q = 0; q < 2; ++q) {
            const int i = lane + 32 * q;
            if (i >= B) break;
            const double vi = q ? v1 : v0, li = level(i);
            const bool h = vi >= hvn_thr, l = vi <= lvn_thr;
            (q ? hvn1 : hvn0) = h;
            (q ? lvn1 : lvn0) = l;
            const double dp = dist_pct(li, c);
            at_h |= h && dp < 0.3;
            at_l |= l && dp < 0.3;
            if (l) {
                const double d = fabs(__dsub_rn(li, c));
                if (d < cd) {
                    cd = d;
                    ci = i;
                }
            }
        }
        for (int m = 16; m > 0; m >>= 1) {
            const double od = shfl_xor_d(cd, m);
            const int oi = __shfl_xor_sync(FULL, ci, m);
            if (oi >= 0 && (ci < 0 || od < cd || (od == cd && oi < ci))) {
                cd = od;
                ci = oi;
            }
        }
        const unsigned h0 = __ballot_sync(FULL, hvn0), h1 = __ballot_sync(FULL, hvn1);
        const unsigned l0 = __ballot_sync(FULL, lvn0), l1 = __ballot_sync(FULL, lvn1);
        const bool any_at_l = __any_sync(FULL, at_l), any_at_h = __any_sync(FULL, at_h);
        __syncwarp();
        if (lane == 0) {
            // value area: the ranked bins until their cumulative volume reaches total * pct
            SmemCursor cur{sw.vol, 0};
            const double total = np_pairwise_sum(cur, B);
            const double thr = __dmul_rn(total, a.p.value_area_pct);
            double cum = 0.0;
            int va_lo = B, va_hi = -1;
            for (int k = 0; k < B; ++k) {
                const int i = sw.order[k];
                cum = __dadd_rn(cum, sw.vol[i]);
                va_lo = min(va_lo, i);
                va_hi = max(va_hi, i);
                if (cum >= thr) break;
            }
            const double poc = level(mi), val = level(va_lo), vah = level(va_hi);
            // _generate_signals :248-314
            int poc_code, va_code;
            if (dist_pct(poc, c) < 0.5) poc_code = c < poc ? 0 : 1;
            else poc_code = c < poc ? 2 : 3;
            if (c > vah) va_code = __dmul_rn(__ddiv_rn(__dsub_rn(c, vah), c), 100.0) < 0.3 ? 0 : 1;
            else if (c < val) va_code = __dmul_rn(__ddiv_rn(__dsub_rn(val, c), c), 100.0) < 0.3 ? 2 : 3;
            else {
                const double rel = __ddiv_rn(__dsub_rn(c, val), __dsub_rn(vah, val));   // NaN (0 / 0): middle
                va_code = rel < 0.3 ? 4 : rel > 0.7 ? 5 : 6;
            }
            if (va_code == 0 || poc_code == 1) label = 0;            // potential_resistance
            else if (va_code == 2 || poc_code == 0) label = 1;       // potential_support
            else if (any_at_l) label = 2;                            // potential_breakout_zone
            else if (va_code == 1) label = 3;                        // overbought
            else if (va_code == 3) label = 4;                        // oversold
            else label = 5;                                          // neutral
            if (row) {
                row->poc_code = poc_code;
                row->value_area_code = va_code;
                row->at_low_volume_node = any_at_l;
                row->at_high_volume_node = any_at_h;
                row->poc_bin = mi;
                row->value_area_low_bin = va_lo;
                row->value_area_high_bin = va_hi;
                row->hvn_count = __popc(h0) + __popc(h1);
                row->lvn_count = __popc(l0) + __popc(l1);
                row->closest_lvn_bin = ci;
                row->poc = poc;
                row->value_area_low = val;
                row->value_area_high = vah;
                row->total_volume = total;
                row->max_volume = mv;
                unsigned m0 = h0, m1 = h1;
                for (int k = 0; k < 3; ++k) {
                    int i = -1;
                    if (m0) {
                        i = __ffs(m0) - 1;
                        m0 &= m0 - 1;
                    } else if (m1) {
                        i = 32 + __ffs(m1) - 1;
                        m1 &= m1 - 1;
                    }
                    row->hvn_price[k] = i >= 0 ? level(i) : NAN;
                }
                row->closest_lvn = ci >= 0 ? level(ci) : NAN;
            }
        }
    } else if (row && lane == 0) {
        row->poc_code = row->value_area_code = -1;
        row->at_low_volume_node = row->at_high_volume_node = 0;
        row->poc_bin = row->value_area_low_bin = row->value_area_high_bin = row->closest_lvn_bin = -1;
        row->hvn_count = row->lvn_count = 0;
        row->poc = row->value_area_low = row->value_area_high = row->total_volume = row->max_volume = NAN;
        row->hvn_price[0] = row->hvn_price[1] = row->hvn_price[2] = row->closest_lvn = NAN;
    }
    if (a.labels && lane == 0) a.labels[r] = (uint8_t)label;
    if (!row) return;
    if (lane == 0) {
        row->n_bars = frame ? W : 0;
        row->valid = valid;
        row->signal = label;
        row->price_min = frame ? pmin : NAN;
        row->price_max = frame ? pmax : NAN;
        row->close = c;
        row->reserved[0] = row->reserved[1] = row->reserved[2] = row->reserved[3] = 0;
    }

    // ---- 4. volume delta (analyze_volume_delta :581-654)
    const int periods = min(VP_RECENT_BARS, W);
    if (lane == 0) {
        if (frame) {
            double cum = 0.0;
            for (int64_t i = t0; i <= t; ++i) {
                const double v = (double)vo[i], d = cl[i] >= op[i] ? v : -v;
                cum = i == t0 ? d : __dadd_rn(cum, d);
            }
            int64_t n_pos = 0, n_neg = 0;
            for (int64_t i = t0; i <= t; ++i) {
                const double v = (double)vo[i], d = cl[i] >= op[i] ? v : -v;
                n_pos += d > 0.0;
                n_neg += d < 0.0;
            }
            DeltaCursor all{op, cl, vo, t0, 0}, pos{op, cl, vo, t0, 1}, neg{op, cl, vo, t0, 2};
            DeltaCursor rec{op, cl, vo, t - periods + 1, 0}, prev{op, cl, vo, t - 39, 0};
            const double net = np_pairwise_sum(all, W);
            const double buy = np_pairwise_sum(pos, n_pos), sell = fabs(np_pairwise_sum(neg, n_neg));
            const double ratio = sell > 0.0 ? __ddiv_rn(buy, sell) : INFINITY;
            const double recent = np_pairwise_sum(rec, periods);
            const bool mom = W >= 40;
            const double momentum = mom ? __dsub_rn(recent, np_pairwise_sum(prev, 20)) : NAN;
            row->cumulative_delta = cum;
            row->net_period_delta = net;
            row->buying_volume = buy;
            row->selling_volume = sell;
            row->buy_sell_ratio = ratio;
            row->recent_delta = recent;
            row->delta_momentum = momentum;
            row->has_momentum = mom;
            row->pressure = ratio > 1.5 ? 0 : ratio > 1.1 ? 1 : ratio < 0.67 ? 2 : ratio < 0.9 ? 3 : 4;
            row->recent_pressure = recent > 0.0 ? 0 : 1;
            const bool price_up = __dsub_rn((double)cl[t], (double)cl[t - periods + 1]) > 0.0, delta_up = recent > 0.0;
            row->divergence = price_up && !delta_up ? 0 : !price_up && delta_up ? 1 : 2;
        } else {
            row->cumulative_delta = row->net_period_delta = row->buying_volume = row->selling_volume = NAN;
            row->buy_sell_ratio = row->recent_delta = row->delta_momentum = NAN;
            row->has_momentum = 0;
            row->pressure = row->recent_pressure = row->divergence = -1;
        }
    }

    // ---- 5. volume anomalies (detect_volume_anomalies :504-556)
    const bool anomalies = frame && W >= w;
    int total = 0, recent = 0, best_off = -1;
    double best_sig = -INFINITY, best_vol = NAN, best_ma = NAN;
    double ring_ma = NAN, ring_sig = NAN;                 // lanes 0..4: ring slot `lane` of the last five anomalies
    int ring_off = -1;
    if (anomalies) {
        const double k = a.p.std_threshold;
        const int64_t first = t0 + w - 1, recent_lo = t - periods + 1;
        for (int64_t base = first; base <= t; base += 32) {
            const int64_t g = base + lane;
            double ma = NAN, sd = NAN, sig = NAN, v = NAN;
            bool flag = false;
            if (g <= t) {
                rolling_stats(vo, g, w, ma, sd);
                v = (double)vo[g];
                flag = v > __dadd_rn(ma, __dmul_rn(k, sd));
                sig = __ddiv_rn(__dsub_rn(v, ma), sd);
            }
            unsigned m = __ballot_sync(FULL, flag);
            total += __popc(m);
            recent += __popc(__ballot_sync(FULL, flag && g >= recent_lo));
            if (flag && sig > best_sig) {                  // each lane's bars ascend: strict > keeps the first
                best_sig = sig;
                best_vol = v;
                best_ma = ma;
                best_off = (int)(g - t0);
            }
            while (m) {                                    // the ring of the last five, in bar order
                const int src = __ffs(m) - 1;
                m &= m - 1;
                const double rm = shfl_d(ma, src), rs = shfl_d(sig, src);
                const int slot = (total - __popc(m) - 1) % B200BT_VP_RECENT;
                if (lane == slot) {
                    ring_ma = rm;
                    ring_sig = rs;
                    ring_off = (int)(base + src - t0);
                }
            }
        }
        for (int m = 16; m > 0; m >>= 1) {
            const double os = shfl_xor_d(best_sig, m), ov = shfl_xor_d(best_vol, m), oa = shfl_xor_d(best_ma, m);
            const int oo = __shfl_xor_sync(FULL, best_off, m);
            if (oo >= 0 && (best_off < 0 || os > best_sig || (os == best_sig && oo < best_off))) {
                best_sig = os;
                best_vol = ov;
                best_ma = oa;
                best_off = oo;
            }
        }
    }
    const int n_recent = min(total, B200BT_VP_RECENT);
    if (lane < B200BT_VP_RECENT) {
        int i = -1;
        if (total > 0) {                                   // ring slot `lane` holds anomaly e; its place among the last n
            const int e = total - 1 - ((total - 1 - lane) % B200BT_VP_RECENT);
            if (e >= total - n_recent) i = e - (total - n_recent);
        }
        // rows of the last five are written by the lane that holds them; the unused places by lane i = place
        if (i >= 0) {
            row->recent_offset[i] = ring_off;
            row->recent_ma[i] = ring_ma;
            row->recent_significance[i] = ring_sig;
        }
        if (lane >= n_recent) {
            row->recent_offset[lane] = -1;
            row->recent_ma[lane] = row->recent_significance[lane] = NAN;
        }
    }
    if (lane == 0) {
        row->anomaly_status = anomalies;
        row->total_anomalies = total;
        row->n_recent = n_recent;
        row->recent_anomaly_pct = anomalies ? __dmul_rn(__ddiv_rn((double)recent, (double)periods), 100.0) : NAN;
        row->strongest_offset = total ? best_off : -1;
        row->strongest_significance = total ? best_sig : NAN;
        row->strongest_volume = total ? best_vol : NAN;
        row->strongest_ma = total ? best_ma : NAN;
    }
}

}  // namespace b200bt

using namespace b200bt;

// services/utils/volume_profile_analyzer.py :43-394, :487-562, :564-684 (see b200bt.h)
extern "C" int b200bt_volume_profile(const float* ohlcv, int64_t ld, int S, int64_t N, const b200bt_vp_params* params,
                                     b200bt_vp_row* rows_or_null, double* bins_or_null, uint8_t* labels_or_null,
                                     int64_t ld_rows, b200bt_stream_t stream) {
    B200BT_REQUIRE(ohlcv && params, B200BT_EINVAL, "volume_profile: null pointer");
    B200BT_REQUIRE(rows_or_null || bins_or_null || labels_or_null, B200BT_EINVAL, "volume_profile: no output");
    B200BT_REQUIRE(S >= 1 && N >= 1 && ld >= N && ld_rows >= N, B200BT_EINVAL, "volume_profile: bad sizes");
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "volume_profile: N must be < 2^30 bars");
    B200BT_REQUIRE(S <= 65535, B200BT_ELIMIT, "volume_profile: at most 65535 symbols");
    const b200bt_vp_params p = *params;
    B200BT_REQUIRE(p.frame_bars >= 1, B200BT_EINVAL, "volume_profile: frame_bars = %d, need >= 1", p.frame_bars);
    B200BT_REQUIRE(p.num_bins >= 1, B200BT_EINVAL, "volume_profile: num_bins = %d, need >= 1", p.num_bins);
    B200BT_REQUIRE(p.num_bins <= B200BT_VP_MAX_BINS, B200BT_ELIMIT, "volume_profile: num_bins = %d above %d", p.num_bins,
                   B200BT_VP_MAX_BINS);
    B200BT_REQUIRE(p.anomaly_window >= 2, B200BT_EINVAL, "volume_profile: anomaly_window = %d, need >= 2",
                   p.anomaly_window);
    B200BT_REQUIRE(isfinite(p.value_area_pct) && isfinite(p.std_threshold), B200BT_EINVAL,
                   "volume_profile: value_area_pct and std_threshold must be finite");
    int rc = check_device();
    if (rc) return rc;
    VpArgs a;
    a.open = ohlcv;
    a.high = ohlcv + (int64_t)S * ld;
    a.low = ohlcv + 2 * (int64_t)S * ld;
    a.close = ohlcv + 3 * (int64_t)S * ld;
    a.vol = ohlcv + 4 * (int64_t)S * ld;
    a.ld = ld;
    a.N = N;
    a.ld_rows = ld_rows;
    a.p = p;
    a.rows = rows_or_null;
    a.bins = bins_or_null;
    a.labels = labels_or_null;
    const dim3 grid((unsigned)((N + VP_WARPS - 1) / VP_WARPS), (unsigned)S);
    vp_frame_kernel<<<grid, VP_WARPS * 32, 0, (cudaStream_t)stream>>>(a);
    B200BT_LAUNCH_CHECK("volume_profile");
    return B200BT_OK;
}
