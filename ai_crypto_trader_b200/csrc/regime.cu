// Market regimes (sm_90a): regime windows and per-bar labels of a market, and the trade metrics of a sweep's records split
// by the label of their bar.
//
// The reference labels the market bull / bear / ranging / volatile from monitor snapshots (services/market_regime_service.py
// detect_regime_from_data :503-603) and segments its history into 24-hour windows (update_strategy_performance_by_regime
// :844-889).  Its per-regime backtest stops at a TODO (:909-911); the class pass below is that backtest.
//
// regime_window_kernel  one warp per (window, symbol).  Every CTA first finds its symbol's first point (a sample bucket's
//                       last bar where SMA20, SMA50 and the aligned 5-minute SMA20 are all defined) with a block-wide
//                       search of the head; lane 0 then walks the window's points twice (sums, then the squared
//                       deviations of the returns) and the warp writes the window's label on the window's bars.  The
//                       work is O(points) per symbol: a few points per window, one window per 1440 minutes.
// class_stats_kernel    one warp per (individual, symbol) lane walks the lane's records once, 32 at a time, as
//                       daily_pnl_kernel does (record_batch: a coalesced word load, record_pnl with the entry by shuffle),
//                       one label byte per record.  For each class present in the batch (ballot) its records are compacted into that
//                       class's shared-memory staging (<= 63 entries); each full 32 goes through batch_records with the
//                       class's own WarpAcc, the rest is flushed at the end, and finalize_lane gives every class's stats.
#include <math.h>
#include "sweep_dev.cuh"

namespace b200bt {

constexpr int RG_WARPS = 8;                  // windows per CTA of the labelling pass
constexpr int CL_WARPS = 4;                  // lanes per CTA of the class pass
constexpr int CL_MAX = 8;                    // classes per call
constexpr int CL_STAGE = 64;                 // staged records per class: < 32 left over + 32 new

// ---- regime windows and bar labels ---------------------------------------------------------------------------------
struct RegimeClock {
    int64_t N, ld, ld_labels, minute0, n_windows_max;
    int bar_minutes, sample_minutes;
};

__device__ __forceinline__ int64_t bar_minute(const RegimeClock& c, int64_t t) { return c.minute0 + t * c.bar_minutes; }

// bar t is the last bar of its sample bucket: the next bar starts in a later bucket (align_kernel's "completes" rule)
__device__ __forceinline__ bool is_point(const RegimeClock& c, int64_t t) {
    const int64_t m = bar_minute(c, t);
    return (m + c.bar_minutes) / c.sample_minutes != m / c.sample_minutes;
}

// first bar at or after minute m (may be N or beyond)
__device__ __forceinline__ int64_t first_bar_from(const RegimeClock& c, int64_t m) {
    const int64_t d = m - c.minute0;
    return d <= 0 ? 0 : (d + c.bar_minutes - 1) / c.bar_minutes;
}

__global__ void __launch_bounds__(RG_WARPS * 32)
regime_window_kernel(const float* __restrict__ close, const float* __restrict__ sma20, const float* __restrict__ sma50,
                     const float* __restrict__ sma5, const RegimeClock c, const b200bt_regime_params p,
                     uint8_t* __restrict__ labels, b200bt_regime_window* __restrict__ rows) {
    __shared__ long long first_pt;
    const int s = blockIdx.y, lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * RG_WARPS + (threadIdx.x >> 5);
    const float* cr = close + (int64_t)s * c.ld;
    const float* a20 = sma20 + (int64_t)s * c.ld;
    const float* a50 = sma50 + (int64_t)s * c.ld;
    const float* a5 = sma5 + (int64_t)s * c.ld;
    // the symbol's first point: the head is short (SMA50 / the 5-minute SMA20), so a block-wide search from bar 0
    if (threadIdx.x == 0) first_pt = c.N;
    __syncthreads();
    for (int64_t t0 = 0; t0 < c.N; t0 += blockDim.x) {
        const int64_t t = t0 + threadIdx.x;
        const bool ok = t < c.N && is_point(c, t) && !isnan(a20[t]) && !isnan(a50[t]) && !isnan(a5[t]);
        if (ok) atomicMin(&first_pt, (long long)t);
        if (__syncthreads_or(ok)) break;
    }
    const int64_t t_first = first_pt;
    // the last point: the last bar of the last bucket that a later bar would leave (a bucket cut by the series end is not one)
    const int64_t m_end = bar_minute(c, c.N);                       // start of the bar after the series
    const int64_t t_last = first_bar_from(c, (m_end / c.sample_minutes) * c.sample_minutes) - 1;
    const bool any = t_first < c.N && t_last >= t_first;
    const int64_t m0 = any ? bar_minute(c, t_first) : 0, m_last = any ? bar_minute(c, t_last) : 0;
    const int64_t K = any ? (m_last - m0 + 1439) / 1440 : 0;       // windows start while their start < the last point
    if (k >= c.n_windows_max) return;
    b200bt_regime_window* row = rows ? rows + (int64_t)s * c.n_windows_max + k : nullptr;
    if (k >= K) {
        if (row && lane == 0) {
            row->start_minute = -1;
            row->n_points = 0;
            row->label = B200BT_REGIME_UNKNOWN;
            row->volatility = row->change_pct = row->mean_strength = NAN;
            row->up_frac = row->down_frac = row->sideways_frac = NAN;
        }
        return;
    }
    const int64_t w0 = m0 + 1440 * k, w1 = w0 + 1440;
    int label = B200BT_REGIME_UNKNOWN;
    if (lane == 0) {
        // the window's points: t in [t_first, t_last] that are points and start in [w0, w1)
        const int64_t lo = max(first_bar_from(c, w0), t_first), hi = min(first_bar_from(c, w1) - 1, t_last);
        int n = 0, n_up = 0, n_down = 0, n_side = 0;
        double first = 0.0, last = 0.0, prev = 0.0, sum_r = 0.0, sum_ts = 0.0;
        for (int64_t t = lo; t <= hi; ++t) {
            if (!is_point(c, t)) continue;
            const double px = (double)cr[t], s20 = (double)a20[t], s50 = (double)a50[t], s5 = (double)a5[t];
            // market_monitor_service.py:263-280 (indicators.multi_timeframe_indicators at bar t)
            const double st1 = __dmul_rn(__ddiv_rn(__dsub_rn(px, s20), s20), 100.0);
            const double st5 = __dmul_rn(__ddiv_rn(__dsub_rn(px, s5), s5), 100.0);
            sum_ts = __dadd_rn(sum_ts, fabs(__dadd_rn(__dmul_rn(st1, 0.6), __dmul_rn(st5, 0.4))));
            if (px > s20 && s20 > s50) ++n_up;
            else if (px < s20 && s20 < s50) ++n_down;
            else ++n_side;
            if (n == 0) first = px;
            else sum_r = __dadd_rn(sum_r, __dsub_rn(__ddiv_rn(px, prev), 1.0));
            prev = last = px;
            ++n;
        }
        double vol = NAN;
        if (n >= 3) {                               // pandas' std (ddof 1) of the n - 1 returns
            const double mean = __ddiv_rn(sum_r, (double)(n - 1));
            double ss = 0.0, pv = first;
            bool head = true;
            for (int64_t t = lo; t <= hi; ++t) {
                if (!is_point(c, t)) continue;
                const double px = (double)cr[t];
                if (!head) {
                    const double d = __dsub_rn(__dsub_rn(__ddiv_rn(px, pv), 1.0), mean);
                    ss = __dadd_rn(ss, __dmul_rn(d, d));
                }
                head = false;
                pv = px;
            }
            vol = __dmul_rn(sqrt(__ddiv_rn(ss, (double)(n - 2))), sqrt(24.0));
        }
        const double nn = (double)n;
        const double change = n ? __dmul_rn(__ddiv_rn(__dsub_rn(last, first), first), 100.0) : NAN;
        const double ts = n ? __ddiv_rn(sum_ts, nn) : NAN;
        const double up = n ? n_up / nn : NAN, down = n ? n_down / nn : NAN, side = n ? n_side / nn : NAN;
        if (n >= 2) {                               // detect_regime_from_data :571-597, in its order
            if (vol > p.volatile_volatility) label = B200BT_REGIME_VOLATILE;
            else if (change > p.bull_price_change && up > p.bull_trend_strength) label = B200BT_REGIME_BULL;
            else if (change < p.bear_price_change && down > p.bear_trend_strength) label = B200BT_REGIME_BEAR;
            else if (fabs(change) < p.ranging_price_range && ts < p.ranging_trend_strength) label = B200BT_REGIME_RANGING;
            else if (up > down && up > side) label = B200BT_REGIME_BULL;
            else if (down > up && down > side) label = B200BT_REGIME_BEAR;
            else label = B200BT_REGIME_RANGING;
        }
        if (row) {
            row->start_minute = w0;
            row->n_points = n;
            row->label = label;
            row->volatility = vol;
            row->change_pct = change;
            row->mean_strength = ts;
            row->up_frac = up;
            row->down_frac = down;
            row->sideways_frac = side;
        }
    }
    label = __shfl_sync(FULL, label, 0);
    if (label == B200BT_REGIME_UNKNOWN) return;     // the rows were set to UNKNOWN before this kernel
    uint8_t* lab = labels + (int64_t)s * c.ld_labels;
    const int64_t b_lo = first_bar_from(c, w0), b_hi = min(first_bar_from(c, w1), c.N);
    for (int64_t t = b_lo + lane; t < b_hi; t += 32) lab[t] = (uint8_t)label;
}

// ---- trade metrics per bar label -----------------------------------------------------------------------------------
struct ClassWarp {
    WarpAcc acc[CL_MAX];
    double pnl[CL_MAX][CL_STAGE];
    uint32_t word[CL_MAX][CL_STAGE];
    unsigned carry_bar[CL_MAX];      // bar of the class's previous record (duration pairs of the class list)
    int fill[CL_MAX];                // staged records of the class
};

// Run `n` (<= 32) staged records of class `cls` through the metrics step as one merged list, as book_kernel runs a book.
__device__ __forceinline__ void flush_class(ClassWarp& cw, int cls, int n, const b200bt_sweep_config& cfg) {
    const int lane = threadIdx.x & 31;
    const bool act = lane < n;
    const unsigned wd = act ? cw.word[cls][lane] : 0u;
    const double pnl = act ? cw.pnl[cls][lane] : 0.0;
    const unsigned carry = merged_records(&cw.acc[cls], n, act, wd, wd, pnl, cw.carry_bar[cls], cfg);
    if (lane == 0) cw.carry_bar[cls] = carry;
    __syncwarp();
}

__global__ void __launch_bounds__(CL_WARPS * 32)
class_stats_kernel(const float* __restrict__ price, int64_t ld_price, int S, const b200bt_individual* __restrict__ indiv,
                   const b200bt_sweep_config cfg, const b200bt_lane_stats* __restrict__ lane_stats,
                   const uint32_t* __restrict__ events, int64_t event_cap, const uint8_t* __restrict__ labels,
                   int64_t ld_labels, int R, b200bt_lane_stats* __restrict__ out, int64_t n_lanes) {
    __shared__ ClassWarp shared[CL_WARPS];
    const int lane = threadIdx.x & 31;
    const int64_t w = (int64_t)blockIdx.x * CL_WARPS + (threadIdx.x >> 5);
    if (w >= n_lanes) return;
    ClassWarp& cw = shared[threadIdx.x >> 5];
    LaneRecords r;
    if (!read_lane(r, w, S, price, ld_price, indiv, lane_stats, events, event_cap)) {   // lost records: no class stats
        if (lane < R) out[lane * n_lanes + w] = lost_lane_stats();
        return;
    }
    const int s = (int)(w % S);
    if (lane < R) {
        init_acc(cw.acc[lane], indiv[w / S], cfg, nullptr);
        cw.carry_bar[lane] = 0u;
        cw.fill[lane] = 0;
    }
    __syncwarp();
    const uint8_t* lab = labels + (int64_t)s * ld_labels;
    const unsigned below = (1u << lane) - 1u;
    for (int64_t base = 0; base < r.n; base += 32) {
        const RecordBatch b = record_batch(r, base);
        const int cls = b.active ? (int)__ldg(lab + b.bar) : 0xff;
        unsigned todo = __ballot_sync(FULL, cls < R);
        while (todo) {
            const int c = __shfl_sync(FULL, cls, __ffs(todo) - 1);
            const unsigned mask = __ballot_sync(FULL, cls == c);
            todo &= ~mask;
            int f = cw.fill[c];
            if (cls == c) {
                const int pos = f + __popc(mask & below);
                cw.word[c][pos] = b.w;
                cw.pnl[c][pos] = b.pnl;
            }
            f += __popc(mask);
            __syncwarp();
            if (f >= 32) {
                flush_class(cw, c, 32, cfg);
                f -= 32;
                const bool mv = lane < f;
                const unsigned mw = mv ? cw.word[c][32 + lane] : 0u;
                const double mp = mv ? cw.pnl[c][32 + lane] : 0.0;
                if (mv) {
                    cw.word[c][lane] = mw;
                    cw.pnl[c][lane] = mp;
                }
            }
            if (lane == 0) cw.fill[c] = f;
            __syncwarp();
        }
    }
    for (int c = 0; c < R; ++c) {
        const int f = cw.fill[c];
        if (f) flush_class(cw, c, f, cfg);
    }
    if (lane < R) {
        b200bt_lane_stats o;
        finalize_lane(cw.acc[lane], cfg, o);
        out[lane * n_lanes + w] = o;
    }
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_regime_labels(const float* close, const float* sma20, const float* sma50,
                                    const float* sma20_5m_aligned, int S, int64_t N, int64_t ld, int64_t minute0,
                                    int bar_minutes, const b200bt_regime_params* params, uint8_t* labels,
                                    int64_t ld_labels, b200bt_regime_window* window_stats_or_null, int64_t max_windows,
                                    b200bt_stream_t stream) {
    B200BT_REQUIRE(close && sma20 && sma50 && sma20_5m_aligned && params && labels, B200BT_EINVAL,
                   "regime_labels: null pointer");
    B200BT_REQUIRE(S >= 1 && N >= 1 && ld >= N && (S == 1 || ld_labels >= N), B200BT_EINVAL, "regime_labels: bad sizes");
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "regime_labels: N must be < 2^30 bars");
    B200BT_REQUIRE(minute0 >= 0, B200BT_EINVAL, "regime_labels: minute0 must be >= 0 (labels are made on the unbroken clock)");
    B200BT_REQUIRE(bar_minutes > 0 && minute0 + N * (int64_t)bar_minutes < (1ll << 62), B200BT_EINVAL,
                   "regime_labels: bad bar clock");
    const int sm = params->sample_minutes;
    B200BT_REQUIRE(sm > 0 && sm % 5 == 0 && sm % bar_minutes == 0, B200BT_EINVAL,
                   "regime_labels: sample_minutes = %d must be a positive multiple of 5 and of bar_minutes = %d", sm,
                   bar_minutes);
    const int64_t kmax = b200bt_regime_max_windows(N, bar_minutes);
    B200BT_REQUIRE(!window_stats_or_null || max_windows >= kmax, B200BT_EINVAL,
                   "regime_labels: max_windows = %lld below the %lld windows the series can hold", (long long)max_windows,
                   (long long)kmax);
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t ldl = S == 1 ? N : ld_labels;
    rc = cuda_status(cudaMemset2DAsync(labels, (size_t)ldl, B200BT_REGIME_UNKNOWN, (size_t)N, (size_t)S, st),
                     "regime_labels memset");
    if (rc) return rc;
    RegimeClock c;
    c.N = N;
    c.ld = ld;
    c.ld_labels = ldl;
    c.minute0 = minute0;
    c.bar_minutes = bar_minutes;
    c.sample_minutes = sm;
    c.n_windows_max = window_stats_or_null ? max_windows : kmax;
    const dim3 grid((unsigned)((c.n_windows_max + RG_WARPS - 1) / RG_WARPS), (unsigned)S);
    regime_window_kernel<<<grid, RG_WARPS * 32, 0, st>>>(close, sma20, sma50, sma20_5m_aligned, c, *params, labels,
                                                          window_stats_or_null);
    B200BT_LAUNCH_CHECK("regime_labels");
    return B200BT_OK;
}

extern "C" int64_t b200bt_regime_max_windows(int64_t N, int bar_minutes) {
    if (N < 1 || bar_minutes < 1) return 0;
    return ((N - 1) * (int64_t)bar_minutes + 1439) / 1440 + 1;
}

extern "C" int b200bt_class_stats(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv,
                                  int pop, const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats,
                                  const uint32_t* events, int64_t event_cap, const uint8_t* labels, int64_t ld_labels, int R,
                                  b200bt_lane_stats* class_stats, b200bt_stream_t stream) {
    B200BT_REQUIRE(cfg && labels && class_stats, B200BT_EINVAL, "class_stats: null pointer");
    int rc = check_record_args("class_stats", price, ld_price, S, N, indiv, pop, cfg, lane_stats, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE(ld_labels == 0 || ld_labels >= N, B200BT_EINVAL,
                   "class_stats: ld_labels must be 0 (one shared row) or >= N");
    B200BT_REQUIRE(R >= 1, B200BT_EINVAL, "class_stats: R = %d classes, need at least 1", R);
    B200BT_REQUIRE(R <= CL_MAX, B200BT_ELIMIT, "class_stats: at most %d classes (R = %d)", CL_MAX, R);
    rc = check_device();
    if (rc) return rc;
    const int64_t lanes = (int64_t)pop * S;
    class_stats_kernel<<<(unsigned)((lanes + CL_WARPS - 1) / CL_WARPS), CL_WARPS * 32, 0, (cudaStream_t)stream>>>(
        price, ld_price, S, indiv, *cfg, lane_stats, events, event_cap, labels, ld_labels, R, class_stats, lanes);
    B200BT_LAUNCH_CHECK("class_stats");
    return B200BT_OK;
}
