// Strategy selection replay (sm_90a): StrategySelectionService (services/strategy_selection_service.py) run over history.
// At every check every candidate is scored from its cached metrics snapshot, the best is reduced over candidates, and a
// single-warp pass applies the switch rule (:884-934) to the per-check rows.
//
// selection_kernel  one warp per candidate.  The warp merges the candidate's records on every symbol in book order (bar,
//                   symbol, record index) -- a warp-wide minimum over the symbols' next records, 16 staged words per symbol
//                   -- and walks them 32 at a time through the book's metrics step (merged_records) for the overall
//                   fields, through one more WarpAcc per scored regime for the records whose bar carries that regime
//                   (compacted by ballot), and into 24 hour counters.  A batch stops at the bar of the check being
//                   refreshed, so a snapshot is the state after exactly the records with bar <= t_c.  Lane j of a pass
//                   evaluates check c + j from the current snapshot; the first lane whose check refreshes the cache
//                   (ballot) ends the pass, the records up to that check are consumed and the snapshot retaken.
//                   Each lane merges its check's (score, candidate) into the row under a per-check lock; only a score
//                   strictly below the row's (which never decreases) is skipped without it, so every tie is decided
//                   under the lock.  The maximum over a total order (score desc, index asc) does not depend on the
//                   order of arrival, and no floating-point atomic is used.  The score
//                   expressions use explicitly rounded operations (no FMA contraction), in the reference's order.
// selection_init_kernel   the rows of a first batch: bar, regime label, no best yet; the check locks zeroed.
// selection_switch_kernel one warp scans the rows in order, 32 at a time: the first lane of a block whose row switches
//                   under the current (active, active score) is found by ballot, the state is updated, and the scan goes on
//                   from the next lane.
#include <math.h>
#include "sweep_dev.cuh"

namespace b200bt {

constexpr int SL_WARPS = 4;             // candidates per CTA
constexpr int SL_MIN_BLOCKS = 4;        // CTAs per SM the register budget is held to (no spills at 111 registers)
constexpr int SL_RING = 16;             // staged event words per symbol
constexpr int SL_MAX_SYMBOLS = 64;
constexpr int SL_REGIMES = 4;           // bull, bear, ranging, volatile; label >= 4 is "unknown"
constexpr unsigned SL_NONE = 0xffffffffu;
constexpr unsigned SL_SYMBOL_TAG = 0x9E3779B1u;   // trade_hash word of a book record (as csrc/book.cu)

struct SelParams {
    long long start_bar, check_bars;
    double expiry_s;
    double w[6];
    double risk_dd, risk_sharpe;
    int risk_vol;
    int hv_start, hv_end, la_start, la_end;
};

struct SelWarp {
    WarpAcc acc[1 + SL_REGIMES];              // the prefix, then its records of each scored regime
    uint32_t ring[SL_MAX_SYMBOLS][SL_RING];   // word i of symbol s at ring[s][i % SL_RING]
    long long cur[SL_MAX_SYMBOLS];            // next record of each symbol
    long long n_rec[SL_MAX_SYMBOLS];
    uint32_t prev[SL_MAX_SYMBOLS];            // last merged word of each symbol (the entry of its next exit)
    uint32_t bw[32], bprev[32], cw[32];
    unsigned char bs[32], cs[32];
    double cp[32];
    unsigned carry[1 + SL_REGIMES];
    int hour_n[24], hour_w[24];
    double gene[B200BT_SEL_GENES];
    double comb[5], reg[5];                   // per regime label: weighted factor sum, regime score
    double hist, risk;
    int has;                                  // a snapshot is cached
};

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }
// Python's min(a, b) / max(a, b): the first argument unless the second is strictly smaller / larger
__device__ __forceinline__ double py_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }
__device__ __forceinline__ double clamp01(double x) { return py_max(0.0, py_min(1.0, x)); }

__device__ __forceinline__ long long bar_minute(const b200bt_sweep_config& cfg, long long t) {
    return cfg.minute0 + t * cfg.bar_minutes + ((cfg.gap_bar > 0 && t >= cfg.gap_bar) ? cfg.gap_minutes : 0);
}
__device__ __forceinline__ int bar_hour(const b200bt_sweep_config& cfg, long long t) {
    return (int)((bar_minute(cfg, t) / 60) % 24);
}

// _calculate_regime_score's weighted sum (market_regime_service.py:749-760)
__device__ __forceinline__ double regime_sum(double sharpe, double win_rate, double dd, double pf) {
    double a = add(mul(sharpe, 0.3), mul(win_rate, 0.2));
    a = add(a, mul(sub(1.0, dvd(dd, 100.0)), 0.2));
    a = add(a, mul(pf, 0.3));
    return dvd(a, 1.0);
}

__device__ __forceinline__ double gene_or(const SelWarp& w, int g, double def) {
    const double x = w.gene[g];
    return isnan(x) ? def : x;
}

// The snapshot: calculate_advanced_metrics(calculate_metrics(prefix)) with the supplied regime_performance and
// hourly_performance, reduced to the parts of the factor scores that do not depend on the check (lane 0).
__device__ __forceinline__ void take_snapshot(SelWarp& w, const b200bt_sweep_config& cfg, const SelParams& p) {
    b200bt_lane_stats o;
    finalize_lane(w.acc[0], cfg, o);
    const bool one = w.acc[0].n_events < 2;    // calculate_metrics' single-record dict (:48-55)
    const double sharpe = one ? 0.0 : o.sharpe_ratio;
    const double win_rate = one ? (o.net_profit > 0.0 ? 1.0 : 0.0) : o.win_rate;
    const double dd = one ? 0.0 : o.max_drawdown;
    const double pf = one ? 0.0 : o.profit_factor;
    const double recovery = dd > 0.0 ? dvd(o.net_profit, mul(dd, 10000.0)) : INFINITY;
    // historical performance (:393-417); average_trade is absent, so its score is 0.5
    double h = add(mul(py_min(win_rate, 1.0), 0.25), mul(py_min(dvd(pf, 3.0), 1.0), 0.25));
    h = add(h, mul(py_min(dvd(sharpe, 3.0), 1.0), 0.3));
    w.hist = add(h, mul(0.5, 0.2));
    // risk (:322-363); avg_volatility is absent (0.5)
    const double avg_vol = 0.5;
    const double dd_score = dd > 0.0 ? sub(1.0, dvd(dd, p.risk_dd)) : 1.0;
    const double vol_score = p.risk_vol == 0 ? sub(1.0, py_min(avg_vol, 1.0))
                           : p.risk_vol == 1 ? sub(1.0, fabs(sub(avg_vol, 0.5))) : py_min(avg_vol, 1.0);
    const double sharpe_score = py_min(dvd(sharpe, p.risk_sharpe), 1.0);
    const double recovery_score = dvd(py_min(recovery, 2.0), 2.0);
    double r = add(mul(dd_score, 0.3), mul(sharpe_score, 0.3));
    r = add(r, mul(recovery_score, 0.2));
    r = add(r, mul(vol_score, 0.2));
    w.risk = clamp01(r);
    const double base = regime_sum(sharpe, win_rate, dd, pf);
    for (int k = 0; k < 5; ++k) {
        double f = base;
        if (k < SL_REGIMES && w.acc[1 + k].n_events > 0) {
            const WarpAcc& a = w.acc[1 + k];
            b200bt_lane_stats q;
            finalize_lane(a, cfg, q);
            const bool one_r = a.n_events < 2;
            const double rwr = dvd((double)a.n_win, (double)a.n_events);
            const double rpf = a.tot_loss != 0.0 ? dvd(add(a.tot_profit, a.tot_loss), fabs(a.tot_loss)) : 1.0;
            const double rs = regime_sum(one_r ? 0.0 : q.sharpe_ratio, rwr, one_r ? 0.0 : q.max_drawdown, rpf);
            f = add(mul(base, 0.3), mul(rs, 0.7));
        }
        // the parameter multipliers (:800-822); a NaN gene is an absent key
        if (k == B200BT_REGIME_BULL) {
            if (gene_or(w, B200BT_SEL_G_EMA_LONG, 0.0) < 30.0) f = mul(f, 1.1);
            if (gene_or(w, B200BT_SEL_G_TAKE_PROFIT, 0.0) > 5.0) f = mul(f, 1.05);
        } else if (k == B200BT_REGIME_BEAR) {
            if (gene_or(w, B200BT_SEL_G_STOP_LOSS, 100.0) < 3.0) f = mul(f, 1.1);
            if (gene_or(w, B200BT_SEL_G_RSI_OVERSOLD, 0.0) > 30.0) f = mul(f, 1.05);
        } else if (k == B200BT_REGIME_RANGING) {
            if (gene_or(w, B200BT_SEL_G_BOLLINGER_STD, 0.0) > 2.0) f = mul(f, 1.1);
            if (gene_or(w, B200BT_SEL_G_RSI_PERIOD, 0.0) < 14.0) f = mul(f, 1.05);
        } else if (k == B200BT_REGIME_VOLATILE) {
            if (gene_or(w, B200BT_SEL_G_ATR_MULTIPLIER, 0.0) > 2.0) f = mul(f, 1.1);
            if (gene_or(w, B200BT_SEL_G_ATR_PERIOD, 0.0) < 10.0) f = mul(f, 1.05);
        }
        w.reg[k] = clamp01(f);
    }
    for (int k = 0; k < 5; ++k) {     // the weighted sum (:821-828), social and feature importance 0.5, volatility 0.6
        double c = add(mul(w.reg[k], p.w[0]), mul(w.hist, p.w[1]));
        c = add(c, mul(w.risk, p.w[2]));
        c = add(c, mul(0.5, p.w[3]));
        c = add(c, mul(0.6, p.w[4]));
        w.comb[k] = add(c, mul(0.5, p.w[5]));
    }
    w.has = 1;
}

__device__ __forceinline__ unsigned head_bar(const SelWarp& w, int s, int S) {
    if (s >= S) return SL_NONE;
    const long long c = w.cur[s];
    return c < w.n_rec[s] ? (w.ring[s][c % SL_RING] & B200BT_EVENT_BAR_MASK) : SL_NONE;
}

__device__ __forceinline__ unsigned next_bar(const SelWarp& w, int S) {
    const int lane = threadIdx.x & 31;
    return __reduce_min_sync(FULL, min(head_bar(w, lane, S), head_bar(w, lane + 32, S)));
}

// Price and account n <= 32 merged records staged in bw / bs / bprev.
__device__ __forceinline__ void process_records(SelWarp& w, int n, const float* __restrict__ price, int64_t ld_price,
                                const uint8_t* __restrict__ labels, int64_t ld_labels, const b200bt_sweep_config& cfg) {
    const int lane = threadIdx.x & 31;
    const bool act = lane < n;
    const unsigned wd = act ? w.bw[lane] : 0u, wp = act ? w.bprev[lane] : 0u;
    const unsigned s = act ? w.bs[lane] : 0u;
    const unsigned bar = wd & B200BT_EVENT_BAR_MASK;
    const float* row = price + (int64_t)s * ld_price;
    const float pf = act ? __ldg(row + bar) : 0.f;
    const float pp = (act && (wd & B200BT_EVENT_EXIT)) ? __ldg(row + (wp & B200BT_EVENT_BAR_MASK)) : 0.f;
    int dur;
    const double pnl = record_pnl(act, wd, pf, wp, pp, w.acc[0].size, w.acc[0].fee1, w.acc[0].fee2, dur);
    const unsigned c0 = merged_records(&w.acc[0], n, act, wd, wd ^ (s * SL_SYMBOL_TAG), pnl, w.carry[0], cfg);
    if (act) {
        const int h = bar_hour(cfg, bar);
        atomicAdd(&w.hour_n[h], 1);
        if (pnl > 0.0) atomicAdd(&w.hour_w[h], 1);
    }
    const unsigned cls = act ? (unsigned)__ldg(labels + (int64_t)s * ld_labels + bar) : SL_NONE;
    unsigned todo = __ballot_sync(FULL, cls < (unsigned)SL_REGIMES);
    __syncwarp();
    if (lane == 0) w.carry[0] = c0;
    while (todo) {
        const unsigned r = __shfl_sync(FULL, cls, __ffs(todo) - 1);
        const unsigned m = __ballot_sync(FULL, cls == r);
        todo &= ~m;
        if (cls == r) {
            const int rank = __popc(m & ((1u << lane) - 1u));
            w.cw[rank] = wd;
            w.cs[rank] = (unsigned char)s;
            w.cp[rank] = pnl;
        }
        __syncwarp();
        const int nr = __popc(m);
        const bool a2 = lane < nr;
        const unsigned w2 = a2 ? w.cw[lane] : 0u, s2 = a2 ? w.cs[lane] : 0u;
        const double p2 = a2 ? w.cp[lane] : 0.0;
        const unsigned cr = merged_records(&w.acc[1 + r], nr, a2, w2, w2 ^ (s2 * SL_SYMBOL_TAG), p2, w.carry[1 + r], cfg);
        if (lane == 0) w.carry[1 + r] = cr;
        __syncwarp();
    }
}

// Merge and account every record with bar <= limit.
__device__ __forceinline__ void consume(SelWarp& w, unsigned limit, int S, const uint32_t* __restrict__ ev, int64_t event_cap,
                        const float* __restrict__ price, int64_t ld_price, const uint8_t* __restrict__ labels,
                        int64_t ld_labels, const b200bt_sweep_config& cfg) {
    const int lane = threadIdx.x & 31;
    int n = 0;
    while (true) {
        const unsigned h0 = head_bar(w, lane, S), h1 = head_bar(w, lane + 32, S);
        const unsigned b = __reduce_min_sync(FULL, min(h0, h1));
        if (b == SL_NONE || b > limit) break;
        const unsigned sc = __reduce_min_sync(FULL, h0 == b ? (unsigned)lane : h1 == b ? (unsigned)lane + 32u : 255u);
        if (lane == (int)(sc & 31u)) {
            const long long c = w.cur[sc];
            const uint32_t wd = w.ring[sc][c % SL_RING];
            w.bw[n] = wd;
            w.bs[n] = (unsigned char)sc;
            w.bprev[n] = w.prev[sc];
            w.prev[sc] = wd;
            w.cur[sc] = c + 1;
        }
        __syncwarp();
        const long long c = w.cur[sc];
        if (c % SL_RING == 0 && c < w.n_rec[sc]) {
            if (lane < SL_RING)
                w.ring[sc][lane] = c + lane < w.n_rec[sc] ? __ldg(ev + (int64_t)sc * event_cap + c + lane) : 0u;
            __syncwarp();
        }
        if (++n == 32) {
            process_records(w, n, price, ld_price, labels, ld_labels, cfg);
            n = 0;
        }
    }
    if (n) process_records(w, n, price, ld_price, labels, ld_labels, cfg);
}

__global__ void __launch_bounds__(SL_WARPS * 32, SL_MIN_BLOCKS)
selection_kernel(const float* __restrict__ price, int64_t ld_price, int S, const b200bt_individual* __restrict__ indiv,
                 int n_indiv, const b200bt_sweep_config cfg, const b200bt_lane_stats* __restrict__ lane_stats,
                 const uint32_t* __restrict__ events, int64_t event_cap, const uint8_t* __restrict__ labels,
                 int64_t ld_labels, const int32_t* __restrict__ cand_row, const int32_t* __restrict__ cand_index,
                 const double* __restrict__ genes, int n_cand, int K, const SelParams p, int64_t n_checks,
                 double* __restrict__ rows, double* __restrict__ scores, int32_t* __restrict__ locks) {
    __shared__ SelWarp shared[SL_WARPS];
    const int lane = threadIdx.x & 31;
    const int k = blockIdx.x * SL_WARPS + (threadIdx.x >> 5);
    if (k >= n_cand) return;
    SelWarp& w = shared[threadIdx.x >> 5];
    const int row = cand_row[k], idx = cand_index[k];
    if (idx < 0 || idx >= K) return;
    bool bad = row < 0 || row >= n_indiv;
    for (int s = lane; s < S; s += 32) {
        const long long n = bad ? 0 : (long long)lane_stats[(int64_t)row * S + s].n_records;
        w.cur[s] = 0;
        w.n_rec[s] = n;
        w.prev[s] = 0u;
        bad |= n > event_cap;
    }
    if (__any_sync(FULL, bad)) {      // records lost to the event buffer (or a bad row): no scores, never selected
        if (scores)
            for (int64_t c = lane; c < n_checks; c += 32) scores[c * K + idx] = NAN;
        return;
    }
    __syncwarp();                     // n_rec[] of other lanes' symbols is read below
    const uint32_t* ev = events + (int64_t)row * S * event_cap;
    for (int f = lane; f < S * SL_RING; f += 32) {
        const int s = f / SL_RING, j = f - s * SL_RING;
        w.ring[s][j] = j < w.n_rec[s] ? __ldg(ev + (int64_t)s * event_cap + j) : 0u;
    }
    if (lane < B200BT_SEL_GENES) w.gene[lane] = genes[(int64_t)k * B200BT_SEL_GENES + lane];
    if (lane < 24) w.hour_n[lane] = w.hour_w[lane] = 0;
    if (lane <= SL_REGIMES) {
        init_acc(w.acc[lane], indiv[row], cfg, nullptr);
        w.carry[lane] = 0u;
    }
    if (lane == 0) w.has = 0;
    __syncwarp();

    // factor scores of an empty snapshot: regime 0, historical 0, risk 0, social 0.5, volatility 0.5, feature 0.5
    double empty = add(mul(0.0, p.w[0]), mul(0.0, p.w[1]));
    empty = add(add(add(add(empty, mul(0.0, p.w[2])), mul(0.5, p.w[3])), mul(0.5, p.w[4])), mul(0.5, p.w[5]));
    const double atr = gene_or(w, B200BT_SEL_G_ATR_MULTIPLIER, 1.0);
    const double high_term = mul(py_min(dvd(atr, 2.0), 1.0), 0.05);
    const double low_term = mul(py_max(0.0, sub(1.0, dvd(10.0, 20.0))), 0.05);    // avg_trades_per_hour absent (10)

    unsigned first = next_bar(w, S);      // bar of the next record: the first fetch that finds a prefix
    long long tau = 0;                    // minute of the cached snapshot's fetch
    int64_t c = 0;
    while (c < n_checks) {
        const int64_t j = c + lane;
        const bool in = j < n_checks;
        const long long t = p.start_bar + j * p.check_bars;
        bool need = false;
        if (in) need = w.has ? (double)((bar_minute(cfg, t) - tau) * 60) >= p.expiry_s : (unsigned long long)t >= first;
        const unsigned m = __ballot_sync(FULL, need);
        const int stop = m ? __ffs(m) - 1 : 32;
        if (in && lane < stop) {
            const unsigned lab = __ldg(labels + t);
            const int rho = lab < SL_REGIMES ? (int)lab : SL_REGIMES;
            const int h = bar_hour(cfg, t);
            double x = w.has ? w.comb[rho] : empty;
            if (w.has && w.hour_n[h] >= 10) {     // apply_time_based_adjustments (:720-757)
                const double wr = dvd((double)w.hour_w[h], (double)w.hour_n[h]);
                x = add(x, mul(mul(sub(wr, 0.5), 2.0), 0.1));
            }
            if (p.hv_start <= h && h < p.hv_end) x = add(x, high_term);
            if (p.la_start <= h && h < p.la_end) x = add(x, low_term);
            const double score = clamp01(x);
            if (scores) scores[j * K + idx] = score;
            double* r = rows + j * B200BT_SEL_ROW_WORDS;
            // A row's score never decreases, so a strictly higher score read without the lock stays ahead; an equal one
            // is decided under the lock, where BEST and SCORE are read as one pair.
            if (!(__ldcg(r + B200BT_SEL_R_SCORE) > score)) {
                while (atomicCAS(locks + j, 0, 1) != 0) __nanosleep(64);
                __threadfence();
                const double qb = __ldcg(r + B200BT_SEL_R_BEST), qs = __ldcg(r + B200BT_SEL_R_SCORE);
                if (!(qb >= 0.0 && (qs > score || (qs == score && qb < (double)idx)))) {
                    __stcg(r + B200BT_SEL_R_BEST, (double)idx);
                    __stcg(r + B200BT_SEL_R_SCORE, score);
                    __stcg(r + B200BT_SEL_R_MARKET_REGIME, w.has ? w.reg[rho] : 0.0);
                    __stcg(r + B200BT_SEL_R_HISTORICAL_PERFORMANCE, w.has ? w.hist : 0.0);
                    __stcg(r + B200BT_SEL_R_RISK_PROFILE, w.has ? w.risk : 0.0);
                    __stcg(r + B200BT_SEL_R_SOCIAL_SENTIMENT, 0.5);
                    __stcg(r + B200BT_SEL_R_MARKET_VOLATILITY, w.has ? 0.6 : 0.5);
                    __stcg(r + B200BT_SEL_R_FEATURE_IMPORTANCE, 0.5);
                }
                __threadfence();
                atomicExch(locks + j, 0);
            }
        }
        __syncwarp();
        if (!m) {
            c += 32;
            continue;
        }
        c += stop;     // check c refreshes: consume its prefix, retake the snapshot, evaluate it in the next pass
        const long long tc = p.start_bar + c * p.check_bars;
        consume(w, (unsigned)tc, S, ev, event_cap, price, ld_price, labels, ld_labels, cfg);
        if (lane == 0) take_snapshot(w, cfg, p);
        __syncwarp();
        tau = bar_minute(cfg, tc);
        first = next_bar(w, S);
    }
}

__global__ void selection_init_kernel(const uint8_t* __restrict__ labels, long long start_bar, long long check_bars,
                                      int64_t n_checks, double* __restrict__ rows, int32_t* __restrict__ locks) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_checks) return;
    const long long t = start_bar + c * check_bars;
    const unsigned lab = labels[t];
    double* r = rows + c * B200BT_SEL_ROW_WORDS;
    r[B200BT_SEL_R_BAR] = (double)t;
    r[B200BT_SEL_R_REGIME] = (double)(lab < SL_REGIMES ? lab : SL_REGIMES);
    r[B200BT_SEL_R_BEST] = -1.0;
    for (int f = B200BT_SEL_R_SCORE; f <= B200BT_SEL_R_FEATURE_IMPORTANCE; ++f) r[f] = NAN;
    r[B200BT_SEL_R_ACTIVE] = -1.0;
    r[B200BT_SEL_R_ACTIVE_SCORE] = 0.0;
    locks[c] = 0;
}

__global__ void __launch_bounds__(32)
selection_switch_kernel(double* __restrict__ rows, int64_t n_checks, double min_improvement, double min_confidence,
                        int32_t* __restrict__ switches, int32_t* __restrict__ n_switches) {
    const int lane = threadIdx.x;
    double active = -1.0, active_score = 0.0;
    int n_sw = 0;
    for (int64_t base = 0; base < n_checks; base += 32) {
        const int64_t j = base + lane;
        const bool in = j < n_checks;
        double* r = rows + j * B200BT_SEL_ROW_WORDS;
        const double best = in ? r[B200BT_SEL_R_BEST] : -1.0;
        const double score = in ? r[B200BT_SEL_R_SCORE] : NAN;
        double my_active = active, my_score = active_score;
        int from = 0;
        while (true) {
            // should_switch_strategy: another strategy, improvement > threshold, confidence > threshold
            const bool sw = in && lane >= from && best >= 0.0 && best != active &&
                            sub(score, active_score) > min_improvement && score > min_confidence;
            const unsigned m = __ballot_sync(FULL, sw);
            if (!m) break;
            const int l = __ffs(m) - 1;
            active = __shfl_sync(FULL, best, l);
            active_score = __shfl_sync(FULL, score, l);
            if (lane >= l) { my_active = active; my_score = active_score; }
            if (lane == l) switches[n_sw] = (int32_t)j;
            ++n_sw;
            from = l + 1;
        }
        if (in) {
            r[B200BT_SEL_R_ACTIVE] = my_active;
            r[B200BT_SEL_R_ACTIVE_SCORE] = my_score;
        }
    }
    if (lane == 0) *n_switches = n_sw;
}

static bool integral(double x) { return isfinite(x) && x == floor(x); }

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_selection_replay(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv,
                                       int n_indiv, const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats,
                                       const uint32_t* events, int64_t event_cap, const uint8_t* labels, int64_t ld_labels,
                                       const int32_t* cand_row, const int32_t* cand_index, const double* genes, int n_cand,
                                       int K, const double* params_host, int64_t n_checks, int merge, double* rows,
                                       double* scores_or_null, int32_t* check_locks, b200bt_stream_t stream) {
    B200BT_REQUIRE(cfg && labels && cand_row && cand_index && genes && params_host && rows && check_locks && events,
                   B200BT_EINVAL, "selection_replay: null pointer");
    int rc = check_record_args("selection_replay", price, ld_price, S, N, indiv, n_indiv, cfg, lane_stats, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE(event_cap >= 1, B200BT_EINVAL, "selection_replay: event_cap must be >= 1");
    B200BT_REQUIRE(S <= SL_MAX_SYMBOLS, B200BT_ELIMIT, "selection_replay: at most %d symbols (S = %d)", SL_MAX_SYMBOLS, S);
    B200BT_REQUIRE(ld_labels == 0 || ld_labels >= N, B200BT_EINVAL,
                   "selection_replay: ld_labels must be 0 (one shared row) or >= N");
    B200BT_REQUIRE(n_cand >= 1 && K >= 1 && n_cand <= K, B200BT_EINVAL, "selection_replay: need 1 <= n_cand <= K");
    B200BT_REQUIRE(merge == 0 || merge == 1, B200BT_EINVAL, "selection_replay: merge must be 0 or 1");
    const double* q = params_host;
    B200BT_REQUIRE(integral(q[B200BT_SEL_P_CHECK_BARS]) && q[B200BT_SEL_P_CHECK_BARS] >= 1.0 &&
                   q[B200BT_SEL_P_CHECK_BARS] <= (double)N, B200BT_EINVAL,
                   "selection_replay: check_bars must be an integer in [1, N]");
    B200BT_REQUIRE(integral(q[B200BT_SEL_P_START_BAR]) && q[B200BT_SEL_P_START_BAR] >= 0.0 &&
                   q[B200BT_SEL_P_START_BAR] < (double)N, B200BT_EINVAL, "selection_replay: start_bar outside [0, N)");
    B200BT_REQUIRE(q[B200BT_SEL_P_CACHE_EXPIRY] > 0.0 && q[B200BT_SEL_P_CACHE_EXPIRY] < INFINITY, B200BT_EINVAL,
                   "selection_replay: cache expiry must be positive and finite");
    B200BT_REQUIRE(q[B200BT_SEL_P_RISK_MAX_DRAWDOWN] != 0.0 && q[B200BT_SEL_P_RISK_MIN_SHARPE] != 0.0, B200BT_EINVAL,
                   "selection_replay: the risk profile's max_drawdown and min_sharpe must be non-zero");
    const double vp = q[B200BT_SEL_P_RISK_VOLATILITY];
    B200BT_REQUIRE(vp == 0.0 || vp == 1.0 || vp == 2.0, B200BT_EINVAL,
                   "selection_replay: the risk profile's volatility preference must be 0, 1 or 2");
    for (int h = B200BT_SEL_P_HIGH_VOL_START; h <= B200BT_SEL_P_LOW_ACTIVITY_END; ++h)
        B200BT_REQUIRE(integral(q[h]) && fabs(q[h]) <= 48.0, B200BT_EINVAL, "selection_replay: window hours must be integers");
    SelParams p;
    p.start_bar = (long long)q[B200BT_SEL_P_START_BAR];
    p.check_bars = (long long)q[B200BT_SEL_P_CHECK_BARS];
    p.expiry_s = q[B200BT_SEL_P_CACHE_EXPIRY];
    for (int f = 0; f < 6; ++f) p.w[f] = q[B200BT_SEL_P_W_MARKET_REGIME + f];
    p.risk_dd = q[B200BT_SEL_P_RISK_MAX_DRAWDOWN];
    p.risk_sharpe = q[B200BT_SEL_P_RISK_MIN_SHARPE];
    p.risk_vol = (int)vp;
    p.hv_start = (int)q[B200BT_SEL_P_HIGH_VOL_START];
    p.hv_end = (int)q[B200BT_SEL_P_HIGH_VOL_END];
    p.la_start = (int)q[B200BT_SEL_P_LOW_ACTIVITY_START];
    p.la_end = (int)q[B200BT_SEL_P_LOW_ACTIVITY_END];
    const int64_t max_checks = (N - 1 - p.start_bar) / p.check_bars + 1;
    B200BT_REQUIRE(n_checks >= 1 && n_checks <= max_checks, B200BT_EINVAL,
                   "selection_replay: n_checks must be in [1, %lld]", (long long)max_checks);
    rc = check_device();
    if (rc) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    if (!merge) {
        selection_init_kernel<<<(unsigned)((n_checks + 255) / 256), 256, 0, st>>>(labels, p.start_bar, p.check_bars, n_checks,
                                                                                  rows, check_locks);
        B200BT_LAUNCH_CHECK("selection_replay (init)");
    }
    selection_kernel<<<(unsigned)((n_cand + SL_WARPS - 1) / SL_WARPS), SL_WARPS * 32, 0, st>>>(
        price, ld_price, S, indiv, n_indiv, *cfg, lane_stats, events, event_cap, labels, ld_labels, cand_row, cand_index,
        genes, n_cand, K, p, n_checks, rows, scores_or_null, check_locks);
    B200BT_LAUNCH_CHECK("selection_replay");
    return B200BT_OK;
}

extern "C" int b200bt_selection_switch(double* rows, int64_t n_checks, const double* params_host, int32_t* switch_checks,
                                       int32_t* n_switches, b200bt_stream_t stream) {
    B200BT_REQUIRE(rows && params_host && switch_checks && n_switches, B200BT_EINVAL, "selection_switch: null pointer");
    B200BT_REQUIRE(n_checks >= 1, B200BT_EINVAL, "selection_switch: n_checks must be >= 1");
    B200BT_REQUIRE(n_checks < (1ll << 31), B200BT_ELIMIT, "selection_switch: n_checks must be < 2^31");
    const int rc = check_device();
    if (rc) return rc;
    selection_switch_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(rows, n_checks, params_host[B200BT_SEL_P_MIN_IMPROVEMENT],
                                                                params_host[B200BT_SEL_P_MIN_CONFIDENCE], switch_checks,
                                                                n_switches);
    B200BT_LAUNCH_CHECK("selection_switch");
    return B200BT_OK;
}
