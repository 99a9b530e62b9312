// Code shared by the fused population sweep (sweep.cu) and the time-chunked sweep
// (sweep_chunked.cu): the per-warp shared-memory working set; the warp-per-lane bar scan that
// sweep_kernel and the warp-per-chunk scan / repair kernels run (machine, cp.async group ring,
// group step, force-close); the event-batch arithmetic (calculate_metrics) and the score epilogue;
// the host-side argument checks and launch set-up of the warp-per-lane kernels.
#pragma once
#include <math.h>
#include "common.cuh"

namespace b200bt {

// the fused sweep over a device-side list of individuals (sweep.cu): the exact fallback of the time-chunked sweeps
int launch_sweep(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                 const b200bt_individual* indiv, const int32_t* order, int pop, const int* pop_dev,
                 const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats, uint32_t* events, int64_t event_cap,
                 cudaStream_t stream);

// The calendar clock of b200bt_sweep_config, checked on the host by all three sweep entry points (N < 2^30 already checked):
// a negative field (minute0, gap_minutes) or bar_minutes <= 0 is B200BT_EINVAL; minute0 + N * bar_minutes + gap_minutes
// >= 2^32 - 1440 is B200BT_ELIMIT, so that every minute the kernels form fits their unsigned 32-bit arithmetic.
int check_sweep_clock(const char* who, const b200bt_sweep_config* cfg, int64_t N);

// The arguments all three sweep entry points take alike: price / RSI rows and their strides, P, S, N (< 2^30), the calendar
// clock (check_sweep_clock) and the optional event buffer.  B200BT_OK, or the first failing check's status.
int check_sweep_args(const char* who, const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S,
                     int64_t N, const b200bt_sweep_config* cfg_host, const uint32_t* events, int64_t event_cap);

// The checks the passes over a sweep's records share; the clock (check_sweep_clock) only with a `cfg` (trade_pnl has none).
int check_record_args(const char* who, const float* price, int64_t ld_price, int S, int64_t N,
                      const b200bt_individual* indiv, int pop, const b200bt_sweep_config* cfg,
                      const b200bt_lane_stats* lane_stats, const uint32_t* events, int64_t event_cap);

// price and RSI rows that allow 16-byte copies: every (symbol, period) row starts on a 16-byte boundary
bool vec16_rows(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi);

constexpr int SW_WARPS = 8;         // warps (lanes of the sweep) per CTA
#ifndef B200BT_SW_MIN_BLOCKS
#define B200BT_SW_MIN_BLOCKS 2
#endif
constexpr int SW_MIN_BLOCKS = B200BT_SW_MIN_BLOCKS;    // CTAs per SM the register budget is held to (<= 64 regs/thread)
#ifndef B200BT_SW_GROUP
#define B200BT_SW_GROUP 512
#endif
#ifndef B200BT_SW_STAGES
#define B200BT_SW_STAGES 2
#endif
// 512 bars x 2 stages measured best on the C2 workload (256x3: +5 %, 128x4: +18 %; tools/build_variant.py)
constexpr int SW_GROUP = B200BT_SW_GROUP;     // bars per cp.async group (per stream)
constexpr int SW_STAGES = B200BT_SW_STAGES;   // shared-memory ring depth per warp
constexpr int SW_EVQ = 128;         // event queue entries per warp (>= 32 + 64 new events per window pair)
constexpr float SW_MARGIN = 1e-6f;  // relative width of the fp32 screening band

// Warp-uniform per-lane constants of the bar scan (shared memory; read on events only).
struct ScanConst {
    float os_f, ob_f;
    // screening multipliers: candidate (c) and definite (d) bounds
    float hiL_c, hiL_d, loL_c, loL_d;  // long : TP above, SL below
    float hiS_c, hiS_d, loS_c, loS_d;  // short: SL above, TP below
};

// Everything only the event-batch code touches lives in shared memory (one slot
// per warp) so that the bar scan keeps a small register footprint.
struct WarpAcc {
    double tp, sl, size, fee1, fee2;
    double equity, peak, maxdd;
    double tot_profit, tot_loss, largest_p, largest_l;
    double day_sum, pivot, s1, s2;
    long long day_cur;
    long long sum_dur;
    unsigned long long hash;
    uint32_t* ev_out;
    unsigned n_win, n_loss, n_days, n_events;
    int day_valid, pivot_set;
    // chunk-parallel metrics only: the first calendar day of a chunk may continue the previous chunk's
    // last day, so its sum is kept aside instead of being counted as a finished day
    int hold_first, first_done, first_day;
    double first_sum;
    double npivot, ns1, ns2;     // negative days (DayAcc)
    unsigned n_neg;
    unsigned gap_bar, gap_minutes;   // calendar clock of a glued series (b200bt_sweep_config); gap_bar = ~0u: none
};

// Per-warp shared-memory working set.
struct __align__(16) WarpShared {
    float ring[SW_STAGES][2][SW_GROUP];  // cp.async ring: [stage][0 price | 1 rsi][bar]
    uint2 evq[SW_EVQ];                   // event queue: (event word, price bits), consumed 32 at a time
    WarpAcc acc;
    ScanConst sc;
};

// Dynamic shared memory of a warp-per-lane kernel (sweep_kernel, chunk_scan_kernel, chunk_repair_kernel,
// lane_repair_kernel): one WarpShared per warp.
constexpr size_t SW_SMEM = sizeof(WarpShared) * SW_WARPS;
template <class Kernel>
int allow_sw_smem(Kernel kern, const char* what) {
    return cuda_status(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SW_SMEM), what);
}

struct DayAcc {
    double pivot, s1, s2;
    unsigned n_days;
    int pivot_set;
    // the negative days alone (Sortino's downside deviation), same shifted accumulation
    double npivot = 0.0, ns1 = 0.0, ns2 = 0.0;
    unsigned n_neg = 0;
};

__device__ __forceinline__ void day_complete(DayAcc& a, double x) {
    // shifted-data accumulation of the daily pnl sums (exactly 0 variance for equal days)
    if (!a.pivot_set) { a.pivot = x; a.pivot_set = 1; }
    const double y = x - a.pivot;
    a.s1 += y;
    a.s2 += y * y;
    a.n_days += 1;
    if (x < 0.0) {
        if (a.n_neg == 0) a.npivot = x;
        const double z = x - a.npivot;
        a.ns1 += z;
        a.ns2 += z * z;
        a.n_neg += 1;
    }
}

// Append the days of `b` (which come after those of `a`) to `a`: b's moments are shifted from its pivots to a's (an
// empty `a` takes b's pivots, shift 0).
__device__ __forceinline__ void day_merge(DayAcc& a, const DayAcc& b) {
    if (b.n_days) {
        if (a.n_days == 0) { a.pivot = b.pivot; a.pivot_set = 1; }
        const double d = b.pivot - a.pivot, n = (double)b.n_days;
        a.s1 += b.s1 + n * d;
        a.s2 += b.s2 + 2.0 * d * b.s1 + n * d * d;
        a.n_days += b.n_days;
    }
    if (b.n_neg) {
        if (a.n_neg == 0) a.npivot = b.npivot;
        const double d = b.npivot - a.npivot, n = (double)b.n_neg;
        a.ns1 += b.ns1 + n * d;
        a.ns2 += b.ns2 + 2.0 * d * b.ns1 + n * d * d;
        a.n_neg += b.n_neg;
    }
}

// PnL of one trade record (strategy_evaluation.py:798,:819,:836): an entry record costs the entry fee,
// an exit record realises quantity * move - both fees, with quantity = position_size / entry_price.
__device__ __forceinline__ double record_pnl(bool active, unsigned w, float pf, unsigned w_prev, float p_prev,
                                             double size, double fee1, double fee2, int& dur) {
    dur = 0;
    if (!active) return 0.0;
    if (w & B200BT_EVENT_EXIT) {
        const double e = (double)p_prev, px = (double)pf;
        const double qty = __ddiv_rn(size, e);
        const double diff = (w_prev & B200BT_EVENT_SELL) ? __dsub_rn(e, px) : __dsub_rn(px, e);
        dur = (int)((w & B200BT_EVENT_BAR_MASK) - (w_prev & B200BT_EVENT_BAR_MASK));
        return __dsub_rn(__dmul_rn(qty, diff), fee2);
    }
    return -fee1;
}

// One (individual, symbol) lane's records in a sweep's event buffer, as the passes over them read it (lane w = i * S + s).
struct LaneRecords {
    const uint32_t* ev;          // event words
    const float* price;          // close prices of the lane's symbol
    int64_t n;                   // records
    double size, fee1, fee2;     // position size, entry fee, the exit's fees (init_acc's)
};

// Fill `r` for lane w.  False when the event buffer lost records of the lane (n_records > event_cap): only r.n is set then.
__device__ __forceinline__ bool read_lane(LaneRecords& r, int64_t w, int S, const float* __restrict__ price,
                                          int64_t ld_price, const b200bt_individual* __restrict__ indiv,
                                          const b200bt_lane_stats* __restrict__ lane_stats,
                                          const uint32_t* __restrict__ events, int64_t event_cap) {
    r.n = (int64_t)lane_stats[w].n_records;
    if (r.n > event_cap) return false;
    r.size = indiv[w / S].position_size;
    r.fee1 = __dmul_rn(r.size, 0.001);
    r.fee2 = __dmul_rn(r.size, 0.002);
    r.ev = events + w * event_cap;
    r.price = price + (int64_t)(int)(w % S) * ld_price;
    return true;
}

// Records [base, base + 32) of a lane, base even, lane j holding record base + j: an exit is priced against the entry before it.
struct RecordBatch { bool active; int n; unsigned w, bar; double pnl; };

__device__ __forceinline__ RecordBatch record_batch(const LaneRecords& r, int64_t base) {
    RecordBatch b;
    const int64_t j = base + (threadIdx.x & 31);
    b.active = j < r.n;
    b.n = (int)min((int64_t)32, r.n - base);
    b.w = b.active ? __ldg(r.ev + j) : 0u;
    b.bar = b.w & B200BT_EVENT_BAR_MASK;
    const float pf = b.active ? __ldg(r.price + b.bar) : 0.f;
    const unsigned w_prev = __shfl_up_sync(FULL, b.w, 1);
    const float p_prev = __shfl_up_sync(FULL, pf, 1);
    int dur;
    b.pnl = record_pnl(b.active, b.w, pf, w_prev, p_prev, r.size, r.fee1, r.fee2, dur);
    return b;
}

// Stats of a lane or book some of whose records the event buffer lost: n_records = -1, score = NaN, the rest zero.
__device__ __forceinline__ b200bt_lane_stats lost_lane_stats() {
    b200bt_lane_stats o = {};
    o.n_records = -1.0;
    o.score = NAN;
    return o;
}

// Calendar day of bar `bar` in unsigned 32-bit minutes (exact: check_sweep_clock); gap_bar = ~0u: no gap.  The gap goes by
// reference so that batch_records reads its WarpAcc's gap_minutes only for a bar past the gap, as it always has.
__device__ __forceinline__ unsigned record_day(unsigned minute0, unsigned bar, unsigned bar_minutes, const unsigned& gap_bar,
                                               const unsigned& gap_minutes) {
    return (minute0 + bar * bar_minutes + (bar >= gap_bar ? gap_minutes : 0u)) / 1440u;
}

// Inclusive warp sum of `x` over each calendar day of records [0, cnt) in time order; `tail`: the day's last record.
__device__ __forceinline__ double day_segments(double x, int day, bool active, int cnt, bool& tail) {
    const int lane = threadIdx.x & 31;
    const int day_prev = __shfl_up_sync(FULL, day, 1);
    const int day_next = __shfl_down_sync(FULL, day, 1);
    tail = active && (lane == cnt - 1 || day != day_next);
    double seg = x;
    bool flag = active && (lane == 0 || day != day_prev);      // the day's first record
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        double up = shfl_up_d(seg, d);
        int fup = __shfl_up_sync(FULL, (int)flag, d);
        if (lane >= d && !flag) { seg += up; flag = fup; }
    }
    return seg;
}

// Advance the trade-record metrics of calculate_metrics (strategy_evaluation.py:97-188) in `acc` (shared memory, one slot
// per warp) by `cnt` records in time order, already priced: lane j holds record j (event word w, pnl, duration dur counted
// on this record).  `hw` is the word the trade hash mixes (w for a lane; w tagged with its symbol for a book, csrc/book.cu).
__device__ __forceinline__ void batch_records(WarpAcc* __restrict__ acc, int cnt, bool active, unsigned w, unsigned hw,
                                              double pnl, int dur, long long minute0, int bar_minutes, int64_t ev_cap) {
    const int lane = threadIdx.x & 31;
    const unsigned bar = w & B200BT_EVENT_BAR_MASK;
    // wins / losses
    const bool win = active && pnl > 0.0, loss = active && pnl < 0.0;
    const unsigned n_win = acc->n_win + __popc(__ballot_sync(FULL, win));
    const unsigned n_loss = acc->n_loss + __popc(__ballot_sync(FULL, loss));
    double largest_p = acc->largest_p, largest_l = acc->largest_l;
    if (__any_sync(FULL, pnl > largest_p)) largest_p = fmax(largest_p, warp_max_d(win ? pnl : 0.0));   // rare after warm-up
    if (__any_sync(FULL, pnl < largest_l)) largest_l = fmin(largest_l, warp_min_d(loss ? pnl : 0.0));
    const long long sum_dur = acc->sum_dur + __reduce_add_sync(FULL, dur);

    // equity curve: inclusive scan of pnl, running peak, drawdown
    double cs = pnl;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        double up = shfl_up_d(cs, d);
        if (lane >= d) cs += up;
    }
    // gains by one butterfly; losses = batch total - gains (the total comes free from the scan)
    const double gains = warp_sum_d(win ? pnl : 0.0);
    const double tot_profit = acc->tot_profit + gains;
    const double tot_loss = __any_sync(FULL, loss) ? acc->tot_loss + (__shfl_sync(FULL, cs, 31) - gains) : acc->tot_loss;
    const double eq = acc->equity + cs;
    const double peak_in = acc->peak;
    double pk = peak_in;
    if (__any_sync(FULL, active && eq > peak_in)) {   // a new equity peak inside the batch (uncommon for most lanes)
        pk = active ? eq : -INFINITY;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            double up = shfl_up_d(pk, d);
            if (lane >= d) pk = fmax(pk, up);
        }
        pk = fmax(pk, peak_in);
    }
    double maxdd = acc->maxdd;
    {
        // dd_j = (pk-eq)/pk; a new maximum needs (pk-eq) > maxdd*pk (screen with a safety factor, then divide)
        const double gap = __dsub_rn(pk, eq);
        const bool cand = active && gap > 0.0 && gap >= maxdd * pk * (1.0 - 1e-12);
        if (__any_sync(FULL, cand)) maxdd = fmax(maxdd, warp_max_d(cand ? __ddiv_rn(gap, pk) : 0.0));
    }
    const double batch_sum = shfl_d(cs, 31);
    const double equity_out = acc->equity + batch_sum;
    const double peak_out = shfl_d(pk, cnt - 1);

    // daily buckets: segmented sum by calendar day over the batch, merged with the carry day
    const int day = active ? (int)record_day((unsigned)minute0, bar, (unsigned)bar_minutes, acc->gap_bar, acc->gap_minutes) : 0;
    DayAcc da{acc->pivot, acc->s1, acc->s2, acc->n_days, acc->pivot_set, acc->npivot, acc->ns1, acc->ns2, acc->n_neg};
    const int hold_first = acc->hold_first;
    int first_done = acc->first_done, first_id = acc->first_day;
    double first_sum = acc->first_sum;
    auto finish_day = [&](int id, double x) {
        if (hold_first && !first_done) { first_done = 1; first_id = id; first_sum = x; }
        else day_complete(da, x);
    };
    const int day_valid = acc->day_valid;
    const int day_cur = (int)acc->day_cur;
    double day_sum = acc->day_sum;
    const int first_day = __shfl_sync(FULL, day, 0);
    const int last_day = __shfl_sync(FULL, day, cnt - 1);
    if (first_day == last_day && (!day_valid || first_day == day_cur)) {
        // common case: the whole batch falls into the open day
        day_sum = (day_valid ? day_sum : 0.0) + batch_sum;
    } else {
        bool tail;
        double seg = day_segments(pnl, day, active, cnt, tail);
        const bool merge_carry = day_valid && (first_day == day_cur);
        // a tail in the first segment (its day == first_day) absorbs the carry
        if (tail && merge_carry && day == first_day) seg += day_sum;
        const bool last_seg_tail = tail && (lane == cnt - 1);
        // completed days: every tail except the batch's last one (which stays open) ...
        const double x = (tail && !last_seg_tail) ? seg : 0.0;
        unsigned done = __ballot_sync(FULL, tail && !last_seg_tail);
        // ... plus the carried day when the batch starts on a later day;
        // fold in time order (carry first, then lanes ascending)
        if (day_valid && !merge_carry) finish_day(day_cur, day_sum);
        while (done) {
            const int j = __ffs(done) - 1;
            done &= done - 1;
            finish_day(__shfl_sync(FULL, day, j), shfl_d(x, j));
        }
        day_sum = shfl_d(seg, cnt - 1);
    }

    // trade hash + optional event buffer
    const unsigned n_events = acc->n_events;
    const unsigned long long h = active ? event_hash(n_events + lane, hw) : 0ull;
    const unsigned hlo = __reduce_xor_sync(FULL, (unsigned)h);
    const unsigned hhi = __reduce_xor_sync(FULL, (unsigned)(h >> 32));
    uint32_t* ev_out = acc->ev_out;
    if (ev_out && active) {
        const long long idx = (long long)n_events + lane;
        if (idx < ev_cap) ev_out[idx] = w;
    }
    __syncwarp();
    if (lane == 0) {
        acc->n_win = n_win; acc->n_loss = n_loss;
        acc->tot_profit = tot_profit; acc->tot_loss = tot_loss;
        acc->largest_p = largest_p; acc->largest_l = largest_l;
        acc->sum_dur = sum_dur;
        acc->equity = equity_out; acc->peak = peak_out; acc->maxdd = maxdd;
        acc->pivot = da.pivot; acc->s1 = da.s1; acc->s2 = da.s2; acc->n_days = da.n_days; acc->pivot_set = da.pivot_set;
        acc->npivot = da.npivot; acc->ns1 = da.ns1; acc->ns2 = da.ns2; acc->n_neg = da.n_neg;
        acc->day_sum = day_sum; acc->day_cur = last_day; acc->day_valid = 1;
        acc->first_done = first_done; acc->first_day = first_id; acc->first_sum = first_sum;
        acc->hash ^= ((unsigned long long)hhi << 32) | hlo;
        acc->n_events = n_events + cnt;
    }
    __syncwarp();
}

// Run n <= 32 priced records of a merged list through batch_records, pairing durations on the list index (2k, 2k+1)
// (calculate_metrics :166-178) whatever their symbols; takes and returns the bar of the list's previous record.
__device__ __forceinline__ unsigned merged_records(WarpAcc* __restrict__ acc, int n, bool active, unsigned wd, unsigned hw,
                                                   double pnl, unsigned bar_carry, const b200bt_sweep_config& cfg) {
    const int lane = threadIdx.x & 31;
    const unsigned x = wd & B200BT_EVENT_BAR_MASK;
    unsigned x_prev = __shfl_up_sync(FULL, x, 1);
    if (lane == 0) x_prev = bar_carry;
    const unsigned g = acc->n_events + (unsigned)lane;
    const int dur = (active && (g & 1u)) ? (int)(x - x_prev) : 0;
    const unsigned carry = __shfl_sync(FULL, x, n - 1);
    batch_records(acc, n, active, wd, hw, pnl, dur, cfg.minute0, cfg.bar_minutes, 0);
    return carry;
}

// Consume `cnt` events in time order (lane j holds event j: word w, price pf); an exit record is
// priced against the entry record that precedes it -- lane j-1, or for lane 0 the last event of
// the previous batch (w_carry, p_carry).
static __device__ __noinline__ void batch_core(WarpAcc* __restrict__ acc, int cnt, unsigned w, float pf, unsigned w_carry,
                                        float p_carry, long long minute0, int bar_minutes, int64_t ev_cap) {
    const int lane = threadIdx.x & 31;
#ifdef B200BT_SW_NOBATCH   // timing experiment only: skip the batch arithmetic
    if (lane == 0) acc->n_events += cnt;
    __syncwarp();
    return;
#endif
    const bool active = lane < cnt;
    float p_prev = __shfl_up_sync(FULL, pf, 1);
    unsigned w_prev = __shfl_up_sync(FULL, w, 1);
    if (lane == 0) { p_prev = p_carry; w_prev = w_carry; }

    int dur;
    const double pnl = record_pnl(active, w, pf, w_prev, p_prev, acc->size, acc->fee1, acc->fee2, dur);
    batch_records(acc, cnt, active, w, w, pnl, dur, minute0, bar_minutes, ev_cap);
}

// Fused kernel: consume 32 (or the last few) queued events; batches there start on an entry record.
__device__ __forceinline__ void process_batch(WarpShared* __restrict__ ws, unsigned qtail, int cnt,
                                              long long minute0, int bar_minutes, int64_t ev_cap) {
    const uint2 evt = ws->evq[(qtail + (threadIdx.x & 31)) & (SW_EVQ - 1)];
    batch_core(&ws->acc, cnt, evt.x, __uint_as_float(evt.y), 0u, 0.f, minute0, bar_minutes, ev_cap);
}

// Metrics -> calculate_metrics' scalars and _calculate_strategy_score (strategy_evaluation.py:97-228,:579-633).
__device__ __forceinline__ void finalize_lane(const WarpAcc& a, const b200bt_sweep_config& cfg, b200bt_lane_stats& o) {
    DayAcc da{a.pivot, a.s1, a.s2, a.n_days, a.pivot_set, a.npivot, a.ns1, a.ns2, a.n_neg};
    if (a.day_valid) day_complete(da, a.day_sum);
    const double n_rec = (double)a.n_events;
    o.n_records = n_rec;
    o.n_wins = (double)a.n_win;
    o.n_losses = (double)a.n_loss;
    o.total_profit = a.tot_profit;
    o.total_loss = a.tot_loss;
    o.net_profit = a.tot_profit + a.tot_loss;
    o.max_drawdown = a.maxdd;
    o.n_days = (double)da.n_days;
    o.largest_profit = a.largest_p;
    o.largest_loss = a.largest_l;
    o.sum_duration_bars = (double)a.sum_dur;
    o.trade_hash = a.hash;
    double sharpe = 0.0, win_rate = 0.0, pf = 0.0;
    if (a.n_events >= 2) {
        win_rate = (double)a.n_win / n_rec;
        pf = (a.tot_loss != 0.0) ? fabs(a.tot_profit / a.tot_loss) : INFINITY;
        if (da.n_days > 1) {
            const double nd = (double)da.n_days;
            const double mean_y = da.s1 / nd;
            double var = da.s2 / nd - mean_y * mean_y;
            if (var < 0.0) var = 0.0;
            const double sd = sqrt(var);
            const double mean = da.pivot + mean_y;
            sharpe = sd > 0.0 ? (mean / sd) * sqrt(252.0) : 0.0;
        }
    }
    o.sharpe_ratio = sharpe;
    o.win_rate = win_rate;
    o.profit_factor = pf;
    // calculate_advanced_metrics (:250-263, :307-312): only a lane with >= 2 records has daily buckets
    double mean_daily = 0.0, downside = 0.0, sortino = 0.0;
    if (a.n_events >= 2 && da.n_days > 0) {
        mean_daily = da.pivot + da.s1 / (double)da.n_days;
        if (da.n_neg > 0) {
            const double nn = (double)da.n_neg, my = da.ns1 / nn;
            double var = da.ns2 / nn - my * my;
            downside = sqrt(var < 0.0 ? 0.0 : var);
        }
        sortino = downside > 0.0 ? (mean_daily / downside) * sqrt(252.0) : INFINITY;
    }
    o.sortino_ratio = sortino;
    o.n_negative_days = (a.n_events >= 2) ? (double)da.n_neg : 0.0;
    o.downside_deviation = downside;
    o.mean_daily_pnl = mean_daily;
    // every scalar key of the metrics dict can be the primary metric (:589-590)
    const double ret_pct = (o.net_profit / cfg.initial_capital) * 100.0;
    const double avg_p = a.n_win ? a.tot_profit / (double)a.n_win : 0.0, avg_l = a.n_loss ? a.tot_loss / (double)a.n_loss : 0.0;
    // calculate_advanced_metrics :302-310 (total_trades > 0)
    const double expectancy = a.n_events ? win_rate * avg_p - (1.0 - win_rate) * fabs(avg_l) : 0.0;
    double primary;
    switch (cfg.primary) {
        case B200BT_PRIMARY_RETURN_PCT: primary = ret_pct; break;
        case B200BT_PRIMARY_PROFIT_FACTOR: primary = pf; break;
        case B200BT_PRIMARY_WIN_RATE: primary = win_rate; break;
        case B200BT_PRIMARY_NET_PROFIT: primary = o.net_profit; break;
        case B200BT_PRIMARY_TOTAL_TRADES: primary = n_rec; break;
        case B200BT_PRIMARY_MAX_DRAWDOWN: primary = a.maxdd; break;
        case B200BT_PRIMARY_TOTAL_PROFIT: primary = a.tot_profit; break;
        case B200BT_PRIMARY_TOTAL_LOSS: primary = a.tot_loss; break;
        case B200BT_PRIMARY_LARGEST_PROFIT: primary = a.largest_p; break;
        case B200BT_PRIMARY_LARGEST_LOSS: primary = a.largest_l; break;
        case B200BT_PRIMARY_AVERAGE_PROFIT: primary = avg_p; break;
        case B200BT_PRIMARY_AVERAGE_LOSS: primary = avg_l; break;
        case B200BT_PRIMARY_SORTINO: primary = sortino; break;
        case B200BT_PRIMARY_EXPECTANCY: primary = expectancy; break;
        case B200BT_PRIMARY_CALMAR: primary = a.maxdd > 0.0 ? (ret_pct / 100.0) / a.maxdd : INFINITY; break;          // :243-249
        case B200BT_PRIMARY_PROFIT_PER_DAY: primary = mean_daily; break;
        case B200BT_PRIMARY_RECOVERY_FACTOR: primary = a.maxdd > 0.0 ? o.net_profit / (a.maxdd * 10000.0) : INFINITY; break;   // :296-300
        case B200BT_PRIMARY_ZERO: primary = 0.0; break;
        default: primary = sharpe; break;
    }
    double score = primary;
    if (cfg.secondary_mask & B200BT_SEC_MAX_DRAWDOWN) score *= (1.0 - a.maxdd);
    if (cfg.secondary_mask & B200BT_SEC_WIN_RATE) score *= (1.0 + win_rate);
    if (cfg.secondary_mask & B200BT_SEC_PROFIT_FACTOR) score *= (pf / 2.0);
    if (cfg.secondary_mask & B200BT_SEC_EXPECTANCY) score *= (1.0 + fmin(expectancy / 100.0, 1.0));
    o.score = score;
}

// Initial metrics state of a lane.
__device__ __forceinline__ void init_acc(WarpAcc& a, const b200bt_individual& iv, const b200bt_sweep_config& cfg, uint32_t* ev_out) {
    const double initial_capital = cfg.initial_capital;
    a.gap_bar = cfg.gap_bar > 0 ? (unsigned)cfg.gap_bar : 0xffffffffu;
    a.gap_minutes = (unsigned)cfg.gap_minutes;
    a.tp = iv.take_profit; a.sl = iv.stop_loss; a.size = iv.position_size;
    a.fee1 = __dmul_rn(a.size, 0.001); a.fee2 = __dmul_rn(a.size, 0.002);
    a.equity = initial_capital; a.peak = initial_capital; a.maxdd = 0.0;
    a.tot_profit = a.tot_loss = a.largest_p = a.largest_l = 0.0;
    a.day_sum = a.pivot = a.s1 = a.s2 = 0.0;
    a.day_cur = 0; a.sum_dur = 0; a.hash = 0ull;
    a.ev_out = ev_out;
    a.n_win = a.n_loss = a.n_days = a.n_events = 0;
    a.day_valid = a.pivot_set = 0;
    a.hold_first = a.first_done = a.first_day = 0;
    a.first_sum = 0.0;
    a.npivot = a.ns1 = a.ns2 = 0.0;
    a.n_neg = 0;
}

__device__ __forceinline__ void init_scan_const(ScanConst& c, const b200bt_individual& iv) {
    c.os_f = iv.rsi_lo;
    c.ob_f = iv.rsi_hi;
    const double mg = (double)SW_MARGIN, tp = iv.take_profit, sl = iv.stop_loss;
    c.hiL_c = (float)((1.0 + tp) * (1.0 - mg));
    c.hiL_d = (float)((1.0 + tp) * (1.0 + mg));
    c.loL_c = (float)((1.0 - sl) * (1.0 + mg));
    c.loL_d = (float)((1.0 - sl) * (1.0 - mg));
    c.loS_c = (float)((1.0 - tp) * (1.0 + mg));
    c.loS_d = (float)((1.0 - tp) * (1.0 - mg));
    c.hiS_c = (float)((1.0 + sl) * (1.0 - mg));
    c.hiS_d = (float)((1.0 + sl) * (1.0 + mg));
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_) : "memory"); }

// ---- mbarrier + bulk async copies (sm_90+ PTX; the tile ring of the thread-per-lane scan) ------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_inval(unsigned long long* bar) {
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait (there is no unbounded one): false when the phase has not completed `cycles` SM clocks after the first failed poll (the caller gives the
// work up and has it redone by the exact fallback instead of spinning for ever on a copy that does not arrive)
__device__ __forceinline__ bool mbar_wait_bounded(unsigned long long* bar, unsigned parity, long long cycles) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > cycles) return false;
    return true;
}
// global -> shared bulk copy (TMA engine, 16-byte aligned, size a multiple of 16), completion counted on `bar`
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Machine state of one lane (warp-uniform registers).
struct Machine {
    int pos;                                   // 0 flat, +1 long, -1 short
    float e;                                   // entry price
    float rlo, rhi, plo, phi;                  // event thresholds of the current state (screening bounds)
    int entry_bar;                             // bar of the open position's entry (chunk-boundary check)
    unsigned qhead;                            // events pushed so far (queue head)
};

__device__ __forceinline__ bool fires(const Machine& m, float p, float r) {
    return (r < m.rlo) | (r > m.rhi) | (p <= m.plo) | (p >= m.phi);
}

// Flat: only an entry signal (RSI below the oversold threshold os or above the overbought one ob) fires.
__device__ __forceinline__ void set_flat(Machine& m, float os, float ob) {
    m.pos = 0;
    m.rlo = os; m.rhi = ob;
    m.plo = -INFINITY; m.phi = INFINITY;
}

// The machine at the start of a scan: flat, nothing queued.
__device__ __forceinline__ Machine flat_machine(const b200bt_individual& iv) {
    Machine m;
    set_flat(m, iv.rsi_lo, iv.rsi_hi);
    m.e = 0.f; m.entry_bar = 0;
    m.qhead = 0;
    return m;
}

// Open a position (strategy_evaluation.py:784-813): long (`lng`) or short, entered at price e on `bar`; the exit
// thresholds are an RSI reversal and the fp32 candidate bounds of take-profit / stop-loss around e.
__device__ __forceinline__ void set_open(Machine& m, const ScanConst& c, bool lng, float e, int bar) {
    m.e = e;
    m.entry_bar = bar;
    m.pos = lng ? 1 : -1;
    m.rlo = lng ? -INFINITY : c.os_f;
    m.rhi = lng ? c.ob_f : INFINITY;
    m.phi = e * (lng ? c.hiL_c : c.hiS_c);
    m.plo = e * (lng ? c.loL_c : c.loS_c);
}

// Advance the machine through every event of one 32-bar window (lane l holds bar t0+l).
// `emit` = false runs the machine without recording events (warm-up bars of a time chunk).
// `win` points at the window's 32 prices in the shared-memory ring (RSI values SW_GROUP floats further):
// the event bar's price / RSI are re-read from there with a warp-uniform address.
__device__ __forceinline__ void scan_window(const float p, const float r, const float* __restrict__ win, const int t0,
                                            WarpShared* __restrict__ ws, const ScanConst& c, Machine& m,
                                            const bool emit = true) {
    unsigned live = FULL;  // bars of the window not yet consumed
    while (true) {
        const unsigned hit = __ballot_sync(FULL, fires(m, p, r)) & live;
        if (hit == 0) break;
        const int kk = __ffs(hit) - 1;
        const float pk = win[kk];
        const float rk = win[SW_GROUP + kk];
        live = 0xfffffffeu << kk;
        const unsigned bar = (unsigned)(t0 + kk);
        unsigned word;
        bool ev = true;
        if (m.pos == 0) {
            // entry: long has priority over short
            const bool lng = rk < c.os_f;
            set_open(m, c, lng, pk, (int)bar);
            word = lng ? bar : (bar | B200BT_EVENT_SELL);
        } else {
            // exit candidate (:815-847); an RSI reversal is always definite, a price trigger inside the
            // fp32 screening band is decided with the reference's float64 expression
            if (!((rk < m.rlo) || (rk > m.rhi))) {
                const bool lng = m.pos > 0;
                const float hd = m.e * (lng ? c.hiL_d : c.hiS_d), ld = m.e * (lng ? c.loL_d : c.loS_d);
                if (!((pk >= hd) || (pk <= ld))) {
                    const double ed = (double)m.e, pd = (double)pk;
                    const double q = lng ? __ddiv_rn(__dsub_rn(pd, ed), ed) : __ddiv_rn(__dsub_rn(ed, pd), ed);
                    ev = (q >= ws->acc.tp) || (q <= -ws->acc.sl);
                }
            }
            if (ev) {
                word = bar | B200BT_EVENT_EXIT | (m.pos > 0 ? B200BT_EVENT_SELL : 0u);
                set_flat(m, c.os_f, c.ob_f);
            }
        }
        if (ev) {
            // every lane stores the same word to the same slot (one wavefront); while not recording, the
            // head does not advance and the slot is simply overwritten by the next event
            ws->evq[m.qhead & (SW_EVQ - 1)] = make_uint2(word, __float_as_uint(pk));
            m.qhead += emit ? 1u : 0u;
        }
    }
}

// The per-warp cp.async ring of the bar scan: streams groups [g_begin, g_end) of SW_GROUP bars of one (price, RSI) row
// pair through WarpShared::ring, SW_STAGES - 1 groups ahead of the scan, with no registers tied up by prefetch.  Full
// groups are copied 16 B per thread (128 bars per instruction) when the rows start on 16-byte boundaries (VEC16), 4 B per
// thread otherwise; the ragged last group of the series is loaded with guards and padded with NaN (NaN never fires an
// event).  land() issues one more group and returns the oldest one in flight once it has landed; release() hands its
// stage back to be refilled.  Only the producer's running position is kept (the rows themselves are reached through it),
// which keeps the state that lives across the scan loop small.
template <bool VEC16>
struct GroupRing {
    static constexpr int G = SW_GROUP;
    float* sp;                           // the warp's ring
    int n, n_full, g_end;                // bars, groups copied without bounds checks, end of the range
    int issued;                          // producer: next group to issue, its ring slot and sources (this lane's part)
    float* idst;
    const float* ip; const float* ir;
    int cstage;                          // consumer: stage of the next group to land, this lane's first bar of it
    const float* cur;

    // pr, rr: the price and RSI rows from bar 0
    __device__ __forceinline__ GroupRing(WarpShared* ws, const float* pr, const float* rr, int n_, int g_begin, int g_end_)
        : sp(&ws->ring[0][0][0]), n(n_), n_full(n_ / G), g_end(g_end_), issued(g_begin) {
        const int lane = threadIdx.x & 31, off = VEC16 ? lane * 4 : lane;
        idst = sp + (g_begin % SW_STAGES) * (2 * G) + off;
        ip = pr + (int64_t)g_begin * G + off;
        ir = rr + (int64_t)g_begin * G + off;
#pragma unroll
        for (int g = 0; g < SW_STAGES - 1; ++g) issue();
        cstage = g_begin % SW_STAGES;
        cur = sp + cstage * (2 * G) + lane;
    }

    __device__ __forceinline__ void issue() {
        if (issued < g_end) {
            if (issued < n_full) {
                if (VEC16) {
#pragma unroll
                    for (int i = 0; i < G / 128; ++i) {
                        cp_async16(idst + i * 128, ip + i * 128);
                        cp_async16(idst + G + i * 128, ir + i * 128);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < G / 32; ++i) {
                        cp_async4(idst + i * 32, ip + i * 32);
                        cp_async4(idst + G + i * 32, ir + i * 32);
                    }
                }
            } else {
                const float qnan = __int_as_float(0x7fc00000);
                const int lane = threadIdx.x & 31, off = VEC16 ? lane * 4 : lane;
                float* dst = sp + (issued % SW_STAGES) * (2 * G);
                const float* gp = ip - off; const float* gr = ir - off;   // the group's first bar, issued * G
                for (int i = lane; i < G; i += 32) {
                    const int t = issued * G + i;
                    dst[i] = t < n ? __ldg(gp + i) : qnan;
                    dst[G + i] = t < n ? __ldg(gr + i) : qnan;
                }
            }
        }
        cp_async_commit();  // always commit (possibly empty) so the group accounting stays uniform
        ++issued;
        ip += G; ir += G;
        idst = (issued % SW_STAGES == 0) ? idst - (SW_STAGES - 1) * (2 * G) : idst + 2 * G;
    }

    __device__ __forceinline__ const float* land() {
        issue();
        cp_async_wait<SW_STAGES - 1>();
        __syncwarp();
        return cur;
    }

    __device__ __forceinline__ void release() {
        __syncwarp();                         // the stage is refilled by the next land()
        if (++cstage == SW_STAGES) { cstage = 0; cur -= (SW_STAGES - 1) * (2 * G); } else cur += 2 * G;
    }
};

// Event sinks: sink(at, cnt) consumes the `cnt` queued events from queue position `at` on (lane j: event at + j).

// Hand every full batch of 32 queued events to `sink`.
template <class Sink>
__device__ __forceinline__ void drain_full(const Machine& m, unsigned& qtail, Sink& sink) {
    while (m.qhead - qtail >= 32) {
        __syncwarp();
        sink(qtail, 32);
        qtail += 32;
    }
}

// Scan one landed group, bars [t0, t0 + SW_GROUP) (`w`: this lane's first bar of it in the ring), two 32-bar windows
// per step with both ballots issued before either is needed; full batches of queued events go to `sink`.
template <class Sink>
__device__ __forceinline__ void scan_group(const float* w, int t0, WarpShared* ws, const ScanConst& c,
                                           Machine& m, unsigned& qtail, const bool emit, Sink& sink) {
    const int lane = threadIdx.x & 31;
#pragma unroll 1
    for (int v = 0; v < SW_GROUP / 64; ++v, w += 64, t0 += 64) {
        const float p0 = w[0], r0 = w[SW_GROUP];
        const float p1 = w[32], r1 = w[SW_GROUP + 32];
        const unsigned h0 = __ballot_sync(FULL, fires(m, p0, r0));
        const unsigned h1 = __ballot_sync(FULL, fires(m, p1, r1));
        if (h0 | h1) {
            if (h0) scan_window(p0, r0, w - lane, t0, ws, c, m, emit);
            scan_window(p1, r1, w - lane + 32, t0 + 32, ws, c, m, emit);
            drain_full(m, qtail, sink);
        }
    }
}

// End of a scan: wait for the ring's last (empty) copy groups; with `close`, force-close an open position at the last
// bar N - 1 (strategy_evaluation.py:849-876) by queueing its exit event; then hand every queued event to `sink`, the
// last batch partial.
template <class Sink>
__device__ __forceinline__ void finish_scan(WarpShared* ws, Machine& m, unsigned& qtail, const float* pr,
                                            int64_t N, const bool close, Sink& sink) {
    cp_async_wait<0>();
    if (close && m.pos != 0) {
        const float pl = __ldg(pr + (N - 1));
        const unsigned word = (unsigned)(N - 1) | B200BT_EVENT_EXIT | (m.pos > 0 ? B200BT_EVENT_SELL : 0u);
        if ((threadIdx.x & 31) == 0) ws->evq[m.qhead & (SW_EVQ - 1)] = make_uint2(word, __float_as_uint(pl));
        ++m.qhead;
    }
    __syncwarp();
    while (m.qhead != qtail) {
        const int cnt = (int)min(32u, m.qhead - qtail);
        sink(qtail, cnt);
        qtail += cnt;
    }
}

}  // namespace b200bt
