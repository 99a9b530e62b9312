// Book-level metrics of a multi-symbol strategy (sm_90a): calculate_metrics / calculate_advanced_metrics /
// _calculate_strategy_score on ONE trade list that holds an individual's records on every symbol, the way
// StrategyEvaluationSystem.evaluate_strategy (services/strategy_evaluation.py:528-577) passes a mixed list to
// calculate_metrics (:32-228), which sorts it by timestamp (:67) and walks one equity curve and one set of daily buckets.
//
// Merged order.  sorted(..., key=timestamp) is stable and every symbol shares one clock, so the book is ordered by
// (bar, symbol index, record index within the lane).  One symbol holds at most one record per bar, except on the last bar,
// where an entry is followed by its force-close (:849-876).
//
// Scheme: one warp per individual streams through the bar axis in windows [b0, B).  b0 is the bar of the earliest record
// not yet consumed (empty stretches are skipped); B <= b0 + BK_BARS, and B is at most the bar of the K-th staged record of
// every symbol (K = BK_CAP / S), so that a window holds at most BK_CAP records and every record of it is staged.  Inside a
// window each bar gets a bitmask of the symbols with a record on it (and one extra mask for the last bar's second records);
// an exclusive scan of the per-bar popcounts gives the rank of a bar's first record, and a record's rank is that plus
// popc(mask & symbols below it): O(1) per record, deterministic.  Records are priced as trade_pnl_kernel prices them
// (record_pnl), scattered to their rank in shared memory, and walked 32 at a time through batch_records, the lane sweep's
// own metrics step (equity, peak, drawdown, days, counts, hash); finalize_lane gives the scalars and the score.
#include <math.h>
#include "sweep_dev.cuh"

namespace b200bt {

constexpr int BK_WARPS = 2;            // individuals per CTA
constexpr int BK_CAP = 512;            // records per window (staged and merged)
constexpr int BK_BARS = 1024;          // bars per window (per-bar symbol masks)
constexpr int BK_MAX_SYMBOLS = 64;     // one 64-bit symbol mask per bar
constexpr unsigned BK_NO_RECORD = 0x3fffffffu;   // staged word past a lane's last record: its bar is beyond any N < 2^30
constexpr unsigned BK_SYMBOL_TAG = 0x9E3779B1u;  // trade_hash word of a book record: word ^ (symbol * BK_SYMBOL_TAG)

struct BookWarp {
    unsigned long long mask[BK_BARS];    // symbols with a record on bar b0 + b
    unsigned short base[BK_BARS];        // rank of the first record on bar b0 + b
    uint32_t stage[BK_CAP];              // [S][K] the next K words of every symbol
    uint32_t word[BK_CAP];               // merged records of the window: event word, symbol, pnl
    unsigned char sym[BK_CAP];
    double pnl[BK_CAP];
    int64_t cur[BK_MAX_SYMBOLS];         // records of each symbol consumed so far
    int64_t n_rec[BK_MAX_SYMBOLS];
    int take[BK_MAX_SYMBOLS];            // records of each symbol in the current window
    WarpAcc acc;
};

__global__ void __launch_bounds__(BK_WARPS * 32)
book_kernel(const float* __restrict__ price, int64_t ld_price, int S, int64_t N, const b200bt_individual* __restrict__ indiv,
            int pop, const b200bt_sweep_config cfg, const b200bt_lane_stats* __restrict__ lane_stats,
            const uint32_t* __restrict__ events, int64_t event_cap, b200bt_lane_stats* __restrict__ book,
            double* __restrict__ fitness) {
    __shared__ BookWarp shared[BK_WARPS];
    const int lane = threadIdx.x & 31;
    const int ind = blockIdx.x * BK_WARPS + (threadIdx.x >> 5);
    if (ind >= pop) return;
    BookWarp& w = shared[threadIdx.x >> 5];
    WarpAcc* acc = &w.acc;

    bool lost = false;
    for (int s = lane; s < S; s += 32) {
        const int64_t n = (int64_t)lane_stats[(int64_t)ind * S + s].n_records;
        w.cur[s] = 0;
        w.n_rec[s] = n;
        lost |= n > event_cap;
    }
    if (__any_sync(FULL, lost)) {       // the event buffer did not hold every record of some lane: no book
        if (lane == 0) {
            book[ind] = lost_lane_stats();
            if (fitness) fitness[ind] = NAN;
        }
        return;
    }
    const b200bt_individual iv = indiv[ind];
    if (lane == 0) init_acc(*acc, iv, cfg, nullptr);
    __syncwarp();
    const double size = acc->size, fee1 = acc->fee1, fee2 = acc->fee2;
    const int K = BK_CAP / S;
    const int staged = K * S;
    const unsigned last_bar = (unsigned)(N - 1);
    const uint32_t* ev_ind = events + (int64_t)ind * S * event_cap;
    unsigned bar_carry = 0;             // bar of the book's previous record (duration of merged pairs)

    while (true) {
        // stage the next K words of every symbol
        for (int f = lane; f < staged; f += 32) {
            const int s = f / K, j = f - s * K;
            const int64_t idx = w.cur[s] + j;
            w.stage[f] = idx < w.n_rec[s] ? __ldg(ev_ind + (int64_t)s * event_cap + idx) : BK_NO_RECORD;
            if (j == 0) w.take[s] = 0;
        }
        __syncwarp();
        // window [b0, B)
        unsigned b0 = BK_NO_RECORD, B = BK_NO_RECORD;
        for (int s = lane; s < S; s += 32) {
            b0 = min(b0, w.stage[s * K] & B200BT_EVENT_BAR_MASK);
            B = min(B, w.stage[s * K + K - 1] & B200BT_EVENT_BAR_MASK);   // K >= 3 records never share one bar: B > b0
        }
        b0 = __reduce_min_sync(FULL, b0);
        if (b0 >= (unsigned)N) break;
        B = min(__reduce_min_sync(FULL, B), b0 + (unsigned)BK_BARS);
        const int span = (int)(B - b0);
        for (int b = lane; b < span; b += 32) w.mask[b] = 0ull;
        __syncwarp();
        // symbol masks: first records of a (bar, symbol) in mask[], the last bar's second records in `second`
        unsigned long long second = 0ull;
        for (int f = lane; f < staged; f += 32) {
            const unsigned x = w.stage[f] & B200BT_EVENT_BAR_MASK;
            if (x >= B) continue;
            const int s = f / K, j = f - s * K;
            const bool dup = j > 0 && (w.stage[f - 1] & B200BT_EVENT_BAR_MASK) == x;
            if (dup) second |= 1ull << s;
            else atomicOr(&w.mask[x - b0], 1ull << s);
            if (j == K - 1 || (w.stage[f + 1] & B200BT_EVENT_BAR_MASK) >= B) w.take[s] = j + 1;
        }
        second = __reduce_or_sync(FULL, (unsigned)second) | ((unsigned long long)__reduce_or_sync(FULL, (unsigned)(second >> 32)) << 32);
        __syncwarp();
        // rank of each bar's first record: exclusive scan of the per-bar record counts, 32 bars per lane
        const int per = (span + 31) >> 5, lo = lane * per, hi = min(span, lo + per);
        const bool last_in = last_bar >= b0 && last_bar < B;
        int cnt = 0;
        for (int b = lo; b < hi; ++b) cnt += __popcll(w.mask[b]);
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int up = __shfl_up_sync(FULL, incl, d);
            if (lane >= d) incl += up;
        }
        const int T = __shfl_sync(FULL, incl, 31) + (last_in ? __popcll(second) : 0);
        int run = incl - cnt;
        for (int b = lo; b < hi; ++b) {
            w.base[b] = (unsigned short)run;
            run += __popcll(w.mask[b]);
        }
        __syncwarp();
        // price every record of the window and put it at its rank
        for (int f = lane; f < staged; f += 32) {
            const unsigned wd = w.stage[f];
            const unsigned x = wd & B200BT_EVENT_BAR_MASK;
            if (x >= B) continue;
            const int s = f / K, j = f - s * K;
            const unsigned long long below = (1ull << s) - 1ull;
            const bool dup = j > 0 && (w.stage[f - 1] & B200BT_EVENT_BAR_MASK) == x;
            int rank = w.base[x - b0] + __popcll(w.mask[x - b0] & below);
            if (x == last_bar) rank += __popcll(second & below) + (dup ? 1 : 0);   // a force-close follows its entry
            const float* row = price + (int64_t)s * ld_price;
            double pnl = -fee1;
            if (wd & B200BT_EVENT_EXIT) {
                // the entry record precedes the exit in the same lane: staged, or the symbol's last record before the window
                const unsigned we = j > 0 ? w.stage[f - 1] : __ldg(ev_ind + (int64_t)s * event_cap + w.cur[s] - 1);
                int dur;
                pnl = record_pnl(true, wd, __ldg(row + x), we, __ldg(row + (we & B200BT_EVENT_BAR_MASK)), size, fee1, fee2, dur);
            }
            w.word[rank] = wd;
            w.sym[rank] = (unsigned char)s;
            w.pnl[rank] = pnl;
        }
        __syncwarp();
        for (int s = lane; s < S; s += 32) w.cur[s] += w.take[s];
        // walk the merged records through the lane sweep's metrics step
        for (int r0 = 0; r0 < T; r0 += 32) {
            const int r = r0 + lane, n = min(32, T - r0);
            const bool active = r < T;
            const unsigned wd = active ? w.word[r] : 0u;
            const unsigned s = active ? w.sym[r] : 0u;
            const double pnl = active ? w.pnl[r] : 0.0;
            bar_carry = merged_records(acc, n, active, wd, wd ^ (s * BK_SYMBOL_TAG), pnl, bar_carry, cfg);
        }
        __syncwarp();
    }
    if (lane == 0) {
        b200bt_lane_stats o;
        finalize_lane(*acc, cfg, o);
        book[ind] = o;
        if (fitness) fitness[ind] = o.score;
    }
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_book_metrics(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv,
                                   int pop, const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats,
                                   const uint32_t* events, int64_t event_cap, b200bt_lane_stats* book_stats,
                                   double* fitness_or_null, b200bt_stream_t stream) {
    B200BT_REQUIRE(cfg && book_stats, B200BT_EINVAL, "book_metrics: null pointer");
    int rc = check_record_args("book_metrics", price, ld_price, S, N, indiv, pop, cfg, lane_stats, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE(S <= BK_MAX_SYMBOLS, B200BT_ELIMIT, "book_metrics: at most %d symbols (S = %d)", BK_MAX_SYMBOLS, S);
    B200BT_REQUIRE((int64_t)S * (N + 1) < (1ll << 32), B200BT_ELIMIT, "book_metrics: S * (N + 1) records must stay below 2^32");
    rc = check_device();
    if (rc) return rc;
    book_kernel<<<(unsigned)((pop + BK_WARPS - 1) / BK_WARPS), BK_WARPS * 32, 0, (cudaStream_t)stream>>>(
        price, ld_price, S, N, indiv, pop, *cfg, lane_stats, events, event_cap, book_stats, fitness_or_null);
    B200BT_LAUNCH_CHECK("book_metrics");
    return B200BT_OK;
}
