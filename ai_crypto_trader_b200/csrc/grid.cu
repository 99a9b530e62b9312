// Grid trading backtest (sm_90a): services/grid_trading_strategy.py's simulation loop over a market's bars for a whole
// population at once.  Contract and the rule restated: include/b200bt.h (b200bt_grid_sweep); design: DESIGN.md section 3.13.
//
// grid_kernel  one warp per (individual, symbol) lane; a CTA holds GR_WARPS individuals of ONE symbol, which share the
//              symbol's price tiles: GR_TILE closes (plus the previous one) staged into shared memory by cp.async, two
//              stages, the next tile in flight while the current one is scanned.  The grid only changes at check ticks
//              (rebalance / adjustment), so the ticks between two checks are independent given last = price[k - 1]: a pass
//              takes up to 32 ticks, one per thread, and ends at the next check tick or the tile's end.  Each thread
//              estimates the index of the crossed level range in fp32 (a product for arithmetic grids, a log2 for
//              geometric ones), corrects it by exact float64 compares against the warp's level table (rebuilt in shared
//              memory at each regeneration with the reference's expressions), and sums its crossings' profits.  The
//              checks are warp-uniform scalar steps after the pass that ends on their tick.  Counts are integers (exact);
//              profits are summed per thread in tick order and then over the warp.
//              DAY: the CTA runs every symbol of its individuals in turn and each warp adds its per-day profits into its
//              individual's row (no atomics, fixed order).
#include <limits.h>
#include <math.h>
#include "common.cuh"

namespace b200bt {
namespace {

constexpr int GR_WARPS = 16;
constexpr int GR_TILE = 2048;                        // ticks per staged price tile
constexpr int GR_LEVELS = B200BT_GRID_MAX_GRIDS + 1;

struct GridArgs {
    const float* price;
    int64_t ld_price, N, start_bar, minute0, ld_labels, D, first_day;
    int S, pop, bar_minutes, use_rules;
    const b200bt_grid_individual* indiv;
    const double* qty;
    const double* bounds;
    const uint8_t* labels;
    b200bt_grid_stats* stats;
    double* day;
    b200bt_grid_regime_rule rules[B200BT_GRID_REGIME_RULES];
};

__device__ __forceinline__ void cp4(float* dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_) : "memory"); }

// The active grid of a warp (uniform).  Levels live in the warp's shared table L[0 .. n].
struct Grid {
    double lower, upper;
    int n, type;
    float base, scale;           // fp32 index estimate: (x - base) * scale, or log2(x * base) * scale (geometric)
};

// _generate_grid_levels (:347-385) into L, with the reference's float64 expressions
__device__ void build_levels(double* L, Grid& g) {
    const int lane = threadIdx.x & 31, n = g.n;
    if (g.type == B200BT_GRID_ARITHMETIC) {
        const double step = __ddiv_rn(__dsub_rn(g.upper, g.lower), (double)n);
        for (int i = lane; i <= n; i += 32) L[i] = __dadd_rn(g.lower, __dmul_rn((double)i, step));
        g.base = (float)g.lower;
        g.scale = (float)(1.0 / step);
    } else {
        const double ratio = pow(__ddiv_rn(g.upper, g.lower), __ddiv_rn(1.0, (double)n));
        for (int i = lane; i <= n; i += 32) L[i] = __dmul_rn(g.lower, pow(ratio, (double)i));
        g.base = (float)(1.0 / g.lower);
        g.scale = (float)(1.0 / log2(ratio));
    }
    __syncwarp();
}

// first guess of the smallest i with L[i] >= x, clamped to [0, n + 1] (NaN and inf estimates included)
__device__ __forceinline__ int estimate(const Grid& g, double x) {
    const float e = g.type == B200BT_GRID_ARITHMETIC ? ((float)x - g.base) * g.scale : __log2f((float)x * g.base) * g.scale;
    if (!(e > 0.f)) return 0;
    if (!(e < (float)g.n)) return g.n + 1;
    return (int)ceilf(e);
}

// smallest i in [0, n + 1] with L[i] >= x (STRICT: L[i] > x), from any start e; exact for non-decreasing levels
template <bool STRICT>
__device__ __forceinline__ int level_bound(const double* L, int n, int e, double x) {
    if (STRICT) {
        while (e > 0 && L[e - 1] > x) --e;
        while (e <= n && L[e] <= x) ++e;
    } else {
        while (e > 0 && L[e - 1] >= x) --e;
        while (e <= n && L[e] < x) ++e;
    }
    return e;
}

__device__ __forceinline__ bool near(double x, double l) { return fabs(__dsub_rn(x, l)) <= fabs(l) * 0x1p-50; }

// x within 4 ulps of one of the levels a bound on x compared it with last: L[e - 1] and L[e]
__device__ __forceinline__ bool near_bound(const double* L, int n, int e, double x) {
    return (e > 0 && near(x, L[e - 1])) || (e <= n && near(x, L[e]));
}

// One lane's running totals: counts, profit and cash per thread (the thread's ticks), inventory and day state warp-uniform.
struct LaneAcc {
    unsigned long long n_up, n_down, n_prof, n_tie;
    double profit, cash;
    long long net, net_max, net_min;             // inventory in units of qty
    int64_t day_cur;
    double day_val;
};

// One pass (_process_grid_simulation): ticks of bars b .. b + n - 1, one per thread, n <= 32; px[j] is the close of bar
// b - 1 + j - j0.  DAY: the realised profit per calendar day, a day added into row when the next one starts.
template <bool DAY>
__device__ __forceinline__ void grid_pass(const GridArgs& a, const double* L, const Grid& g, double qty, const float* px,
                                          int j0, int64_t b, int n, double* row, LaneAcc& c) {
    const int lane = threadIdx.x & 31;
    double p_tick = 0.0;
    int dnet = 0;
    if (lane < n) {
        const int j = j0 + lane;
        const double last = (double)px[j], cur = (double)px[j + 1];
        const bool upmove = cur > last;
        if (upmove || cur < last) {                   // a NaN price on either side is not a move (nor a near tie)
            const double x_lo = upmove ? last : cur, x_hi = upmove ? cur : last;
            const int e_lo = level_bound<false>(L, g.n, estimate(g, x_lo), x_lo);   // first L >= x_lo
            const int e_hi = level_bound<true>(L, g.n, estimate(g, x_hi), x_hi);    // first L > x_hi
            if (g.type == B200BT_GRID_GEOMETRIC &&
                (near_bound(L, g.n, e_lo, x_lo) || near_bound(L, g.n, e_hi, x_hi)))
                ++c.n_tie;
            if (upmove) {
                for (int l = e_lo; l < e_hi; ++l) {
                    // the reference prices a level by levels.index(lv): every copy of a repeated level earns the step
                    // under its first copy f (the lower bound of lv, as the levels are sorted), and nothing when f = 0
                    const double lv = L[l];
                    int f = l;
                    double below = l > 0 ? L[l - 1] : 0.0;
                    if (l > 0 && below == lv) {
                        do --f;
                        while (f > 0 && L[f - 1] == lv);
                        below = f > 0 ? L[f - 1] : 0.0;
                    }
                    const double pr = f > 0 ? __dmul_rn(__dsub_rn(lv, below), qty) : 0.0;
                    if (pr > 0.0) ++c.n_prof;
                    p_tick = __dadd_rn(p_tick, pr);
                    c.cash = __dadd_rn(c.cash, __dmul_rn(lv, qty));
                }
                if (e_hi > e_lo) {
                    c.n_up += e_hi - e_lo;
                    dnet = -(e_hi - e_lo);
                }
            } else {
                for (int l = e_lo; l < e_hi; ++l) c.cash = __dsub_rn(c.cash, __dmul_rn(L[l], qty));
                if (e_hi > e_lo) {
                    c.n_down += e_hi - e_lo;
                    dnet = e_hi - e_lo;
                }
            }
        }
    }
    c.profit = __dadd_rn(c.profit, p_tick);
    // inventory after each tick of the pass: inclusive scan of dnet
    int sc = dnet;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(FULL, sc, d);
        if (lane >= d) sc += v;
    }
    const int lo_sc = __reduce_min_sync(FULL, lane < n ? sc : INT_MAX);
    const int hi_sc = __reduce_max_sync(FULL, lane < n ? sc : INT_MIN);
    c.net_min = min(c.net_min, c.net + lo_sc);
    c.net_max = max(c.net_max, c.net + hi_sc);
    c.net += __shfl_sync(FULL, sc, 31);
    if (DAY) {                                        // realised profit per calendar day
        const int64_t d0 = (a.minute0 + b * a.bar_minutes) / 1440 - a.first_day;
        const int64_t d1 = (a.minute0 + (b + n - 1) * a.bar_minutes) / 1440 - a.first_day;
        const int64_t my_day = (a.minute0 + (b + lane) * a.bar_minutes) / 1440 - a.first_day;
        for (int64_t d = d0; d <= d1; ++d) {
            const double v = warp_sum_d((lane < n && my_day == d) ? p_tick : 0.0);
            if (d != c.day_cur) {
                if (lane == 0 && c.day_cur >= 0) row[c.day_cur] += c.day_val;
                c.day_cur = d;
                c.day_val = 0.0;
            }
            c.day_val += v;
        }
    }
}

// _rebalance_grid (:781-838) at a rebalance tick with price cur, warp-uniform: regenerates the grid around cur with the
// service's current num_grids and pcts when cur is within 5 % of a boundary, counted in n_regen
__device__ __forceinline__ void rebalance(double* L, Grid& g, double cur, int n_cur, double lo_pct, double up_pct,
                                          int& n_regen) {
    if (cur < __dmul_rn(g.lower, 1.05) || cur > __dmul_rn(g.upper, 0.95)) {
        g.lower = __dmul_rn(cur, __dsub_rn(1.0, __ddiv_rn(lo_pct, 100.0)));
        g.upper = __dmul_rn(cur, __dadd_rn(1.0, __ddiv_rn(up_pct, 100.0)));
        g.n = n_cur;
        __syncwarp();
        build_levels(L, g);
        ++n_regen;
    }
}

template <bool DAY>
__global__ void __launch_bounds__(GR_WARPS * 32)
grid_kernel(const GridArgs a) {
    __shared__ float tile[2][GR_TILE + 1];
    __shared__ double levels[GR_WARPS][GR_LEVELS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int i = blockIdx.x * GR_WARPS + wid;
    const bool active = i < a.pop;
    double* L = levels[wid];
    const int s_begin = DAY ? 0 : (int)blockIdx.y, s_end = DAY ? a.S : s_begin + 1;
    const b200bt_grid_individual iv = active ? a.indiv[i] : b200bt_grid_individual{};
    const bool valid = active && iv.num_grids >= 1 && iv.num_grids <= B200BT_GRID_MAX_GRIDS &&
                       (iv.grid_type == B200BT_GRID_ARITHMETIC || iv.grid_type == B200BT_GRID_GEOMETRIC) &&
                       iv.rebalance_ticks >= 1 && iv.adjust_ticks >= 1;
    double* row = (DAY && active) ? a.day + (int64_t)i * a.D : nullptr;
    if (DAY && active) {
        for (int64_t d = lane; d < a.D; d += 32) row[d] = 0.0;
        __syncwarp();
    }
    const int64_t T = a.N - a.start_bar;
    const int64_t n_tiles = (T - 1 + GR_TILE - 1) / GR_TILE;           // ticks 1 .. T - 1
    for (int s = s_begin; s < s_end; ++s) {
        const float* prow = a.price + (int64_t)s * a.ld_price;
        const uint8_t* lab = a.labels ? a.labels + (int64_t)s * a.ld_labels : nullptr;
        const double qty = a.qty[s];
        const int64_t lane_id = (int64_t)i * a.S + s;
        // _initialize_grid at t0
        Grid g;
        g.lower = active ? a.bounds[2 * lane_id] : 0.0;
        g.upper = active ? a.bounds[2 * lane_id + 1] : 0.0;
        g.n = iv.num_grids;
        g.type = iv.grid_type;
        if (valid) build_levels(L, g);
        int n_cur = iv.num_grids;                                  // service-wide parameters
        double lo_pct = iv.lower_pct, up_pct = iv.upper_pct;
        int64_t next_reb = iv.rebalance_ticks, next_adj = iv.adjust_ticks;   // ticks of the next checks
        LaneAcc c{0, 0, 0, 0, 0.0, 0.0, 0, 0, 0, -1, 0.0};
        int n_regen = 0, n_reb = 0, n_adj = 0;

        const int64_t b0 = a.start_bar + 1;
        auto issue = [&](int64_t t) {
            const int64_t tb = b0 + t * GR_TILE, te = min(tb + GR_TILE, a.N);
            float* dst = tile[t & 1];
            for (int64_t j = threadIdx.x; j <= te - tb; j += GR_WARPS * 32) cp4(dst + j, prow + tb - 1 + j);
            cp_commit();
        };
        if (n_tiles > 0) issue(0);
        for (int64_t t = 0; t < n_tiles; ++t) {
            if (t + 1 < n_tiles) {
                issue(t + 1);
                cp_wait<1>();
            } else {
                cp_wait<0>();
            }
            __syncthreads();
            const float* tp = tile[t & 1];
            const int64_t tb = b0 + t * GR_TILE, te = min(tb + GR_TILE, a.N);
            int64_t b = tb;
            while (valid && b < te) {
                const int64_t k0 = b - a.start_bar;
                const int64_t check = min(next_reb, next_adj);    // tick
                const int n = (int)min((int64_t)32, min(te - b, check - k0 + 1));
                grid_pass<DAY>(a, L, g, qty, tp, (int)(b - tb), b, n, row, c);   // ticks k0 .. k0 + n - 1
                b += n;
                const int64_t kc = b - 1 - a.start_bar;
                if (kc != check) continue;
                // ---- checks at tick kc, warp-uniform ----
                const double cur = (double)tp[b - 1 - tb + 1];
                if (kc == next_reb) {                              // _rebalance_grid (:781-838)
                    ++n_reb;
                    next_reb += iv.rebalance_ticks;
                    rebalance(L, g, cur, n_cur, lo_pct, up_pct, n_regen);
                }
                if (kc == next_adj) {                              // _adjust_grid_parameters (:840-905)
                    ++n_adj;
                    next_adj += iv.adjust_ticks;
                    if ((iv.flags & B200BT_GRID_ADAPT_REGIME) && lab && a.use_rules) {
                        const int r = lab[b - 1];
                        if (r < B200BT_GRID_REGIME_RULES && a.rules[r].apply) {
                            n_cur = a.rules[r].num_grids;
                            lo_pct = a.rules[r].lower_pct;
                            up_pct = a.rules[r].upper_pct;
                        }
                    }
                    const double total = warp_sum_d((double)(c.n_up + c.n_down));
                    if (total > 10.0) {
                        const double wr = __ddiv_rn(warp_sum_d((double)c.n_prof), total);
                        if (wr < 0.4) n_cur = max(5, n_cur - 2);
                        else if (wr > 0.7) n_cur = min(20, n_cur + 2);
                    }
                }
            }
            __syncthreads();                                       // the stage is refilled next iteration
        }
        if (!active) continue;
        if (DAY && lane == 0 && c.day_cur >= 0) row[c.day_cur] += c.day_val;
        const double up = warp_sum_d((double)c.n_up), down = warp_sum_d((double)c.n_down);
        const double prof = warp_sum_d((double)c.n_prof), ties = warp_sum_d((double)c.n_tie);
        const double tot_profit = warp_sum_d(c.profit), tot_cash = warp_sum_d(c.cash);
        if (lane == 0) {
            b200bt_grid_stats o;
            if (!valid) {
                double* w = reinterpret_cast<double*>(&o);
                for (int f = 0; f < 20; ++f) w[f] = NAN;
            } else {
                const double total = up + down;
                const double secs = (double)((T - 1) * (int64_t)a.bar_minutes * 60);
                const double last_px = (double)prow[a.N - 1];
                o.total_profit = tot_profit;
                o.total_trades = total;
                o.profitable_trades = prof;
                o.win_rate = total > 0.0 ? __ddiv_rn(prof, total) : 0.0;
                o.profit_per_day = secs > 0.0 ? __ddiv_rn(tot_profit, __ddiv_rn(secs, 86400.0)) : 0.0;
                o.up_crossings = up;
                o.down_crossings = down;
                o.n_regenerations = (double)n_regen;
                o.num_grids = (double)n_cur;
                o.lower = g.lower;
                o.upper = g.upper;
                o.cash = tot_cash;
                o.position = __dmul_rn((double)c.net, qty);
                o.mark_to_market = __dadd_rn(tot_cash, __dmul_rn(o.position, last_px));
                o.max_position = __dmul_rn((double)c.net_max, qty);
                o.min_position = __dmul_rn((double)c.net_min, qty);
                o.n_rebalance_checks = (double)n_reb;
                o.n_adjustments = (double)n_adj;
                o.n_ticks = (double)T;
                o.near_ties = ties;
            }
            a.stats[lane_id] = o;
        }
        __syncwarp();
    }
}

// A lane's state between two adjust ticks is kept in its own stats record (reduced over the warp: counts, profit and cash
// on lane 0), so a warp can take up the lanes of several symbols in turn.  Fields that hold other things until the end:
// num_grids = the active grid's n, total_trades = up + down (read by the adjustment), position / max_position /
// min_position = inventory in units of qty, n_regenerations / n_rebalance_checks = counts, n_ticks = day_cur,
// mark_to_market = day_val.
__device__ __forceinline__ void save_lane(b200bt_grid_stats* r, const Grid& g, const LaneAcc& c, int n_regen, int n_reb) {
    const double up = warp_sum_d((double)c.n_up), down = warp_sum_d((double)c.n_down);
    const double prof = warp_sum_d((double)c.n_prof), ties = warp_sum_d((double)c.n_tie);
    const double profit = warp_sum_d(c.profit), cash = warp_sum_d(c.cash);
    if ((threadIdx.x & 31) == 0) {
        r->total_profit = profit;
        r->total_trades = up + down;
        r->profitable_trades = prof;
        r->up_crossings = up;
        r->down_crossings = down;
        r->near_ties = ties;
        r->cash = cash;
        r->n_regenerations = (double)n_regen;
        r->n_rebalance_checks = (double)n_reb;
        r->num_grids = (double)g.n;
        r->lower = g.lower;
        r->upper = g.upper;
        r->position = (double)c.net;
        r->max_position = (double)c.net_max;
        r->min_position = (double)c.net_min;
        r->n_ticks = (double)c.day_cur;
        r->mark_to_market = c.day_val;
    }
    __syncwarp();
}

// one CTA per individual (one service instance); warp w runs the lanes of symbols w, w + W, ... between two adjust ticks,
// where the warps meet and thread 0 applies the adjustment of every symbol in order.  DAY: W = 1, so every calendar day's
// profits are added into the row in symbol order.
template <bool DAY>
__global__ void __launch_bounds__(GR_WARPS * 32)
grid_service_kernel(const GridArgs a, b200bt_grid_service_stats* service) {
    __shared__ double levels[DAY ? 1 : GR_WARPS][GR_LEVELS];
    __shared__ double sv_pct[2];
    __shared__ int sv_n, sv_adj;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, W = blockDim.x >> 5;
    const int i = blockIdx.x;
    double* L = levels[wid];
    const b200bt_grid_individual iv = a.indiv[i];
    const bool valid = iv.num_grids >= 1 && iv.num_grids <= B200BT_GRID_MAX_GRIDS &&
                       (iv.grid_type == B200BT_GRID_ARITHMETIC || iv.grid_type == B200BT_GRID_GEOMETRIC) &&
                       iv.rebalance_ticks >= 1 && iv.adjust_ticks >= 1;
    double* row = DAY ? a.day + (int64_t)i * a.D : nullptr;
    b200bt_grid_stats* st = a.stats + (int64_t)i * a.S;
    const int64_t T = a.N - a.start_bar;
    if (DAY)
        for (int64_t d = threadIdx.x; d < a.D; d += blockDim.x) row[d] = 0.0;
    if (!valid) {
        for (int s = threadIdx.x; s < a.S; s += blockDim.x) {
            double* w = reinterpret_cast<double*>(st + s);
            for (int f = 0; f < 20; ++f) w[f] = NAN;
        }
        if (service && threadIdx.x == 0) {
            double* w = reinterpret_cast<double*>(service + i);
            for (int f = 0; f < 12; ++f) w[f] = NAN;
        }
        return;
    }
    // _initialize_grid of every symbol at t0
    for (int s = wid; s < a.S; s += W) {
        Grid g;
        g.lower = a.bounds[2 * ((int64_t)i * a.S + s)];
        g.upper = a.bounds[2 * ((int64_t)i * a.S + s) + 1];
        g.n = iv.num_grids;
        const LaneAcc c{0, 0, 0, 0, 0.0, 0.0, 0, 0, 0, -1, 0.0};
        save_lane(st + s, g, c, 0, 0);
    }
    // the service's num_grids and pcts; thread 0's counts of the adjustments
    int n_adj = 0, n_changed = 0, n_min = iv.num_grids, n_max = iv.num_grids;
    if (threadIdx.x == 0) {
        sv_n = iv.num_grids;
        sv_pct[0] = iv.lower_pct;
        sv_pct[1] = iv.upper_pct;
    }
    __syncthreads();
    const int64_t b0 = a.start_bar + 1;
    for (int64_t ks = 1; ks < T;) {                         // one segment: ticks ks .. ke, ke an adjust tick or T - 1
        const int64_t next_adj = (ks + iv.adjust_ticks - 1) / iv.adjust_ticks * iv.adjust_ticks;
        const int64_t ke = min(next_adj, T - 1);
        const int n_cur = sv_n;
        const double lo_pct = sv_pct[0], up_pct = sv_pct[1];
        for (int s = wid; s < a.S; s += W) {
            const float* prow = a.price + (int64_t)s * a.ld_price;
            const double qty = a.qty[s];
            b200bt_grid_stats* r = st + s;
            Grid g;
            g.lower = r->lower;
            g.upper = r->upper;
            g.n = (int)r->num_grids;
            g.type = iv.grid_type;
            const bool first = lane == 0;
            LaneAcc c{first ? (unsigned long long)r->up_crossings : 0ull, first ? (unsigned long long)r->down_crossings : 0ull,
                      first ? (unsigned long long)r->profitable_trades : 0ull, first ? (unsigned long long)r->near_ties : 0ull,
                      first ? r->total_profit : 0.0, first ? r->cash : 0.0, (long long)r->position,
                      (long long)r->max_position, (long long)r->min_position, (int64_t)r->n_ticks, r->mark_to_market};
            int n_regen = (int)r->n_regenerations, n_reb = (int)r->n_rebalance_checks;
            __syncwarp();
            build_levels(L, g);
            int64_t next_reb = (ks + iv.rebalance_ticks - 1) / iv.rebalance_ticks * iv.rebalance_ticks;
            // the passes of grid_kernel: at most 32 ticks, ending at a check tick or at the end of a GR_TILE tile
            for (int64_t b = a.start_bar + ks; b <= a.start_bar + ke;) {
                const int64_t k0 = b - a.start_bar;
                const int64_t te = min(b0 + (b - b0) / GR_TILE * GR_TILE + GR_TILE, a.N);
                const int64_t check = min(next_reb, next_adj);
                const int n = (int)min((int64_t)32, min(te - b, check - k0 + 1));
                grid_pass<DAY>(a, L, g, qty, prow + (b - 1), 0, b, n, row, c);
                b += n;
                const int64_t kc = b - 1 - a.start_bar;
                if (kc != next_reb) continue;
                ++n_reb;
                next_reb += iv.rebalance_ticks;
                rebalance(L, g, (double)prow[b - 1], n_cur, lo_pct, up_pct, n_regen);
            }
            save_lane(r, g, c, n_regen, n_reb);
        }
        __syncthreads();                                    // every symbol has run its ticks up to ke
        if (ke == next_adj && threadIdx.x == 0) {           // _adjust_grid_parameters (:840-905), symbols in order
            int n = n_cur;
            double lo = lo_pct, up = up_pct;
            int r = B200BT_GRID_REGIME_RULES;
            if ((iv.flags & B200BT_GRID_ADAPT_REGIME) && a.labels && a.use_rules) r = a.labels[a.start_bar + ke];
            const bool rule = r < B200BT_GRID_REGIME_RULES && a.rules[r].apply;
            for (int s = 0; s < a.S; ++s) {
                if (rule) {
                    n = a.rules[r].num_grids;
                    lo = a.rules[r].lower_pct;
                    up = a.rules[r].upper_pct;
                    n_min = min(n_min, n);
                    n_max = max(n_max, n);
                }
                const double total = st[s].total_trades;
                if (total > 10.0) {
                    const double wr = __ddiv_rn(st[s].profitable_trades, total);
                    if (wr < 0.4) n = max(5, n - 2);
                    else if (wr > 0.7) n = min(20, n + 2);
                    n_min = min(n_min, n);
                    n_max = max(n_max, n);
                }
            }
            ++n_adj;
            n_changed += n != n_cur;
            sv_n = n;
            sv_pct[0] = lo;
            sv_pct[1] = up;
        }
        __syncthreads();
        ks = ke + 1;
    }
    if (threadIdx.x == 0) sv_adj = n_adj;
    __syncthreads();
    const double secs = (double)((T - 1) * (int64_t)a.bar_minutes * 60);
    for (int s = wid; s < a.S; s += W) {
        b200bt_grid_stats* r = st + s;
        if (lane == 0) {
            if (DAY && r->n_ticks >= 0.0) row[(int64_t)r->n_ticks] += r->mark_to_market;
            const double qty = a.qty[s], last_px = (double)a.price[(int64_t)s * a.ld_price + a.N - 1];
            b200bt_grid_stats o = *r;
            const double total = o.total_trades, prof = o.profitable_trades;
            o.win_rate = total > 0.0 ? __ddiv_rn(prof, total) : 0.0;
            o.profit_per_day = secs > 0.0 ? __ddiv_rn(o.total_profit, __ddiv_rn(secs, 86400.0)) : 0.0;
            o.position = __dmul_rn(r->position, qty);
            o.mark_to_market = __dadd_rn(o.cash, __dmul_rn(o.position, last_px));
            o.max_position = __dmul_rn(r->max_position, qty);
            o.min_position = __dmul_rn(r->min_position, qty);
            o.n_adjustments = (double)sv_adj;
            o.n_ticks = (double)T;
            *r = o;
        }
    }
    if (!service) return;
    __syncthreads();
    if (threadIdx.x == 0) {                                 // _update_performance_metrics (:941-958)
        b200bt_grid_service_stats v;
        v.total_profit = 0.0;
        v.total_trades = 0.0;
        v.profitable_trades = 0.0;
        for (int s = 0; s < a.S; ++s) {
            v.total_profit = __dadd_rn(v.total_profit, st[s].total_profit);
            v.total_trades += st[s].total_trades;
            v.profitable_trades += st[s].profitable_trades;
        }
        v.win_rate = v.total_trades > 0.0 ? __ddiv_rn(v.profitable_trades, v.total_trades) : 0.0;
        v.profit_per_day = secs > 0.0 ? __ddiv_rn(v.total_profit, __ddiv_rn(secs, 86400.0)) : 0.0;
        v.num_grids = (double)sv_n;
        v.lower_pct = sv_pct[0];
        v.upper_pct = sv_pct[1];
        v.n_adjustments = (double)n_adj;
        v.n_num_grids_changes = (double)n_changed;
        v.min_num_grids = (double)n_min;
        v.max_num_grids = (double)n_max;
        service[i] = v;
    }
}

}  // namespace
}  // namespace b200bt

using namespace b200bt;

// The argument checks of both grid entry points (messages prefixed by `what`) and their GridArgs.  The lane sweep reads a
// label row per symbol or one shared row; the service reads one row.
static int grid_args(const char* what, bool service, const float* price, int64_t ld_price, int S, int64_t N,
                     int64_t start_bar, int bar_minutes, int64_t minute0, const b200bt_grid_individual* indiv, int pop,
                     const double* qty, const double* init_bounds, const uint8_t* labels_or_null, int64_t ld_labels,
                     const b200bt_grid_regime_rule* regime_table_host_or_null, b200bt_grid_stats* stats,
                     double* day_profit_or_null, int64_t D, GridArgs& a) {
    B200BT_REQUIRE(price && indiv && qty && init_bounds && stats, B200BT_EINVAL, "%s: null pointer", what);
    B200BT_REQUIRE(S >= 1 && pop >= 1 && N >= 1 && ld_price >= N, B200BT_EINVAL, "%s: bad sizes", what);
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "%s: N must be < 2^30 bars", what);
    B200BT_REQUIRE(start_bar >= 0 && start_bar < N, B200BT_EINVAL, "%s: start_bar = %lld outside [0, N = %lld)", what,
                   (long long)start_bar, (long long)N);
    B200BT_REQUIRE(bar_clock_ok(minute0, N, bar_minutes), B200BT_EINVAL,
                   "%s: bad bar clock (bar_minutes > 0, minute0 >= 0)", what);
    if (service) {
        B200BT_REQUIRE(!labels_or_null || ld_labels == 0, B200BT_EINVAL,
                       "%s: ld_labels must be 0: the service reads one regime label row", what);
    } else {
        B200BT_REQUIRE(!labels_or_null || ld_labels == 0 || ld_labels >= N, B200BT_EINVAL,
                       "%s: ld_labels must be 0 (one shared row) or >= N", what);
        // the stats launch's grid.y is S
        B200BT_REQUIRE(S <= 65535, B200BT_ELIMIT, "%s: at most 65535 symbols (S = %d)", what, S);
    }
    const int64_t need_days = series_days(minute0, N, bar_minutes);
    B200BT_REQUIRE(!day_profit_or_null || D >= need_days, B200BT_EINVAL, "%s: D = %lld days, the series spans %lld", what,
                   (long long)D, (long long)need_days);
    for (int r = 0; r < B200BT_GRID_REGIME_RULES; ++r) {
        a.rules[r] = regime_table_host_or_null ? regime_table_host_or_null[r] : b200bt_grid_regime_rule{0, 0, 0.0, 0.0};
        B200BT_REQUIRE(!a.rules[r].apply || (a.rules[r].num_grids >= 1 && a.rules[r].num_grids <= B200BT_GRID_MAX_GRIDS),
                       B200BT_EINVAL, "%s: regime rule %d sets num_grids = %d outside 1 .. %d", what, r,
                       a.rules[r].num_grids, B200BT_GRID_MAX_GRIDS);
    }
    int rc = check_device();
    if (rc) return rc;
    a.price = price;
    a.ld_price = ld_price;
    a.N = N;
    a.start_bar = start_bar;
    a.minute0 = minute0;
    a.ld_labels = service ? 0 : ld_labels;
    a.D = D;
    a.first_day = minute0 / 1440;
    a.S = S;
    a.pop = pop;
    a.bar_minutes = bar_minutes;
    a.use_rules = regime_table_host_or_null != nullptr;
    a.indiv = indiv;
    a.qty = qty;
    a.bounds = init_bounds;
    a.labels = labels_or_null;
    a.stats = stats;
    a.day = day_profit_or_null;
    return B200BT_OK;
}

extern "C" int b200bt_grid_sweep(const float* price, int64_t ld_price, int S, int64_t N, int64_t start_bar, int bar_minutes,
                                 int64_t minute0, const b200bt_grid_individual* indiv, int pop, const double* qty,
                                 const double* init_bounds, const uint8_t* labels_or_null, int64_t ld_labels,
                                 const b200bt_grid_regime_rule* regime_table_host_or_null, b200bt_grid_stats* stats,
                                 double* day_profit_or_null, int64_t D, b200bt_stream_t stream) {
    GridArgs a;
    int rc = grid_args("grid_sweep", false, price, ld_price, S, N, start_bar, bar_minutes, minute0, indiv, pop, qty,
                       init_bounds, labels_or_null, ld_labels, regime_table_host_or_null, stats, day_profit_or_null, D, a);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned groups = (unsigned)((pop + GR_WARPS - 1) / GR_WARPS);
    if (day_profit_or_null) {
        grid_kernel<true><<<dim3(groups, 1), GR_WARPS * 32, 0, st>>>(a);
    } else {
        grid_kernel<false><<<dim3(groups, (unsigned)S), GR_WARPS * 32, 0, st>>>(a);
    }
    B200BT_LAUNCH_CHECK("grid_sweep");
    return B200BT_OK;
}

extern "C" int b200bt_grid_service_sweep(const float* price, int64_t ld_price, int S, int64_t N, int64_t start_bar,
                                         int bar_minutes, int64_t minute0, const b200bt_grid_individual* indiv, int pop,
                                         const double* qty, const double* init_bounds, const uint8_t* labels_or_null,
                                         int64_t ld_labels, const b200bt_grid_regime_rule* regime_table_host_or_null,
                                         b200bt_grid_stats* stats, b200bt_grid_service_stats* service_or_null,
                                         double* day_profit_or_null, int64_t D, b200bt_stream_t stream) {
    GridArgs a;
    int rc = grid_args("grid_service_sweep", true, price, ld_price, S, N, start_bar, bar_minutes, minute0, indiv, pop, qty,
                       init_bounds, labels_or_null, ld_labels, regime_table_host_or_null, stats, day_profit_or_null, D, a);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (day_profit_or_null) {
        grid_service_kernel<true><<<(unsigned)pop, 32, 0, st>>>(a, service_or_null);
    } else {
        grid_service_kernel<false><<<(unsigned)pop, min(S, GR_WARPS) * 32, 0, st>>>(a, service_or_null);
    }
    B200BT_LAUNCH_CHECK("grid_service_sweep");
    return B200BT_OK;
}
