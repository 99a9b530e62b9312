// Dollar-cost averaging backtest (sm_90a): services/dca_strategy.py's simulation loop over a market's bars for a whole
// population at once.  Contract and the rule restated: include/b200bt.h (b200bt_dca_*); design: DESIGN.md section 3.14.
//
// dca_dip_kernel    the market-only drop series of _check_for_dips: one warp per (symbol, run of DIP_RUN days) walks its
//                   days in order, keeping the highs' maxima of the 7 days before in registers, and scans each day's bars
//                   32 at a time (an inclusive max scan carried across the day): O(N (1 + 7 / DIP_RUN)) reads per symbol.
// dca_level_kernel  block maxima of the drop series over 32, 1 024 and 32 768 bars (fmax: NaN is no dip) in the workspace.
// dca_kernel        one CTA per individual, one warp per symbol (groups of 32 symbols in turn when S > 32).  Purchases are
//                   sparse, so a warp jumps from event to event -- the next scheduled tick, the next dip tick, the next day
//                   end -- with warp-uniform scalar float64 code.  The next dip tick comes from a warp search of the
//                   pyramid: 32 entries per step, a ballot of >= threshold, every block below the threshold skipped.  It
//                   stays valid until the lane's next dip purchase (only the cooldown moves it).  The warps meet with
//                   __syncthreads at rebalance ticks (thread 0 sums the values in symbol order and decides) and, with day
//                   rows, at day ends (thread 0 adds the symbols' changes in order).  No atomics.
#include <math.h>
#include "common.cuh"

namespace b200bt {
namespace {

constexpr int DIP_RUN = 16;                          // days per warp of the drop series
constexpr int LEVELS = 3;                            // pyramid levels above the series: 32, 1 024, 32 768 bars
constexpr int KIND_SCHEDULED = 0, KIND_DIP = 1, KIND_REBALANCE = 2;

__host__ __device__ inline int64_t level_len(int64_t N, int l) {          // blocks of 32^l bars, l = 1 .. 3
    const int64_t span = (int64_t)1 << (5 * l);
    return (((N + span - 1) / span) + 1) & ~(int64_t)1;
}

// first bar whose start minute is >= x (x relative to minute0), clamped to >= 0
__device__ __forceinline__ int64_t bar_at_or_after(int64_t x, int bm) { return x <= 0 ? 0 : (x + bm - 1) / bm; }

__global__ void dca_dip_kernel(const float* __restrict__ high, const float* __restrict__ close, int64_t ld, int S, int64_t N,
                               int64_t minute0, int bm, double* __restrict__ out, int64_t ld_out, int64_t first_day,
                               int64_t n_days) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t runs = (n_days + DIP_RUN - 1) / DIP_RUN;
    if (warp >= runs * S) return;
    const int s = (int)(warp / runs);
    const int64_t d0 = first_day + (warp % runs) * DIP_RUN, d1 = min(d0 + DIP_RUN, first_day + n_days);
    const float* hr = high + (int64_t)s * ld;
    const float* cr = close + (int64_t)s * ld;
    double* o = out + (int64_t)s * ld_out;
    double ring[7];                                  // ring[j]: high of day d - 1 - j, -inf for a day without bars
#pragma unroll
    for (int j = 0; j < 7; ++j) ring[j] = -INFINITY;
    for (int64_t d = max(first_day, d0 - 7); d < d1; ++d) {
        const int64_t blo = bar_at_or_after(d * 1440 - minute0, bm), bhi = min(N, bar_at_or_after((d + 1) * 1440 - minute0, bm));
        double m6 = -INFINITY, m7;                   // days d-6 .. d-1, and d-7 .. d-1 (a bar at midnight reaches d - 7)
        int c6 = 0, c7;
#pragma unroll
        for (int j = 0; j < 6; ++j)
            if (ring[j] > -INFINITY) {
                m6 = fmax(m6, ring[j]);
                ++c6;
            }
        m7 = m6;
        c7 = c6;
        if (ring[6] > -INFINITY) {
            m7 = fmax(m7, ring[6]);
            ++c7;
        }
        double carry = -INFINITY;                    // the day's high so far
        for (int64_t b0 = blo; b0 < bhi; b0 += 32) {
            const int64_t b = b0 + lane;
            const bool in = b < bhi;
            double h = in ? (double)hr[b] : -INFINITY;
#pragma unroll
            for (int k = 1; k < 32; k <<= 1) {
                const double v = __shfl_up_sync(FULL, h, k);
                if (lane >= k) h = fmax(h, v);
            }
            h = fmax(h, carry);
            carry = __shfl_sync(FULL, h, 31);
            if (d >= d0 && in) {
                const bool midnight = (minute0 + b * bm) % 1440 == 0;
                const double H = fmax(midnight ? m7 : m6, h);
                const int klines = (midnight ? c7 : c6) + 1;
                double r = NAN;
                if (klines >= 2 && H != 0.0) r = __dmul_rn(__ddiv_rn(__dsub_rn(H, (double)cr[b]), H), 100.0);
                o[b] = r;
            }
        }
#pragma unroll
        for (int j = 6; j > 0; --j) ring[j] = ring[j - 1];
        ring[0] = carry;
    }
}

__global__ void dca_level_kernel(const double* __restrict__ src, int64_t ld_src, int64_t n_src, double* __restrict__ dst,
                                 int64_t ld_dst, int64_t n_dst, int S) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)S * n_dst) return;
    const int s = (int)(idx / n_dst);
    const int64_t j = idx % n_dst;
    double m = NAN;
    for (int t = 0; t < 32; ++t) {
        const int64_t b = j * 32 + t;
        if (b < n_src) m = fmax(m, src[(int64_t)s * ld_src + b]);
    }
    dst[(int64_t)s * ld_dst + j] = m;
}

struct DcaArgs {
    const float* close;
    const double* dip;
    const double* lv[LEVELS];
    int64_t ld_close, ld_dip, ld_lv[LEVELS], N, start_bar, minute0, ld_labels, D, first_day, tick_us;
    int S, pop, bar_minutes;
    const b200bt_dca_individual* indiv;
    const int64_t* first_us;
    const double* target;
    const double* pow10;
    const uint8_t* labels;
    double usdc;
    b200bt_dca_stats* stats;
    b200bt_dca_service* service;
    double* day;
};

__device__ __forceinline__ uint32_t fmix32(uint32_t h) {
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h;
}

// smallest bar b in [p, N) with dip[b] >= thr (N if none): warp-cooperative, uniform result.  At level l (blocks of 32^l
// bars) a step reads up to 32 entries, never past the next 32^(l+1) boundary below the top level; a miss climbs, a hit
// descends into the first block that holds a value >= thr (block maxima are exact, so it holds one).
__device__ int64_t next_dip(const DcaArgs& a, int s, int64_t p, double thr) {
    const int lane = threadIdx.x & 31;
    int l = 0;
    while (p < a.N) {
        const int64_t span = (int64_t)1 << (5 * l);
        const int64_t b = p / span;
        const int64_t nb = (a.N + span - 1) / span;
        const int n = l == LEVELS ? 32 : 32 - (int)(b & 31);
        const int64_t idx = b + lane;
        bool hit = false;
        if (lane < n && idx < nb) {
            const double v = l == 0 ? a.dip[(int64_t)s * a.ld_dip + idx] : a.lv[l - 1][(int64_t)s * a.ld_lv[l - 1] + idx];
            hit = v >= thr;
        }
        const unsigned m = __ballot_sync(FULL, hit);
        if (m) {
            p = (b + __ffs(m) - 1) * span;
            if (l == 0) return p;
            --l;
        } else {
            p = (b + n) * span;
            l = min(l + 1, LEVELS);
        }
    }
    return a.N;
}

// one symbol's service state (warp-uniform)
struct Lane {
    double Q, I, order_sum, last_price, min_day, v_prev;
    int64_t next_us, ks, kd, kday, last_tick, last_dip, n_sched, n_dip, n_reb, n_zero;
    uint32_t hash;
};

struct Ctx {
    const DcaArgs& a;
    const b200bt_dca_individual& iv;
    const float* crow;
    const uint8_t* lab;
    int64_t T, cool_ticks;
    double pw;
    int s, last;

    __device__ double price(int64_t k) const { return (double)crow[a.start_bar + k]; }
    __device__ int label(int64_t k) const {
        if (!lab) return B200BT_REGIME_UNKNOWN;
        const int r = lab[a.start_bar + k];
        return r < 5 ? r : B200BT_REGIME_UNKNOWN;
    }
    __device__ int64_t minute(int64_t k) const { return a.minute0 + (a.start_bar + k) * a.bar_minutes; }
    __device__ int weekend(int64_t k) const { return (minute(k) / 1440 + 3) % 7 >= 5; }
    // last tick of the day holding tick k (k < T)
    __device__ int64_t day_last(int64_t k) const {
        const int64_t d = minute(k) / 1440;
        return min(T - 1, ((d + 1) * 1440 - 1 - a.minute0) / a.bar_minutes - a.start_bar);
    }
    __device__ int64_t sched_tick(int64_t now_us, int64_t next_us, int64_t k_min) const {
        if (next_us <= now_us) return k_min;
        return max(k_min, (next_us + a.tick_us - 1) / a.tick_us);
    }
    __device__ void buy(Lane& L, int64_t k, int kind, double order) const {
        const double p = price(k);
        const double q = __ddiv_rn(floor(__dmul_rn(__ddiv_rn(order, p), pw)), pw);
        L.I = __dadd_rn(L.I, __dmul_rn(p, q));
        L.Q = __dadd_rn(L.Q, q);
        L.last_price = p;
        L.last_tick = k;
        L.hash ^= fmix32((uint32_t)(4 * k + kind));
        if (q == 0.0) ++L.n_zero;
    }
    __device__ void scheduled(Lane& L, int64_t k) const {
        const int lb = label(k);
        const double order = iv.order[last][0][lb == B200BT_REGIME_BEAR];
        buy(L, k, KIND_SCHEDULED, order);
        L.order_sum = __dadd_rn(L.order_sum, order);
        ++L.n_sched;
        const int64_t now = k * a.tick_us;
        L.next_us = now + iv.later_us[last][lb][weekend(k)];
        L.ks = sched_tick(now, L.next_us, k + 1);
    }
    __device__ void dip(Lane& L, int64_t k) const {
        const double order = iv.order[last][1][label(k) == B200BT_REGIME_BEAR];
        buy(L, k, KIND_DIP, order);
        L.order_sum = __dadd_rn(L.order_sum, order);
        ++L.n_dip;
        L.last_dip = k;
        const int64_t from = k + cool_ticks;
        L.kd = from < T ? next_dip(a, s, a.start_bar + from, iv.dip_threshold_pct) - a.start_bar : T;
    }
    // the day-end value Q * c - I; returns the change since the previous day end
    __device__ double day_end(Lane& L, int64_t k) const {
        const double v = __dsub_rn(__dmul_rn(L.Q, price(k)), L.I);
        if (v < L.min_day) L.min_day = v;
        const double dv = __dsub_rn(v, L.v_prev);
        L.v_prev = v;
        L.kday = k + 1 < T ? day_last(k + 1) : T;
        return dv;
    }
    // every event before tick stop, then the scheduled purchase at stop (stop < T): the part of tick stop that precedes a
    // rebalance
    __device__ void run_until(Lane& L, int64_t stop) const {
        while (true) {
            const int64_t k = min(L.ks, min(L.kd, L.kday));
            if (k >= stop) break;
            if (L.ks == k) scheduled(L, k);
            if (L.kd == k) dip(L, k);
            if (L.kday == k) day_end(L, k);
        }
        if (stop < T && L.ks == stop) scheduled(L, stop);
    }
};

template <bool DAY>
__global__ void __launch_bounds__(B200BT_DCA_MAX_COUPLED * 32) dca_kernel(const __grid_constant__ DcaArgs a) {
    __shared__ double sh_v[B200BT_DCA_MAX_COUPLED];
    __shared__ double sh_buy[B200BT_DCA_MAX_COUPLED];
    __shared__ double sh_dv[B200BT_DCA_MAX_COUPLED];
    __shared__ double sh_inv[B200BT_DCA_MAX_COUPLED], sh_val[B200BT_DCA_MAX_COUPLED], sh_cnt[B200BT_DCA_MAX_COUPLED];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, W = blockDim.x >> 5;
    const int i = blockIdx.x;
    const b200bt_dca_individual& iv = a.indiv[i];
    const int64_t T = a.N - a.start_bar;
    const bool reb = (iv.flags & B200BT_DCA_REBALANCE) != 0;
    const bool valid = !reb || (a.S <= B200BT_DCA_MAX_COUPLED && iv.rebalance_period >= 1 && iv.rebalance_first >= 0);
    double* row = DAY ? a.day + (int64_t)i * a.D : nullptr;
    if (DAY) {
        for (int64_t d = threadIdx.x; d < a.D; d += blockDim.x) row[d] = 0.0;
        __syncthreads();
    }
    const int64_t cool = iv.dip_cooldown_minutes;
    const int64_t cool_ticks = cool <= 0 ? 1 : max((int64_t)1, (cool + a.bar_minutes - 1) / a.bar_minutes);
    double svc_n = 0.0, svc_inv = 0.0, svc_val = 0.0;                 // thread 0: the service sums, symbols in order
    const int groups = (a.S + W - 1) / W;
    for (int g = 0; g < groups; ++g) {
        const int s = g * W + w;
        const int nw = min(W, a.S - g * W);                         // symbols of this group
        const bool act = valid && s < a.S;
        const int sc = act ? s : 0;
        const Ctx c{a, iv, a.close + (int64_t)sc * a.ld_close,
                    a.labels ? a.labels + (int64_t)sc * a.ld_labels : nullptr, T, cool_ticks, act ? a.pow10[sc] : 1.0, sc,
                    sc == a.S - 1};
        Lane L{};
        L.min_day = INFINITY;
        L.last_tick = L.last_dip = -1;
        L.kd = L.ks = L.kday = T;
        if (act) {
            L.next_us = a.first_us[((int64_t)i * a.S + s) * 10 + c.label(0) * 2 + c.weekend(0)];
            L.ks = c.sched_tick(0, L.next_us, 0);
            if (iv.flags & B200BT_DCA_DIP) L.kd = next_dip(a, s, a.start_bar, iv.dip_threshold_pct) - a.start_bar;
            L.kday = c.day_last(0);
        }
        int64_t k_reb = (reb && valid) ? iv.rebalance_first : T;
        int64_t k_day = (DAY && valid) ? c.day_last(0) : T;
        int64_t n_checks = 0;
        while (true) {
            const int64_t k = min(k_reb, k_day);
            if (act) c.run_until(L, k);
            if (k >= T) break;
            if (k == k_reb) {                                         // _rebalance_portfolio
                if (act && lane == 0) sh_v[w] = __dmul_rn(L.Q, c.price(k));
                __syncthreads();
                if (threadIdx.x == 0) {
                    double total = 0.0;
                    for (int j = 0; j < nw; ++j) total = __dadd_rn(total, sh_v[j]);
                    total = __dadd_rn(total, a.usdc);
                    for (int j = 0; j < nw; ++j) {
                        const double v = sh_v[j], t = a.target[g * W + j];
                        const double alloc = total > 0.0 ? __ddiv_rn(v, total) : 0.0;
                        const double dev = t > 0.0 ? __dmul_rn(fabs(__ddiv_rn(__dsub_rn(alloc, t), t)), 100.0) : 0.0;
                        double buy = NAN;
                        if (dev > iv.max_deviation_pct) {
                            const double tv = __dmul_rn(total, t);
                            if (v < tv) buy = __dsub_rn(tv, v);
                        }
                        sh_buy[j] = buy;
                    }
                }
                __syncthreads();
                if (act && !isnan(sh_buy[w])) {
                    c.buy(L, k, KIND_REBALANCE, sh_buy[w]);
                    ++L.n_reb;
                }
                ++n_checks;
                k_reb += iv.rebalance_period;
            }
            if (act && L.kd == k) c.dip(L, k);
            if (act && L.kday == k) {
                const double dv = c.day_end(L, k);
                if (DAY && lane == 0) sh_dv[w] = dv;
            }
            if (DAY && k == k_day) {
                __syncthreads();
                if (threadIdx.x == 0) {
                    const int64_t d = c.minute(k) / 1440 - a.first_day;
                    double acc = g == 0 ? 0.0 : row[d];
                    for (int j = 0; j < nw; ++j) acc = __dadd_rn(acc, sh_dv[j]);
                    row[d] = acc;
                }
                __syncthreads();
                k_day = k + 1 < T ? c.day_last(k + 1) : T;
            }
        }
        // the last tick's _update_performance_metrics
        const double p_last = c.price(T - 1);
        const double cv = __dmul_rn(L.Q, p_last);
        if (lane == 0 && s < a.S) {
            b200bt_dca_stats o;
            if (!valid) {
                double* f = reinterpret_cast<double*>(&o);
                for (int j = 0; j < 20; ++j) f[j] = NAN;
            } else {
                o.total_invested = L.I;
                o.total_quantity = L.Q;
                o.average_price = L.Q > 0.0 ? __ddiv_rn(L.I, L.Q) : 0.0;
                o.current_value = cv;
                o.profit_loss = L.I > 0.0 ? __dsub_rn(cv, L.I) : 0.0;
                o.profit_loss_pct = L.I > 0.0 ? __dmul_rn(__ddiv_rn(o.profit_loss, L.I), 100.0) : 0.0;
                o.n_scheduled = (double)L.n_sched;
                o.n_dip = (double)L.n_dip;
                o.n_rebalance = (double)L.n_reb;
                o.order_usdc = L.order_sum;
                o.last_purchase_price = L.last_price;
                o.last_purchase_tick = (double)L.last_tick;
                o.next_scheduled_us = (double)L.next_us;
                o.last_dip_tick = (double)L.last_dip;
                o.n_zero_quantity = (double)L.n_zero;
                o.n_rebalance_checks = (double)n_checks;
                o.min_day_profit_loss = L.min_day;
                o.purchase_hash = (double)L.hash;
                o.n_ticks = (double)T;
                o.reserved = 0.0;
            }
            a.stats[(int64_t)i * a.S + s] = o;
            sh_inv[w] = L.I;
            sh_val[w] = cv;
            sh_cnt[w] = (double)(L.n_sched + L.n_dip);
        }
        if (a.service) {
            __syncthreads();
            if (threadIdx.x == 0) {
                for (int j = 0; j < nw; ++j) {
                    svc_n += sh_cnt[j];
                    svc_inv = __dadd_rn(svc_inv, sh_inv[j]);
                    svc_val = __dadd_rn(svc_val, sh_val[j]);
                }
            }
            __syncthreads();
        }
    }
    if (a.service && threadIdx.x == 0) {
        b200bt_dca_service o;
        if (!valid) {
            o = b200bt_dca_service{NAN, NAN, NAN, NAN, NAN};
        } else {
            o.total_purchases = svc_n;
            o.total_invested = svc_inv;
            o.total_value = svc_val;
            o.total_profit = __dsub_rn(svc_val, svc_inv);
            o.total_profit_pct = svc_inv > 0.0 ? __dmul_rn(__ddiv_rn(o.total_profit, svc_inv), 100.0) : 0.0;
        }
        a.service[i] = o;
    }
}

}  // namespace
}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_dca_dip_pct(const float* high, const float* close, int64_t ld, int S, int64_t N, int64_t minute0,
                                  int bar_minutes, double* dip_pct, int64_t ld_dip, b200bt_stream_t stream) {
    B200BT_REQUIRE(high && close && dip_pct, B200BT_EINVAL, "dca_dip_pct: null pointer");
    B200BT_REQUIRE(S >= 1 && N >= 1 && ld >= N && ld_dip >= N, B200BT_EINVAL, "dca_dip_pct: bad sizes");
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "dca_dip_pct: N must be < 2^30 bars");
    B200BT_REQUIRE(bar_clock_ok(minute0, N, bar_minutes), B200BT_EINVAL,
                   "dca_dip_pct: bad bar clock (bar_minutes > 0, minute0 >= 0)");
    int rc = check_device();
    if (rc) return rc;
    const int64_t first_day = minute0 / 1440;
    const int64_t n_days = series_days(minute0, N, bar_minutes);
    const int64_t warps = (n_days + DIP_RUN - 1) / DIP_RUN * S;
    dca_dip_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(high, close, ld, S, N, minute0, bar_minutes,
                                                                                 dip_pct, ld_dip, first_day, n_days);
    B200BT_LAUNCH_CHECK("dca_dip_pct");
    return B200BT_OK;
}

extern "C" int64_t b200bt_dca_workspace_bytes(int S, int64_t N) {
    if (S < 1 || N < 1) return 0;
    int64_t n = 0;
    for (int l = 1; l <= LEVELS; ++l) n += level_len(N, l);
    return n * (int64_t)S * (int64_t)sizeof(double);
}

extern "C" int b200bt_dca_sweep(const float* close, int64_t ld_close, const double* dip_pct, int64_t ld_dip, int S, int64_t N,
                                int64_t start_bar, int bar_minutes, int64_t minute0, void* workspace,
                                int64_t workspace_bytes, const b200bt_dca_individual* indiv, const int64_t* first_us,
                                int pop, int rebalance_any, const double* target, const double* pow10,
                                const uint8_t* labels_or_null, int64_t ld_labels, double usdc_balance,
                                b200bt_dca_stats* stats, b200bt_dca_service* service_or_null, double* day_or_null,
                                int64_t D, b200bt_stream_t stream) {
    B200BT_REQUIRE(close && dip_pct && workspace && indiv && first_us && target && pow10 && stats, B200BT_EINVAL,
                   "dca_sweep: null pointer");
    B200BT_REQUIRE(S >= 1 && pop >= 1 && N >= 1 && ld_close >= N && ld_dip >= N, B200BT_EINVAL, "dca_sweep: bad sizes");
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "dca_sweep: N must be < 2^30 bars");
    B200BT_REQUIRE(start_bar >= 0 && start_bar < N, B200BT_EINVAL, "dca_sweep: start_bar = %lld outside [0, N = %lld)",
                   (long long)start_bar, (long long)N);
    B200BT_REQUIRE(bar_clock_ok(minute0, N, bar_minutes) && N * (int64_t)bar_minutes < (1ll << 62) / 60000000ll,
                   B200BT_EINVAL, "dca_sweep: bad bar clock (bar_minutes > 0, minute0 >= 0, N * bar_minutes us < 2^62)");
    B200BT_REQUIRE(!labels_or_null || ld_labels == 0 || ld_labels >= N, B200BT_EINVAL,
                   "dca_sweep: ld_labels must be 0 (one shared row) or >= N");
    B200BT_REQUIRE(workspace_bytes >= b200bt_dca_workspace_bytes(S, N), B200BT_EINVAL,
                   "dca_sweep: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                   (long long)b200bt_dca_workspace_bytes(S, N));
    const int64_t need_days = series_days(minute0, N, bar_minutes);
    B200BT_REQUIRE(!day_or_null || D >= need_days, B200BT_EINVAL, "dca_sweep: D = %lld days, the series spans %lld",
                   (long long)D, (long long)need_days);
    B200BT_REQUIRE(!(rebalance_any || day_or_null) || S <= B200BT_DCA_MAX_COUPLED, B200BT_ELIMIT,
                   "dca_sweep: S = %d symbols; rebalancing and day rows couple at most %d", S, B200BT_DCA_MAX_COUPLED);
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    DcaArgs a;
    a.close = close;
    a.dip = dip_pct;
    a.ld_close = ld_close;
    a.ld_dip = ld_dip;
    double* ws = static_cast<double*>(workspace);
    const double* src = dip_pct;
    int64_t ld_src = ld_dip, n_src = N;
    for (int l = 1; l <= LEVELS; ++l) {                               // the pyramid, level by level
        const int64_t n = level_len(N, l);
        dca_level_kernel<<<(unsigned)(((int64_t)S * n + 255) / 256), 256, 0, st>>>(src, ld_src, n_src, ws, n, n, S);
        B200BT_LAUNCH_CHECK("dca_sweep: block maxima");
        a.lv[l - 1] = ws;
        a.ld_lv[l - 1] = n;
        src = ws;
        ld_src = n_src = n;
        ws += (int64_t)S * n;
    }
    a.N = N;
    a.start_bar = start_bar;
    a.minute0 = minute0;
    a.ld_labels = ld_labels;
    a.D = D;
    a.first_day = minute0 / 1440;
    a.tick_us = (int64_t)bar_minutes * 60000000ll;
    a.S = S;
    a.pop = pop;
    a.bar_minutes = bar_minutes;
    a.indiv = indiv;
    a.first_us = first_us;
    a.target = target;
    a.pow10 = pow10;
    a.labels = labels_or_null;
    a.usdc = usdc_balance;
    a.stats = stats;
    a.service = service_or_null;
    a.day = day_or_null;
    const int threads = 32 * (S < B200BT_DCA_MAX_COUPLED ? S : B200BT_DCA_MAX_COUPLED);
    if (day_or_null) {
        dca_kernel<true><<<(unsigned)pop, threads, 0, st>>>(a);
    } else {
        dca_kernel<false><<<(unsigned)pop, threads, 0, st>>>(a);
    }
    B200BT_LAUNCH_CHECK("dca_sweep");
    return B200BT_OK;
}
