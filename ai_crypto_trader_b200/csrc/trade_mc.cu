// Trade-sequence Monte-Carlo of backtested strategies (sm_90a): how much of a strategy's final equity and maximum
// drawdown comes from the order in which its round trips happened to arrive.
//
// Reference semantics: services/strategy_evaluation.py.
//   trade records of one lane (entry pnl -fee, exit pnl = trip pnl)   _simulate_trades :746-878
//   equity walk, peak and per-record drawdown                         calculate_metrics :119-139
// Resampling rule: services/monte_carlo_service.py:277-298 (iid bootstrap) applied to round trips.
//
// Two kernels:
//   trade_pnl_kernel  a sweep's event words -> per lane (n_trips, fee, trip_pnl[]), one CTA per lane: each exit priced by
//                     record_pnl, the sweep's exact float64 expression of _simulate_trades (explicit _rn intrinsics).
//   trade_mc_kernel   one CTA = TMC_THREADS paths of ONE lane, one thread per path.  The lane's trip PnL is staged in
//                     shared memory when it fits (TMC_SMEM_TRIPS) and read through L2 otherwise.  Each path draws T trip
//                     indices (bootstrap, block bootstrap or a keyed permutation) and walks the equity in float64 in the
//                     reference's record order: E -= fee (entry record), E += trip_pnl (exit record).
// Drawdown in closed form: for a fixed peak P, (P - E) / P is monotone in E under correctly rounded subtraction and
// division, so the largest per-record drawdown of a stretch below P is (P - min E) / P, evaluated once when the stretch
// ends (a new peak or the end of the path) -- bit-identical to the per-record maximum (DESIGN 3.8).
#include <math.h>
#include <string.h>
#include <algorithm>
#include <numeric>
#include <vector>
#include "philox.cuh"
#include "sweep_dev.cuh"

namespace b200bt {

constexpr int PNL_THREADS = 128;

// ---- round-trip PnL from the sweep's event words ------------------------------------------------------------------
// Lane = i * S + s.  Records come in (entry, exit) pairs; a position still open at the end was force-closed by the sweep
// (:849-876), so n_records is even.  qty = size / entry, pnl = qty * move - size * 0.002 (:819-820, :836-837, :852-853,
// :866-867) with move = price - entry for a long trip, entry - price for a short one (entry word's SELL bit).
__global__ void __launch_bounds__(PNL_THREADS)
trade_pnl_kernel(const float* __restrict__ price, int64_t ld, int S, const b200bt_individual* __restrict__ indiv,
                 const b200bt_lane_stats* __restrict__ stats, const uint32_t* __restrict__ events, int64_t event_cap,
                 double* __restrict__ trip_pnl, int64_t ld_trip, int32_t* __restrict__ n_trips, double* __restrict__ fee) {
    const int64_t lane = blockIdx.x;
    const int s = (int)(lane % S);
    const double size = indiv[lane / S].position_size;
    const int64_t n_rec = (int64_t)stats[lane].n_records;
    const bool lost = n_rec > event_cap;          // the event buffer did not hold every record of the lane
    if (threadIdx.x == 0) {
        n_trips[lane] = lost ? -1 : (int32_t)(n_rec / 2);
        fee[lane] = __dmul_rn(size, 0.001);       // :796-797, :810-811
    }
    if (lost) return;
    const float* row = price + (int64_t)s * ld;
    const uint32_t* ev = events + lane * event_cap;
    double* out = trip_pnl + lane * ld_trip;
    const double fee2 = __dmul_rn(size, 0.002);
    for (int64_t j = threadIdx.x; j < n_rec / 2; j += blockDim.x) {
        const uint32_t a = ev[2 * j], b = ev[2 * j + 1];     // entry, exit: record_pnl charges an exit no entry fee
        int dur;
        out[j] = record_pnl(true, b, row[b & B200BT_EVENT_BAR_MASK], a, row[a & B200BT_EVENT_BAR_MASK], size, 0.0, fee2, dur);
    }
}

// ---- the Monte-Carlo walk -----------------------------------------------------------------------------------------
constexpr int TMC_THREADS = 256;
constexpr int TMC_MIN_CTAS = 4;                     // resident CTAs per SM the register budget is set for
constexpr int TMC_SMEM_TRIPS = 6144;                // 48 KB of trip PnL per CTA: 4 CTAs fit in the SM's 228 KB
constexpr int TMC_LANES_PER_LAUNCH = 1024;          // lane table passed by value (24 KB of kernel parameters)
constexpr uint32_t TMC_SHUFFLE_BLOCK = 0xFFFFFFFEu; // Philox blocks of the shuffle's round keys: this one and the next
                                                    // (trip / 4 < 2^28: never a bootstrap block)
constexpr int FEISTEL_ROUNDS = 6;                   // with FEISTEL_MIN_HALF: position marginals pass chi-square tests
constexpr int FEISTEL_MIN_HALF = 4;                 // a domain of at least 256: Feistel networks on a few bits are skewed

struct TradeLane {
    double fee;
    int32_t row;       // row of trip_pnl / finals / maxdd
    int32_t T;         // round trips
    uint32_t lane_id;  // Philox counter word 3
    int32_t staged;    // 1: trip PnL staged in shared memory
};

struct TradeMcBatch {
    TradeLane lane[TMC_LANES_PER_LAUNCH];
};

// One trade record: equity, running peak P, smallest equity m since P was set, largest closed-stretch drawdown dd.
__device__ __forceinline__ void equity_record(double x, double& E, double& P, double& m, double& dd) {
    E = __dadd_rn(E, x);
    if (E > P) {                                                        // a new peak needs strict > (:139-144)
        if (m < P) dd = fmax(dd, __ddiv_rn(__dsub_rn(P, m), P));        // the stretch below the old peak ends
        P = E;
        m = E;
    } else {
        m = fmin(m, E);
    }
}

// Balanced Feistel network on 2h bits, FEISTEL_ROUNDS rounds; the round function is a multiply-xorshift hash of (half ^ key)
// whose top h bits are kept.  A bijection of [0, 2^2h) for any keys; cycle-walking restricts it to [0, T).
__device__ __forceinline__ uint32_t feistel(uint32_t v, const uint32_t (&k)[FEISTEL_ROUNDS], int h, uint32_t mask) {
    uint32_t L = v >> h, R = v & mask;
#pragma unroll
    for (int r = 0; r < FEISTEL_ROUNDS; ++r) {
        uint32_t y = (R ^ k[r]) * 0x9E3779B1u;
        y ^= y >> 15;
        y *= 0x85EBCA77u;
        const uint32_t t = L ^ (y >> (32 - h));
        L = R;
        R = t;
    }
    return (L << h) | R;
}

// half width h of the smallest even bit width 2h >= 2 * FEISTEL_MIN_HALF whose range covers [0, T)
__device__ __forceinline__ int feistel_half_bits(int T) {
    const int b = T > 1 ? 32 - __clz(T - 1) : 0;
    return b > 2 * FEISTEL_MIN_HALF ? (b + 1) >> 1 : FEISTEL_MIN_HALF;
}

template <bool STAGED>
__device__ __forceinline__ double trip_at(const double* __restrict__ pnl, int j) {
    return STAGED ? pnl[j] : __ldg(pnl + j);
}

template <bool STAGED>
__device__ __forceinline__ void walk(const double* __restrict__ pnl, const TradeLane& ln, int method, int block_len,
                                     uint64_t seed, uint64_t path_offset, int64_t path, double& E, double& dd) {
    const int T = ln.T;
    const double nfee = -ln.fee;
    double P = E, m = E;
    if (method == 0) {
        // bootstrap: b200bt_mc_bootstrap's block rule on the trip table
        BlockBootstrap boot;
        for (int t0 = 0; t0 < T; t0 += 4) {
            uint32_t x[4];
            philox_path(seed, path_offset, path, (uint32_t)(t0 >> 2), ln.lane_id, x);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (t0 + j < T) {
                    const double p = trip_at<STAGED>(pnl, boot.next(x[j], T, block_len));
                    equity_record(nfee, E, P, m, dd);
                    equity_record(p, E, P, m, dd);
                }
            }
        }
    } else if (T > 0) {
        // shuffle: position j holds trip pi(j), pi = the keyed Feistel bijection cycle-walked into [0, T)
        uint32_t x[8], k[FEISTEL_ROUNDS];
        philox_path(seed, path_offset, path, TMC_SHUFFLE_BLOCK, ln.lane_id, x);
        philox_path(seed, path_offset, path, TMC_SHUFFLE_BLOCK + 1, ln.lane_id, x + 4);
#pragma unroll
        for (int r = 0; r < FEISTEL_ROUNDS; ++r) k[r] = x[r];
        const int h = feistel_half_bits(T);
        const uint32_t mask = (1u << h) - 1u;
        for (int j = 0; j < T; ++j) {
            uint32_t v = (uint32_t)j;
            do {
                v = feistel(v, k, h, mask);
            } while (v >= (uint32_t)T);
            const double p = trip_at<STAGED>(pnl, (int)v);
            equity_record(nfee, E, P, m, dd);
            equity_record(p, E, P, m, dd);
        }
    }
    if (m < P) dd = fmax(dd, __ddiv_rn(__dsub_rn(P, m), P));            // the stretch open at the end of the path
}

// Grid: blocks_per_lane CTAs per lane of the batch, lanes in batch order (heaviest first).
__global__ void __launch_bounds__(TMC_THREADS, TMC_MIN_CTAS)
trade_mc_kernel(const __grid_constant__ TradeMcBatch B, const double* __restrict__ trip_pnl, int64_t ld_trip, int method,
                int block_len, double initial_capital, int64_t n_paths, int blocks_per_lane, uint64_t seed,
                uint64_t path_offset, float* __restrict__ finals, float* __restrict__ maxdd) {
    extern __shared__ double s_pnl[];
    const int slot = (int)(blockIdx.x / (unsigned)blocks_per_lane);
    const int64_t p = (int64_t)(blockIdx.x - (unsigned)slot * (unsigned)blocks_per_lane) * TMC_THREADS + threadIdx.x;
    const TradeLane ln = B.lane[slot];
    const double* src = trip_pnl + (int64_t)ln.row * ld_trip;
    if (ln.staged) {
        for (int i = threadIdx.x; i < ln.T; i += TMC_THREADS) s_pnl[i] = src[i];
        __syncthreads();
    }
    if (p >= n_paths) return;
    double E = initial_capital, dd = 0.0;
    if (ln.staged)
        walk<true>(s_pnl, ln, method, block_len, seed, path_offset, p, E, dd);
    else
        walk<false>(src, ln, method, block_len, seed, path_offset, p, E, dd);
    const int64_t o = (int64_t)ln.row * n_paths + p;
    finals[o] = (float)E;
    maxdd[o] = (float)dd;
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_trade_pnl(const float* price, int64_t ld, int S, int64_t N, const b200bt_individual* indiv, int pop,
                                const b200bt_lane_stats* stats, const uint32_t* events, int64_t event_cap,
                                double* trip_pnl, int64_t ld_trip, int32_t* n_trips, double* fee,
                                b200bt_stream_t stream) {
    B200BT_REQUIRE(trip_pnl && n_trips && fee, B200BT_EINVAL, "trade_pnl: null pointer");
    int rc = check_record_args("trade_pnl", price, ld, S, N, indiv, pop, nullptr, stats, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE(ld_trip >= 1 && 2 * ld_trip >= event_cap, B200BT_EINVAL,
                   "trade_pnl: ld_trip (%lld) must hold event_cap / 2 trips", (long long)ld_trip);
    B200BT_REQUIRE((int64_t)pop * S <= 0x7fffffff, B200BT_ELIMIT, "trade_pnl: at most 2^31 - 1 lanes");
    rc = check_device();
    if (rc) return rc;
    trade_pnl_kernel<<<(unsigned)((int64_t)pop * S), PNL_THREADS, 0, (cudaStream_t)stream>>>(
        price, ld, S, indiv, stats, events, event_cap, trip_pnl, ld_trip, n_trips, fee);
    B200BT_LAUNCH_CHECK("trade_pnl");
    return B200BT_OK;
}

extern "C" int b200bt_trade_mc(const double* trip_pnl, int64_t ld_trip, const int32_t* n_trips_host,
                               const double* fee_host, const uint32_t* lane_ids_host, int L, int method, int block_len,
                               double initial_capital, int64_t n_paths, uint64_t seed, uint64_t path_offset,
                               float* finals, float* maxdd, b200bt_stream_t stream) {
    B200BT_REQUIRE(trip_pnl && n_trips_host && fee_host && finals && maxdd, B200BT_EINVAL, "trade_mc: null pointer");
    B200BT_REQUIRE(L >= 1, B200BT_EINVAL, "trade_mc: need at least one lane (L = %d)", L);
    B200BT_REQUIRE(method == B200BT_TRADE_MC_BOOTSTRAP || method == B200BT_TRADE_MC_SHUFFLE, B200BT_EINVAL,
                   "trade_mc: unknown method %d", method);
    B200BT_REQUIRE(block_len >= 1, B200BT_EINVAL, "trade_mc: block_len must be >= 1 (%d)", block_len);
    B200BT_REQUIRE(n_paths >= 1, B200BT_EINVAL, "trade_mc: n_paths must be >= 1");
    B200BT_REQUIRE(n_paths <= ((int64_t)1 << 38), B200BT_ELIMIT, "trade_mc: n_paths <= 2^38");
    B200BT_REQUIRE(initial_capital > 0.0 && isfinite(initial_capital), B200BT_EINVAL,
                   "trade_mc: initial capital must be positive");
    std::vector<TradeLane> lanes((size_t)L);
    for (int r = 0; r < L; ++r) {
        const int32_t T = n_trips_host[r];
        B200BT_REQUIRE(T >= 0, B200BT_EINVAL, "trade_mc: lane %d has n_trips = %d", r, T);
        B200BT_REQUIRE(T < (1 << 30), B200BT_ELIMIT, "trade_mc: lane %d has %d >= 2^30 trips", r, T);
        B200BT_REQUIRE(T <= ld_trip, B200BT_EINVAL, "trade_mc: lane %d has more trips than ld_trip", r);
        B200BT_REQUIRE(isfinite(fee_host[r]), B200BT_EINVAL, "trade_mc: lane %d fee is not finite", r);
        lanes[r] = TradeLane{fee_host[r], r, T, lane_ids_host ? lane_ids_host[r] : (uint32_t)r, T <= TMC_SMEM_TRIPS};
    }
    int rc = check_device();
    if (rc) return rc;
    // heaviest lanes first: they are dispatched first and the light ones fill the tail of the grid
    std::stable_sort(lanes.begin(), lanes.end(), [](const TradeLane& a, const TradeLane& b) { return a.T > b.T; });
    const int64_t bpl = (n_paths + TMC_THREADS - 1) / TMC_THREADS;
    const int per_launch = (int)std::min<int64_t>(TMC_LANES_PER_LAUNCH, 0x7fffffff / bpl);
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<TradeMcBatch> holder(1);   // 24 KB, off the stack; a launch copies it into its parameters
    TradeMcBatch& batch = holder[0];
    for (int lo = 0; lo < L; lo += per_launch) {
        const int n = std::min(per_launch, L - lo);
        memset(&batch, 0, sizeof(batch));
        int staged_trips = 0;
        for (int i = 0; i < n; ++i) {
            batch.lane[i] = lanes[lo + i];
            if (batch.lane[i].staged) staged_trips = std::max(staged_trips, batch.lane[i].T);
        }
        trade_mc_kernel<<<(unsigned)(n * bpl), TMC_THREADS, (size_t)staged_trips * sizeof(double), st>>>(
            batch, trip_pnl, ld_trip, method, block_len, initial_capital, n_paths, (int)bpl, seed, path_offset, finals,
            maxdd);
        B200BT_LAUNCH_CHECK("trade_mc");
    }
    return B200BT_OK;
}
