// Backtest overfitting of an evolved population (sm_90a): per-day PnL rows of a sweep's records, and the combinatorially
// symmetric cross-validation (CSCV) of Bailey, Borwein, Lopez de Prado and Zhu (2015) on a matrix of such rows.
//
// daily_pnl_kernel  one warp per (individual, symbol) lane walks the lane's event words 32 at a time: coalesced word
//                   loads and the entry word of an exit by shuffle (record_batch), record_pnl as trade_pnl_kernel /
//                   book_kernel price, batch_records' segmented warp sum by calendar day (day_segments), and the open day
//                   carried to the next batch.  Each (lane, day) cell is written once by its warp.
// book_rows_kernel  one thread per (individual, day): the sum over symbols 0..S-1, in that order, of the lane rows.
// cscv_*            moments (one thread per trial), a trial-tile-major combination pass that stages a tile's block
//                   statistics in registers once and walks a run of combinations, a reduction to the selected trial,
//                   and a second tile pass that counts the trials below / tied with the selected one out of sample.
// spa_*             data-snooping tests (White's Reality Check, Hansen's SPA, Romano-Wolf StepM): per-trial moments and
//                   Hansen's stationary-bootstrap variance (one CTA per trial), and the stationary-bootstrap maxima (one
//                   CTA per 32-trial tile x resample range, one warp per resample, one lane per trial).
// Every fp64 operation of the CSCV and SPA paths is an explicit _rn intrinsic: nothing is contracted into an FMA, so
// that tests/cscv_ref.py and tests/spa_ref.py restate the arithmetic bit for bit.
#include <math.h>
#include <algorithm>
#include "philox.cuh"
#include "sweep_dev.cuh"

namespace b200bt {

constexpr int DP_WARPS = 4;                  // lanes per CTA of the row pass
constexpr int CS_THREADS = 256;              // trials per tile of the combination passes
constexpr int CS_WARPS = CS_THREADS / 32;
constexpr int CS_RUN = 64;                   // combinations per shared-memory run of a tile pass
constexpr int CS_MAX_BLOCKS = 20;

// ---- per-day PnL rows ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DP_WARPS * 32)
daily_pnl_kernel(const float* __restrict__ price, int64_t ld_price, int S, const b200bt_individual* __restrict__ indiv,
                 const b200bt_sweep_config cfg, const b200bt_lane_stats* __restrict__ lane_stats,
                 const uint32_t* __restrict__ events, int64_t event_cap, double* __restrict__ lane_pnl, int64_t D,
                 int first_day, int64_t n_lanes) {
    const int lane = threadIdx.x & 31;
    const int64_t w = (int64_t)blockIdx.x * DP_WARPS + (threadIdx.x >> 5);
    if (w >= n_lanes) return;
    double* row = lane_pnl + w * D;
    LaneRecords r;
    if (!read_lane(r, w, S, price, ld_price, indiv, lane_stats, events, event_cap)) {   // lost records: no row
        for (int64_t d = lane; d < D; d += 32) row[d] = NAN;
        return;
    }
    const unsigned gap_bar = cfg.gap_bar > 0 ? (unsigned)cfg.gap_bar : 0xffffffffu;
    const unsigned gap_minutes = (unsigned)cfg.gap_minutes, minute0 = (unsigned)cfg.minute0;
    const unsigned bar_minutes = (unsigned)cfg.bar_minutes;
    int carry_day = -1;                      // open day of the previous batch (-1: none)
    double carry = 0.0;
    for (int64_t base = 0; base < r.n; base += 32) {
        const RecordBatch b = record_batch(r, base);
        const int day = b.active ? (int)record_day(minute0, b.bar, bar_minutes, gap_bar, gap_minutes) : 0x7fffffff;
        bool tail;
        double seg = day_segments(b.pnl, day, b.active, b.n, tail);
        const int batch_first = __shfl_sync(FULL, day, 0);
        if (carry_day >= 0 && carry_day != batch_first && lane == 0) row[carry_day - first_day] = carry;
        if (tail && day == carry_day) seg = __dadd_rn(carry, seg);  // only the first segment can continue the open day
        if (tail && lane != b.n - 1) row[day - first_day] = seg;
        carry = shfl_d(seg, b.n - 1);
        carry_day = __shfl_sync(FULL, day, b.n - 1);
    }
    if (carry_day >= 0 && lane == 0) row[carry_day - first_day] = carry;
}

__global__ void book_rows_kernel(const double* __restrict__ lane_pnl, int S, int64_t D, int64_t n, double* __restrict__ book) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int64_t i = k / D, d = k - i * D;
    const double* p = lane_pnl + i * S * D + d;
    double acc = p[0];
    for (int s = 1; s < S; ++s) acc = __dadd_rn(acc, p[(int64_t)s * D]);
    book[k] = acc;
}

// ---- CSCV -----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int binom(int n, int r) {
    if (r < 0 || r > n) return 0;
    int c = 1;
    for (int i = 1; i <= r; ++i) c = c * (n - r + i) / i;
    return c;
}

// Combination c of itertools.combinations(range(B), B / 2) as a mask g: block b is in the set iff bit B-1-b of g is 0.
// Lexicographic order of the index tuples is decreasing order of their bit-reversed masks, i.e. increasing order of the
// complements g, which is the order of the combinatorial number system: g = sum over its set bits p_i of C(p_i, i).
__device__ __forceinline__ unsigned unrank(int c, int B) {
    unsigned g = 0u;
    for (int i = B / 2, p = B - 1; i >= 1; --i) {
        while (binom(p, i) > c) --p;
        g |= 1u << p;
        c -= binom(p, i);
        --p;
    }
    return g;
}

__device__ __forceinline__ unsigned next_mask(unsigned g) {   // next mask with as many bits (Gosper)
    const unsigned t = g | (g - 1u);
    return (t + 1u) | (((~t & (0u - ~t)) - 1u) >> __ffs(g));
}

// Sharpe of a set of blocks: in-sample (the blocks of combination g) or out-of-sample (its complement).
template <int B>
__device__ __forceinline__ double set_sharpe(const double (&a)[B], const double (&q)[B], unsigned g, bool in_sample,
                                             double mu, double n_set) {
    double A = 0.0, Q = 0.0;
#pragma unroll
    for (int b = 0; b < B; ++b) {
        const bool in = (((g >> (B - 1 - b)) & 1u) == 0u) == in_sample;
        A = __dadd_rn(A, in ? a[b] : 0.0);          // A starts at +0.0: adding +0.0 leaves it bit-identical
        Q = __dadd_rn(Q, in ? q[b] : 0.0);
    }
    const double m = __ddiv_rn(A, n_set);
    const double v = __dsub_rn(__ddiv_rn(Q, n_set), __dmul_rn(m, m));
    return v > 0.0 ? __dmul_rn(__ddiv_rn(__dadd_rn(mu, m), __dsqrt_rn(v)), __dsqrt_rn(252.0)) : 0.0;
}

__device__ __forceinline__ bool key_better(double s, int n, double bs, int bn) { return s > bs || (s == bs && n < bn); }

__global__ void cscv_moments_kernel(const double* __restrict__ pnl, int64_t ld, int N, int64_t r, int B, int64_t L,
                                    double* __restrict__ ab, double* __restrict__ qb, double* __restrict__ mu_out,
                                    double* __restrict__ m2_out, double* __restrict__ m3_out, double* __restrict__ m4_out,
                                    double* __restrict__ sr_out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const double* x = pnl + (int64_t)n * ld + r;
    const int64_t T = (int64_t)B * L;
    double s = 0.0;
    for (int64_t t = 0; t < T; ++t) s = __dadd_rn(s, x[t]);
    const double nt = (double)T;
    const double mu = __ddiv_rn(s, nt);
    double m2 = 0.0, m3 = 0.0, m4 = 0.0;
    for (int b = 0; b < B; ++b) {
        double a = 0.0, q = 0.0;
        for (int64_t t = b * L; t < (b + 1) * L; ++t) {
            const double d = __dsub_rn(x[t], mu), d2 = __dmul_rn(d, d);
            a = __dadd_rn(a, d);
            q = __dadd_rn(q, d2);
            m2 = __dadd_rn(m2, d2);
            m3 = __dadd_rn(m3, __dmul_rn(d2, d));
            m4 = __dadd_rn(m4, __dmul_rn(d2, d2));
        }
        ab[(int64_t)b * N + n] = a;
        qb[(int64_t)b * N + n] = q;
    }
    m2 = __ddiv_rn(m2, nt);
    mu_out[n] = mu;
    m2_out[n] = m2;
    m3_out[n] = __ddiv_rn(m3, nt);
    m4_out[n] = __ddiv_rn(m4, nt);
    sr_out[n] = m2 > 0.0 ? __dmul_rn(__ddiv_rn(mu, __dsqrt_rn(m2)), __dsqrt_rn(252.0)) : 0.0;
}

template <int B>
__device__ __forceinline__ void load_trial(const double* __restrict__ ab, const double* __restrict__ qb, int N, int n,
                                           double (&a)[B], double (&q)[B]) {
#pragma unroll
    for (int b = 0; b < B; ++b) {
        a[b] = n < N ? ab[(int64_t)b * N + n] : 0.0;
        q[b] = n < N ? qb[(int64_t)b * N + n] : 0.0;
    }
}

// Pass 1: per (combination, tile) the in-sample argmax of the tile's trials, key (SR, -n).
template <int B>
__global__ void __launch_bounds__(CS_THREADS)
cscv_select_kernel(const double* __restrict__ ab, const double* __restrict__ qb, const double* __restrict__ mu_in, int N,
                   double n_set, int C, double* __restrict__ part_sr, int* __restrict__ part_n) {
    __shared__ double wsr[CS_WARPS][CS_RUN];
    __shared__ int wn[CS_WARPS][CS_RUN];
    const int tiles = gridDim.x, tile = blockIdx.x;
    const int n = tile * CS_THREADS + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool valid = n < N;
    double a[B], q[B];
    load_trial<B>(ab, qb, N, n, a, q);
    const double mu = valid ? mu_in[n] : 0.0;
    const int runs = (C + CS_RUN - 1) / CS_RUN;
    for (int run = blockIdx.y; run < runs; run += gridDim.y) {
        const int c0 = run * CS_RUN, cnt = min(CS_RUN, C - c0);
        unsigned g = unrank(c0, B);
        for (int k = 0; k < cnt; ++k) {
            double s = valid ? set_sharpe<B>(a, q, g, true, mu, n_set) : -INFINITY;
            int id = valid ? n : 0x7fffffff;
#pragma unroll
            for (int m = 16; m > 0; m >>= 1) {
                const double os = shfl_xor_d(s, m);
                const int on = __shfl_xor_sync(FULL, id, m);
                if (key_better(os, on, s, id)) { s = os; id = on; }
            }
            if (lane == 0) { wsr[warp][k] = s; wn[warp][k] = id; }
            g = next_mask(g);
        }
        __syncthreads();
        if ((int)threadIdx.x < cnt) {
            const int k = threadIdx.x;
            double s = wsr[0][k];
            int id = wn[0][k];
            for (int v = 1; v < CS_WARPS; ++v)
                if (key_better(wsr[v][k], wn[v][k], s, id)) { s = wsr[v][k]; id = wn[v][k]; }
            part_sr[(int64_t)(c0 + k) * tiles + tile] = s;
            part_n[(int64_t)(c0 + k) * tiles + tile] = id;
        }
        __syncthreads();
    }
}

// Pass 2: per combination, the tiles' partials in ascending order (ties stay with the lowest trial), and the selected
// trial's out-of-sample Sharpe.
template <int B>
__global__ void cscv_reduce_kernel(const double* __restrict__ ab, const double* __restrict__ qb, const double* __restrict__ mu_in,
                                   int N, double n_set, int C, int tiles, const double* __restrict__ part_sr,
                                   const int* __restrict__ part_n, int32_t* __restrict__ sel, double* __restrict__ is_sr,
                                   double* __restrict__ oos_sr) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s = part_sr[(int64_t)c * tiles];
    int id = part_n[(int64_t)c * tiles];
    for (int t = 1; t < tiles; ++t) {
        const double ts = part_sr[(int64_t)c * tiles + t];
        const int tn = part_n[(int64_t)c * tiles + t];
        if (key_better(ts, tn, s, id)) { s = ts; id = tn; }
    }
    double a[B], q[B];
    load_trial<B>(ab, qb, N, id, a, q);
    sel[c] = id;
    is_sr[c] = s;
    oos_sr[c] = set_sharpe<B>(a, q, unrank(c, B), false, mu_in[id], n_set);
}

// Pass 3: per combination, trials whose out-of-sample Sharpe is below / equal to the selected trial's (integer counts,
// added with integer atomics: the totals do not depend on the order).
template <int B>
__global__ void __launch_bounds__(CS_THREADS)
cscv_count_kernel(const double* __restrict__ ab, const double* __restrict__ qb, const double* __restrict__ mu_in, int N,
                  double n_set, int C, const int32_t* __restrict__ sel, const double* __restrict__ oos_sr,
                  int32_t* __restrict__ n_below, int32_t* __restrict__ n_tied) {
    __shared__ double o_sr[CS_RUN];
    __shared__ int o_sel[CS_RUN], below[CS_RUN], tied[CS_RUN];
    const int n = blockIdx.x * CS_THREADS + threadIdx.x, lane = threadIdx.x & 31;
    const bool valid = n < N;
    double a[B], q[B];
    load_trial<B>(ab, qb, N, n, a, q);
    const double mu = valid ? mu_in[n] : 0.0;
    const int runs = (C + CS_RUN - 1) / CS_RUN;
    for (int run = blockIdx.y; run < runs; run += gridDim.y) {
        const int c0 = run * CS_RUN, cnt = min(CS_RUN, C - c0);
        if ((int)threadIdx.x < cnt) {
            o_sr[threadIdx.x] = oos_sr[c0 + threadIdx.x];
            o_sel[threadIdx.x] = sel[c0 + threadIdx.x];
            below[threadIdx.x] = 0;
            tied[threadIdx.x] = 0;
        }
        __syncthreads();
        unsigned g = unrank(c0, B);
        for (int k = 0; k < cnt; ++k) {
            const double s = valid ? set_sharpe<B>(a, q, g, false, mu, n_set) : 0.0;
            const unsigned lo = __ballot_sync(FULL, valid && s < o_sr[k]);
            const unsigned eq = __ballot_sync(FULL, valid && n != o_sel[k] && s == o_sr[k]);
            if (lane == 0 && (lo | eq)) {
                atomicAdd(&below[k], __popc(lo));
                atomicAdd(&tied[k], __popc(eq));
            }
            g = next_mask(g);
        }
        __syncthreads();
        if ((int)threadIdx.x < cnt) {
            if (below[threadIdx.x]) atomicAdd(n_below + c0 + threadIdx.x, below[threadIdx.x]);
            if (tied[threadIdx.x]) atomicAdd(n_tied + c0 + threadIdx.x, tied[threadIdx.x]);
        }
        __syncthreads();
    }
}

struct CscvArgs {
    const double* ab;
    const double* qb;
    const double* mu;
    int N, C, tiles;
    double n_set;
    double* part_sr;
    int* part_n;
    int32_t *sel, *n_below, *n_tied;
    double *is_sr, *oos_sr;
};

template <int B>
int cscv_passes(const CscvArgs& A, cudaStream_t st) {
    const int runs = (A.C + CS_RUN - 1) / CS_RUN;
    const unsigned ny = (unsigned)max(1, min(runs, (4 * device_sm_count() + A.tiles - 1) / A.tiles));
    cscv_select_kernel<B><<<dim3((unsigned)A.tiles, ny), CS_THREADS, 0, st>>>(A.ab, A.qb, A.mu, A.N, A.n_set, A.C, A.part_sr,
                                                                               A.part_n);
    B200BT_LAUNCH_CHECK("cscv select");
    cscv_reduce_kernel<B><<<(unsigned)((A.C + 127) / 128), 128, 0, st>>>(A.ab, A.qb, A.mu, A.N, A.n_set, A.C, A.tiles,
                                                                         A.part_sr, A.part_n, A.sel, A.is_sr, A.oos_sr);
    B200BT_LAUNCH_CHECK("cscv reduce");
    cscv_count_kernel<B><<<dim3((unsigned)A.tiles, ny), CS_THREADS, 0, st>>>(A.ab, A.qb, A.mu, A.N, A.n_set, A.C, A.sel,
                                                                              A.oos_sr, A.n_below, A.n_tied);
    B200BT_LAUNCH_CHECK("cscv count");
    return B200BT_OK;
}

int64_t host_binom(int n, int r) {
    int64_t c = 1;
    for (int i = 1; i <= r; ++i) c = c * (n - r + i) / i;
    return c;
}

// workspace: ab, qb [B][N] float64, then per (combination, tile) the argmax partials (float64 SR, int32 trial)
int64_t cscv_layout(int N, int B, int64_t* part_off, int64_t* n_part) {
    const int64_t tiles = (N + CS_THREADS - 1) / CS_THREADS;
    const int64_t parts = host_binom(B, B / 2) * tiles;
    const int64_t stats = 2 * (int64_t)B * N * 8;
    if (part_off) *part_off = stats;
    if (n_part) *n_part = parts;
    return stats + parts * 12;
}

// ---- data snooping: Reality Check, SPA, StepM -----------------------------------------------------------------------
constexpr int SPA_MAX_T = 8192;              // 13-bit day indices
constexpr int SPA_MAX_STATS = 8;
constexpr int SPA_MOM_THREADS = 256;
constexpr int SPA_WARPS = 16;                // resamples walked at once per CTA of the bootstrap pass
constexpr int SPA_TILE = 32;                 // trials per CTA of the bootstrap pass: one per lane
constexpr int SPA_STAGE_T = 768;             // rows of up to this many days are staged in shared memory (192 KB)

// Moments of trial k (one CTA): the row, then (1-q)^i by running products and the mean (one thread each, ascending),
// the lag sums (threads over lags, each in ascending t), and the kappa-weighted sum of the lags (one thread, ascending).
__global__ void __launch_bounds__(SPA_MOM_THREADS)
spa_moments_kernel(const double* __restrict__ d, int64_t ld, int T, double q, double* __restrict__ mean_out,
                   double* __restrict__ omega2_out) {
    extern __shared__ double sm[];
    double* c = sm;                          // [T] the row, then the row minus its mean
    double* p = sm + T;                      // [T + 1] (1-q)^i
    double* g = p + T + 1;                   // [T] gamma_0, then kappa_i * gamma_i
    __shared__ double mean_s;
    const double* x = d + (int64_t)blockIdx.x * ld;
    for (int t = threadIdx.x; t < T; t += blockDim.x) c[t] = x[t];
    __syncthreads();
    const double nt = (double)T;
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int t = 0; t < T; ++t) s = __dadd_rn(s, c[t]);
        mean_s = __ddiv_rn(s, nt);
    } else if (threadIdx.x == 32) {
        const double a = __dsub_rn(1.0, q);
        double r = 1.0;
        p[0] = r;
        for (int i = 1; i <= T; ++i) p[i] = r = __dmul_rn(r, a);
    }
    __syncthreads();
    const double mu = mean_s;
    for (int t = threadIdx.x; t < T; t += blockDim.x) c[t] = __dsub_rn(c[t], mu);
    __syncthreads();
    for (int i = threadIdx.x; i < T; i += blockDim.x) {
        double s = 0.0;
        for (int t = 0; t + i < T; ++t) s = __dadd_rn(s, __dmul_rn(c[t], c[t + i]));
        const double gam = __ddiv_rn(s, nt);
        if (i == 0) {
            g[0] = gam;
        } else {
            const double kappa = __dadd_rn(__dmul_rn(__ddiv_rn((double)(T - i), nt), p[i]),
                                           __dmul_rn(__ddiv_rn((double)i, nt), p[T - i]));
            g[i] = __dmul_rn(kappa, gam);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 1; i < T; ++i) s = __dadd_rn(s, g[i]);
        mean_out[blockIdx.x] = mu;
        omega2_out[blockIdx.x] = __dadd_rn(g[0], __dmul_rn(2.0, s));
    }
}

// Unsigned image of a double whose order is the numeric order (-inf lowest), for the cross-CTA atomicMax.
__device__ __forceinline__ unsigned long long ordered(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

__device__ __forceinline__ double unordered(unsigned long long o) {
    return __longlong_as_double((long long)((o >> 63) ? (o & 0x7fffffffffffffffull) : ~o));
}

// Days 64w + 2*lane and 64w + 2*lane + 1 of the resample whose Philox key is (k0, k1) and counter words 0, 1 are
// (c0, c1), packed as theta0 | theta1 << 16.  A block start on day t with index s has the key (t + 1) << 13 | s, so the
// latest start at or before a day is a max-scan of keys; `carry` holds the latest start before the window and is
// advanced past it.  Days >= T get unspecified values.
__device__ __forceinline__ unsigned spa_window(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, int w, int T,
                                               uint64_t q32, int& carry) {
    const int lane = threadIdx.x & 31;
    const int t0 = 64 * w + 2 * lane, t1 = t0 + 1;
    uint32_t x[4];
    philox4x32_10(c0, c1, (uint32_t)(32 * w + lane), 0u, k0, k1, x);
    const bool st0 = t0 == 0 || (uint64_t)x[0] < q32;
    const bool st1 = (uint64_t)x[2] < q32;
    const int s0 = (int)__umulhi(x[1], (uint32_t)T), s1 = (int)__umulhi(x[3], (uint32_t)T);
    int inc = st1 ? ((t1 + 1) << 13 | s1) : st0 ? ((t0 + 1) << 13 | s0) : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc = max(inc, v);
    }
    int prev = __shfl_up_sync(FULL, inc, 1);
    prev = max(lane == 0 ? 0 : prev, carry);
    carry = max(carry, __shfl_sync(FULL, inc, 31));
    const int ls = prev & 8191, lt = (prev >> 13) - 1;
    int th0 = s0, th1;
    if (!st0) {
        th0 = ls + (t0 - lt);
        th0 = th0 >= T ? th0 - T : th0;
    }
    if (st1) {
        th1 = s1;
    } else {
        th1 = th0 + 1;
        th1 = th1 >= T ? th1 - T : th1;
    }
    return (unsigned)(th0 & 0xffff) | (unsigned)(th1 & 0xffff) << 16;
}

// m* of one resample for the lane's trial: (sum_t row[theta(t)]) / T in ascending t.  The warp walks the resample's
// index stream 64 days at a time (spa_window) and every lane gathers its own row: from the tile's [t][32] shared-memory
// stage xs (STAGED; every lane of the warp reads the same day, so no bank conflicts) or through L1/L2 from `row`.
// Called by the SPA maxima and the MCS bootstrap means, so both see the same m*.
template <bool STAGED>
__device__ __forceinline__ double spa_gather_mean(const double* __restrict__ xs, const double* __restrict__ row,
                                                  uint32_t key0, uint32_t key1, uint64_t gid, int T, uint64_t q32) {
    const int lane = threadIdx.x & 31;
    const int windows = (T + 63) / 64;
    int carry = 0;
    double acc = 0.0;
    for (int w = 0; w < windows; ++w) {
        const unsigned packed = spa_window(key0, key1, (uint32_t)gid, (uint32_t)(gid >> 32), w, T, q32, carry);
        const int nd = min(64, T - 64 * w);
#pragma unroll 4
        for (int pr = 0; pr < 32; ++pr) {
            if (2 * pr >= nd) break;
            const unsigned v = __shfl_sync(FULL, packed, pr);
            const int a = (int)(v & 0xffffu), e = (int)(v >> 16);
            acc = __dadd_rn(acc, STAGED ? xs[a * SPA_TILE + lane] : __ldg(row + a));
            if (2 * pr + 1 < nd) acc = __dadd_rn(acc, STAGED ? xs[e * SPA_TILE + lane] : __ldg(row + e));
        }
    }
    return __ddiv_rn(acc, (double)T);
}

// Stage trials [k0, k0 + 32) of d as [t][32] in shared memory (zeros past N).
__device__ __forceinline__ void spa_stage_tile(double* __restrict__ xs, const double* __restrict__ d, int64_t ld, int N,
                                               int T, int64_t k0) {
    for (int i = threadIdx.x; i < SPA_TILE * T; i += blockDim.x) {
        const int j = i & (SPA_TILE - 1), t = i / SPA_TILE;
        xs[i] = k0 + j < N ? d[(k0 + j) * ld + t] : 0.0;
    }
    __syncthreads();
}

// One CTA: trials [32 * blockIdx.x, +32) x resamples [b_lo, b_hi) of this CTA's range; warp v walks resamples b_lo + v,
// b_lo + v + SPA_WARPS, ...  STAGED: the tile's rows sit in shared memory as [t][32]; otherwise each lane reads its row
// through L1/L2.
template <bool STAGED>
__global__ void __launch_bounds__(SPA_WARPS * 32)
spa_bootstrap_kernel(const double* __restrict__ d, int64_t ld, int N, int T, uint64_t q32, int64_t n_boot, int64_t per_cta,
                     uint64_t seed, uint64_t boot_offset, int n_stats, const double* __restrict__ shift,
                     const double* __restrict__ scale, unsigned long long* __restrict__ out) {
    extern __shared__ double xs[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t k0 = (int64_t)blockIdx.x * SPA_TILE;
    const int64_t k = k0 + lane;
    const bool valid = k < N;
    if (STAGED) spa_stage_tile(xs, d, ld, N, T, k0);
    const double* row = d + (valid ? k : (int64_t)N - 1) * ld;
    double sh[SPA_MAX_STATS], sc[SPA_MAX_STATS];
#pragma unroll
    for (int j = 0; j < SPA_MAX_STATS; ++j) {
        sh[j] = valid && j < n_stats ? shift[(int64_t)j * N + k] : INFINITY;
        sc[j] = valid && j < n_stats ? scale[(int64_t)j * N + k] : 0.0;
    }
    const uint32_t key0 = (uint32_t)seed, key1 = (uint32_t)(seed >> 32);
    const int64_t b_lo = (int64_t)blockIdx.y * per_cta, b_hi = min(n_boot, b_lo + per_cta);
    for (int64_t b = b_lo + warp; b < b_hi; b += SPA_WARPS) {
        const double m = spa_gather_mean<STAGED>(xs, row, key0, key1, boot_offset + (uint64_t)b, T, q32);
        for (int j = 0; j < n_stats; ++j) {
            double v = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < SPA_MAX_STATS; ++jj)
                if (jj == j && sh[jj] != INFINITY) v = __dmul_rn(__dsub_rn(m, sh[jj]), sc[jj]);
            v = warp_max_d(v);                               // fmax: NaN values drop out
            if (lane == 0 && !isnan(v)) atomicMax(out + (int64_t)j * n_boot + b, ordered(v));
        }
    }
}

__global__ void spa_fill_kernel(unsigned long long* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = ordered(-INFINITY);
}

__global__ void spa_decode_kernel(unsigned long long* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) reinterpret_cast<double*>(out)[i] = unordered(out[i]);
}

static int spa_check(const double* d, int64_t ld, int N, int T, const char* fn) {
    B200BT_REQUIRE(d, B200BT_EINVAL, "%s: null pointer", fn);
    B200BT_REQUIRE(N >= 1, B200BT_EINVAL, "%s: need at least 1 trial (N = %d)", fn, N);
    B200BT_REQUIRE(T >= 2, B200BT_EINVAL, "%s: need at least 2 days (T = %d)", fn, T);
    B200BT_REQUIRE(T <= SPA_MAX_T, B200BT_ELIMIT, "%s: at most %d days (T = %d)", fn, SPA_MAX_T, T);
    B200BT_REQUIRE(ld >= T, B200BT_EINVAL, "%s: row stride %lld below T = %d", fn, (long long)ld, T);
    return B200BT_OK;
}

// ---- model confidence set ---------------------------------------------------------------------------------------------
constexpr int MCS_MAX_N = 16384;
constexpr int MCS_TILE = 64;                 // pairwise and range-maxima tiles: 64 x 64 cells, 4 x 4 per thread
constexpr int MCS_CHUNK = 16;                // resamples (pairwise) or columns (range maxima) staged per step
constexpr int MCS_THREADS = 256;
constexpr int MCS_ORDER_THREADS = 1024;

// Bootstrap means: spa_bootstrap_kernel's schedule, writing m* (minus center[k] when given) at out[b][k].
template <bool STAGED>
__global__ void __launch_bounds__(SPA_WARPS * 32)
boot_means_kernel(const double* __restrict__ d, int64_t ld, int N, int T, uint64_t q32, int64_t n_boot, int64_t per_cta,
                  uint64_t seed, uint64_t boot_offset, const double* __restrict__ center, double* __restrict__ out,
                  int64_t ld_out) {
    extern __shared__ double xs[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t k0 = (int64_t)blockIdx.x * SPA_TILE;
    const int64_t k = k0 + lane;
    const bool valid = k < N;
    if (STAGED) spa_stage_tile(xs, d, ld, N, T, k0);
    const double* row = d + (valid ? k : (int64_t)N - 1) * ld;
    const double c = center && valid ? center[k] : 0.0;
    const uint32_t key0 = (uint32_t)seed, key1 = (uint32_t)(seed >> 32);
    const int64_t b_lo = (int64_t)blockIdx.y * per_cta, b_hi = min(n_boot, b_lo + per_cta);
    for (int64_t b = b_lo + warp; b < b_hi; b += SPA_WARPS) {
        const double m = spa_gather_mean<STAGED>(xs, row, key0, key1, boot_offset + (uint64_t)b, T, q32);
        if (valid) out[b * ld_out + k] = center ? __dsub_rn(m, c) : m;
    }
}

// Autocovariances of row blockIdx.x: spa_moments_kernel's mean and gamma_i for i = 0..K.
__global__ void __launch_bounds__(SPA_MOM_THREADS)
autocov_kernel(const double* __restrict__ d, int64_t ld, int T, int K, double* __restrict__ out,
               double* __restrict__ mean_out) {
    extern __shared__ double c[];
    __shared__ double mean_s;
    const double* x = d + (int64_t)blockIdx.x * ld;
    for (int t = threadIdx.x; t < T; t += blockDim.x) c[t] = x[t];
    __syncthreads();
    const double nt = (double)T;
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int t = 0; t < T; ++t) s = __dadd_rn(s, c[t]);
        mean_s = __ddiv_rn(s, nt);
    }
    __syncthreads();
    const double mu = mean_s;
    for (int t = threadIdx.x; t < T; t += blockDim.x) c[t] = __dsub_rn(c[t], mu);
    __syncthreads();
    for (int i = threadIdx.x; i <= K; i += blockDim.x) {
        double s = 0.0;
        for (int t = 0; t + i < T; ++t) s = __dadd_rn(s, __dmul_rn(c[t], c[t + i]));
        out[(int64_t)blockIdx.x * (K + 1) + i] = __ddiv_rn(s, nt);
    }
    if (mean_out && threadIdx.x == 0) mean_out[blockIdx.x] = mu;
}

// Pairwise pass: s2[i][j] += sum over this launch's resamples b (ascending) of (z[b][j] - z[b][i])^2, for i < j only.
// One CTA per upper-triangle (i-tile, j-tile) pair; MCS_CHUNK resample rows of both tiles are staged in shared memory
// and each thread keeps a 4 x 4 register tile of accumulators (rows ty + 16a, columns tx + 16c).
__global__ void __launch_bounds__(MCS_THREADS, 1)
mcs_pairwise_kernel(const double* __restrict__ z, int64_t ld_z, int N, int64_t n_boot, int tiles,
                    double* __restrict__ s2) {
    __shared__ double zi[MCS_CHUNK][MCS_TILE], zj[MCS_CHUNK][MCS_TILE];
    int p = blockIdx.x, ti = 0;                   // upper-triangle pair p -> (ti, tj), tj >= ti
    while (p >= tiles - ti) { p -= tiles - ti; ++ti; }
    const int tj = ti + p;
    const int i0 = ti * MCS_TILE, j0 = tj * MCS_TILE;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * c;
            acc[a][c] = (i < j && j < N) ? s2[(int64_t)i * N + j] : 0.0;
        }
    for (int64_t b0 = 0; b0 < n_boot; b0 += MCS_CHUNK) {
        const int nb = (int)min((int64_t)MCS_CHUNK, n_boot - b0);
        for (int e = threadIdx.x; e < MCS_CHUNK * MCS_TILE; e += MCS_THREADS) {
            const int r = e / MCS_TILE, col = e % MCS_TILE;
            const bool in = r < nb;
            const double* zr = z + (b0 + r) * ld_z;
            zi[r][col] = in && i0 + col < N ? zr[i0 + col] : 0.0;
            zj[r][col] = in && j0 + col < N ? zr[j0 + col] : 0.0;
        }
        __syncthreads();
        for (int r = 0; r < nb; ++r) {
            double a4[4], c4[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) a4[a] = zi[r][ty + 16 * a];
#pragma unroll
            for (int c = 0; c < 4; ++c) c4[c] = zj[r][tx + 16 * c];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const double df = __dsub_rn(c4[c], a4[a]);
                    acc[a][c] = __dadd_rn(acc[a][c], __dmul_rn(df, df));
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * c;
            if (i < j && j < N) s2[(int64_t)i * N + j] = acc[a][c];
        }
}

// t for a mean difference dm over a standard deviation s, with the zero-variance rule.
__device__ __forceinline__ double mcs_t(double dm, double s) {
    if (s > 0.0) return __ddiv_rn(dm, s);
    return dm == 0.0 ? 0.0 : (dm > 0.0 ? INFINITY : -INFINITY);
}

// w: s2 (upper triangle) in, rho out (symmetric, zero diagonal); t[i][j] = (mean_j - mean_i) / sigma_ij.
__global__ void mcs_range_stats_kernel(const double* __restrict__ mean, int N, double nb, double* __restrict__ w,
                                       double* __restrict__ t) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)N * N) return;
    const int i = (int)(e / N), j = (int)(e - (int64_t)i * N);
    if (i == j) {
        w[e] = 0.0;
        t[e] = 0.0;
    }
    if (i >= j) return;
    const double sigma = __dsqrt_rn(__ddiv_rn(w[e], nb));
    const double rho = sigma > 0.0 ? __ddiv_rn(1.0, sigma) : 0.0;
    w[e] = rho;
    w[(int64_t)j * N + i] = rho;
    t[e] = mcs_t(__dsub_rn(mean[j], mean[i]), sigma);
    t[(int64_t)j * N + i] = mcs_t(__dsub_rn(mean[i], mean[j]), sigma);
}

__device__ __forceinline__ bool mcs_better(double v, int i, double bv, int bi) { return v > bv || (v == bv && i < bi); }

// Warp-wide (max, lowest index) of row i of t over the live columns.
__device__ __forceinline__ void mcs_row_max(const double* __restrict__ t, int N, int i, const unsigned char* alive,
                                            double& v, int& col) {
    const int lane = threadIdx.x & 31;
    v = -INFINITY;
    col = 0x7fffffff;
    const double* row = t + (int64_t)i * N;
    for (int j = lane; j < N; j += 32)
        if (alive[j] && mcs_better(row[j], j, v, col)) { v = row[j]; col = j; }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
        const double ov = shfl_xor_d(v, m);
        const int oc = __shfl_xor_sync(FULL, col, m);
        if (mcs_better(ov, oc, v, col)) { v = ov; col = oc; }
    }
}

// T_R elimination order in one CTA: each live row keeps its max over the live columns and that column; after e leaves,
// only the rows whose column was e are rescanned (a warp per row).  Shared memory: rm [N] doubles, col [N] ints,
// alive [N] bytes.
__global__ void __launch_bounds__(MCS_ORDER_THREADS)
mcs_range_order_kernel(const double* __restrict__ t, int N, int32_t* __restrict__ order, double* __restrict__ stat) {
    extern __shared__ double rm[];
    int* col = reinterpret_cast<int*>(rm + N);
    unsigned char* alive = reinterpret_cast<unsigned char*>(col + N);
    __shared__ double red_v[MCS_ORDER_THREADS / 32];
    __shared__ int red_i[MCS_ORDER_THREADS / 32];
    __shared__ int e_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = MCS_ORDER_THREADS / 32;
    for (int i = threadIdx.x; i < N; i += blockDim.x) alive[i] = 1;
    __syncthreads();
    for (int i = warp; i < N; i += warps) {
        double v;
        int c;
        mcs_row_max(t, N, i, alive, v, c);
        if (lane == 0) { rm[i] = v; col[i] = c; }
    }
    __syncthreads();
    for (int k = 0; k + 1 < N; ++k) {
        double v = -INFINITY;
        int bi = 0x7fffffff;
        for (int i = threadIdx.x; i < N; i += blockDim.x)
            if (alive[i] && mcs_better(rm[i], i, v, bi)) { v = rm[i]; bi = i; }
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) {
            const double ov = shfl_xor_d(v, m);
            const int oi = __shfl_xor_sync(FULL, bi, m);
            if (mcs_better(ov, oi, v, bi)) { v = ov; bi = oi; }
        }
        if (lane == 0) { red_v[warp] = v; red_i[warp] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < warps; ++w)
                if (mcs_better(red_v[w], red_i[w], v, bi)) { v = red_v[w]; bi = red_i[w]; }
            order[k] = bi;
            stat[k] = v;
            alive[bi] = 0;
            e_s = bi;
        }
        __syncthreads();
        const int e = e_s;
        for (int i = warp; i < N; i += warps)
            if (alive[i] && col[i] == e) {
                double rv;
                int c;
                mcs_row_max(t, N, i, alive, rv, c);
                if (lane == 0) { rm[i] = rv; col[i] = c; }
            }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < N; i += blockDim.x)
        if (alive[i]) order[N - 1] = i;
}

// rho in elimination-rank order, strictly upper triangular: out[r][c] = rho[order[r]][order[c]] for c > r, else 0.
__global__ void mcs_rank_rho_kernel(const double* __restrict__ rho, const int32_t* __restrict__ order, int N,
                                   double* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)N * N) return;
    const int r = (int)(e / N), c = (int)(e - (int64_t)r * N);
    out[e] = c > r ? rho[(int64_t)order[r] * N + order[c]] : 0.0;
}

// Range maxima: R[b][r] = max over c of |z[b][order[c]] - z[b][order[r]]| * rho_rank[r][c] (0 below the diagonal), for
// a 64-resample x 64-rank tile per CTA (4 x 4 per thread), columns staged MCS_CHUNK at a time; column chunks wholly at
// or below the tile's first rank are skipped.
__global__ void __launch_bounds__(MCS_THREADS, 1)
mcs_range_boot_kernel(const double* __restrict__ z, int64_t ld_z, int N, int64_t n_boot, const int32_t* __restrict__ order,
                      const double* __restrict__ rho_rank, double* __restrict__ R) {
    __shared__ double zc[MCS_TILE][MCS_CHUNK + 1], pc[MCS_TILE][MCS_CHUNK + 1];
    const int64_t b0 = (int64_t)blockIdx.y * MCS_TILE;
    const int r0 = blockIdx.x * MCS_TILE;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;     // ranks r0 + tx + 16c, resamples b0 + ty + 16a
    double own[4][4], mx[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int64_t b = b0 + ty + 16 * a;
            const int r = r0 + tx + 16 * c;
            own[a][c] = b < n_boot && r < N ? z[b * ld_z + order[r]] : 0.0;
            mx[a][c] = 0.0;
        }
    for (int c0 = (r0 / MCS_CHUNK) * MCS_CHUNK; c0 < N; c0 += MCS_CHUNK) {
        for (int e = threadIdx.x; e < MCS_TILE * MCS_CHUNK; e += MCS_THREADS) {
            const int row = e / MCS_CHUNK, cc = e % MCS_CHUNK, cg = c0 + cc;
            const int64_t b = b0 + row;
            zc[row][cc] = b < n_boot && cg < N ? z[b * ld_z + order[cg]] : 0.0;
            pc[row][cc] = r0 + row < N && cg < N ? rho_rank[(int64_t)(r0 + row) * N + cg] : 0.0;
        }
        __syncthreads();
#pragma unroll 4
        for (int cc = 0; cc < MCS_CHUNK; ++cc) {
            double zb[4], pr[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) zb[a] = zc[ty + 16 * a][cc];
#pragma unroll
            for (int c = 0; c < 4; ++c) pr[c] = pc[tx + 16 * c][cc];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    mx[a][c] = fmax(mx[a][c], __dmul_rn(fabs(__dsub_rn(zb[a], own[a][c])), pr[c]));
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int64_t b = b0 + ty + 16 * a;
            const int r = r0 + tx + 16 * c;
            if (b < n_boot && r < N) R[b * N + r] = mx[a][c];
        }
}

// count[k] += #{b : max over r >= k of R[b][r] >= stat[k]}, k = 0..N-2: a warp per resample walks the ranks from the top
// 32 at a time with a suffix-max scan; counts gather in shared memory (N ints) and go out once per CTA.
__global__ void __launch_bounds__(MCS_THREADS)
mcs_range_count_kernel(const double* __restrict__ R, int N, int64_t n_boot, const double* __restrict__ stat,
                       unsigned long long* __restrict__ count) {
    extern __shared__ int cnt[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = MCS_THREADS / 32;
    for (int k = threadIdx.x; k < N; k += blockDim.x) cnt[k] = 0;
    __syncthreads();
    for (int64_t b = (int64_t)blockIdx.x * warps + warp; b < n_boot; b += (int64_t)gridDim.x * warps) {
        const double* row = R + b * N;
        double carry = 0.0;
        for (int top = N; top > 0; top -= 32) {
            const int r = top - 32 + lane;
            double v = r >= 0 ? row[r] : 0.0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double u = __shfl_down_sync(FULL, v, o);
                if (lane + o < 32) v = fmax(v, u);
            }
            v = fmax(v, carry);
            carry = __shfl_sync(FULL, v, 0);
            if (r >= 0 && r + 1 < N && v >= stat[r]) atomicAdd(&cnt[r], 1);
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k + 1 < N; k += blockDim.x)
        if (cnt[k]) atomicAdd(count + k, (unsigned long long)cnt[k]);
}

// ---- T_max step loop.  Workspace: zbar [B] doubles, s [N] doubles, tv [N] doubles, xbar_M (1 double), two [N] int lists
// of the live models in ascending index, the eliminated model (1 int).
struct McsMaxWs {
    double *zbar, *s, *tv, *xm;
    int *list0, *list1, *e;
};

__host__ __device__ inline int64_t mcs_max_ws_layout(int N, int64_t B, McsMaxWs* w, char* base) {
    const int64_t zb = 0, s = zb + 8 * B, tv = s + 8 * (int64_t)N, xm = tv + 8 * (int64_t)N, l0 = xm + 8,
                  l1 = l0 + 4 * (int64_t)N, e = l1 + 4 * (int64_t)N, end = e + 4;
    if (w) {
        w->zbar = (double*)(base + zb);
        w->s = (double*)(base + s);
        w->tv = (double*)(base + tv);
        w->xm = (double*)(base + xm);
        w->list0 = (int*)(base + l0);
        w->list1 = (int*)(base + l1);
        w->e = (int*)(base + e);
    }
    return end;
}

// list = 0..N-1, xbar_M = (sum of mean ascending) / N.
__global__ void mcs_max_init_kernel(const double* __restrict__ mean, int N, McsMaxWs w) {
    for (int i = threadIdx.x; i < N; i += blockDim.x) w.list0[i] = i;
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < N; ++i) s = __dadd_rn(s, mean[i]);
        *w.xm = __ddiv_rn(s, (double)N);
        *w.e = -1;
    }
}

// One thread per resample over the m live models `list` (ascending).  With `stat` (step k): T*_b(M_k) = max over i of
// (zbar_b - z_bi) / s_i (0 where s_i = 0), counted into *count when >= *stat.  Then zbar_b of the set without *e (all
// of `list` when *e < 0): the sum of z_bj over the kept j, ascending, over their number.
constexpr int MCS_ROWS_THREADS = 64;         // T_max passes: small CTAs, so that B = 10^4 resamples or ~10^3 models
constexpr int MCS_VAR_THREADS = 32;          // spread over every SM rather than a few

__global__ void __launch_bounds__(MCS_ROWS_THREADS)
mcs_max_rows_kernel(const double* __restrict__ z, int64_t ld_z, int64_t n_boot, const int* __restrict__ list, int m,
                    McsMaxWs w, const double* __restrict__ stat, unsigned long long* __restrict__ count) {
    __shared__ int red[MCS_ROWS_THREADS / 32];
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int e = *w.e;
    bool hit = false;
    if (b < n_boot) {
        const double* row = z + b * ld_z;
        const double zb = w.zbar[b];
        double acc = 0.0, mx = -INFINITY;
        for (int p = 0; p < m; ++p) {
            const int j = list[p];
            const double v = row[j];
            if (stat) {
                const double sj = w.s[j];
                mx = fmax(mx, sj > 0.0 ? __ddiv_rn(__dsub_rn(zb, v), sj) : 0.0);
            }
            if (j != e) acc = __dadd_rn(acc, v);
        }
        w.zbar[b] = __ddiv_rn(acc, (double)(e >= 0 ? m - 1 : m));
        hit = stat && mx >= *stat;
    }
    if (!stat) return;
    const unsigned bal = __ballot_sync(FULL, hit);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int v = 0; v < MCS_ROWS_THREADS / 32; ++v) s += red[v];
        if (s) atomicAdd(count, (unsigned long long)s);
    }
}

// One thread per live model i = list[p]: v_i = (sum over b ascending of (zbar_b - z_bi)^2) / B, s_i = sqrt(v_i),
// t_i = (xbar_M - mean_i) / s_i with the zero-variance rule.
__global__ void __launch_bounds__(MCS_VAR_THREADS)
mcs_max_var_kernel(const double* __restrict__ z, int64_t ld_z, int64_t n_boot, const int* __restrict__ list, int m,
                   const double* __restrict__ mean, McsMaxWs w) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const int i = list[p];
    double acc = 0.0;
#pragma unroll 8
    for (int64_t b = 0; b < n_boot; ++b) {
        const double df = __dsub_rn(w.zbar[b], z[b * ld_z + i]);
        acc = __dadd_rn(acc, __dmul_rn(df, df));
    }
    const double s = __dsqrt_rn(__ddiv_rn(acc, (double)n_boot));
    w.s[i] = s;
    w.tv[i] = mcs_t(__dsub_rn(*w.xm, mean[i]), s);
}

// Step k in one CTA: e = argmax of t over `list` (lowest index on ties), order[k], stat[k]; `next` = list without e;
// xbar_M of `next`.
__global__ void __launch_bounds__(MCS_ORDER_THREADS)
mcs_max_step_kernel(const int* __restrict__ list, int m, const double* __restrict__ mean, McsMaxWs w, int k,
                    int* __restrict__ next, int32_t* __restrict__ order, double* __restrict__ stat) {
    __shared__ double red_v[MCS_ORDER_THREADS / 32];
    __shared__ int red_i[MCS_ORDER_THREADS / 32];
    __shared__ int e_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double v = -INFINITY;
    int bi = 0x7fffffff;
    for (int p = threadIdx.x; p < m; p += blockDim.x) {
        const int i = list[p];
        if (mcs_better(w.tv[i], i, v, bi)) { v = w.tv[i]; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = shfl_xor_d(v, o);
        const int oi = __shfl_xor_sync(FULL, bi, o);
        if (mcs_better(ov, oi, v, bi)) { v = ov; bi = oi; }
    }
    if (lane == 0) { red_v[warp] = v; red_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int u = 1; u < MCS_ORDER_THREADS / 32; ++u)
            if (mcs_better(red_v[u], red_i[u], v, bi)) { v = red_v[u]; bi = red_i[u]; }
        order[k] = bi;
        stat[k] = v;
        *w.e = bi;
        e_s = bi;
    }
    __syncthreads();
    const int e = e_s;
    for (int p = threadIdx.x; p < m; p += blockDim.x) {
        const int i = list[p];
        if (i < e) next[p] = i;
        else if (i > e) next[p - 1] = i;
    }
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int p = 0; p < m; ++p)
            if (list[p] != e) s = __dadd_rn(s, mean[list[p]]);
        *w.xm = __ddiv_rn(s, (double)(m - 1));
        if (m == 2) order[k + 1] = list[0] == e ? list[1] : list[0];
    }
}

static int mcs_check_n(int N, const char* fn) {
    B200BT_REQUIRE(N >= 2, B200BT_EINVAL, "%s: need at least 2 models (N = %d)", fn, N);
    B200BT_REQUIRE(N <= MCS_MAX_N, B200BT_ELIMIT, "%s: at most %d models (N = %d)", fn, MCS_MAX_N, N);
    return B200BT_OK;
}

static int mcs_check_budget(int64_t need_or_neg, int64_t max_bytes, const char* fn) {
    B200BT_REQUIRE(need_or_neg >= 0 && need_or_neg <= max_bytes, B200BT_ELIMIT,
                   "%s: %lld bytes of [B][N] / [N][N] buffers exceed the budget of %lld", fn, (long long)need_or_neg,
                   (long long)max_bytes);
    return B200BT_OK;
}

// a * b * 8 bytes, or -1 when it does not fit int64
static int64_t mcs_bytes(int64_t a, int64_t b) {
    if (a < 0 || b < 0 || (b > 0 && a > (INT64_MAX / 8) / b)) return -1;
    return a * b * 8;
}

static int64_t mcs_sum(int64_t a, int64_t b) { return a < 0 || b < 0 || a > INT64_MAX - b ? -1 : a + b; }

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_daily_pnl(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv,
                                int pop, const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats,
                                const uint32_t* events, int64_t event_cap, double* lane_pnl, int64_t D,
                                double* book_pnl_or_null, b200bt_stream_t stream) {
    B200BT_REQUIRE(cfg && lane_pnl, B200BT_EINVAL, "daily_pnl: null pointer");
    int rc = check_record_args("daily_pnl", price, ld_price, S, N, indiv, pop, cfg, lane_stats, events, event_cap);
    if (rc) return rc;
    // calendar days of bar 0 and bar N - 1 (the kernels' unsigned 32-bit expression; the clock check keeps it exact)
    const int64_t last = N - 1;
    const int64_t gap = (cfg->gap_bar > 0 && last >= cfg->gap_bar) ? cfg->gap_minutes : 0;
    const int64_t first_day = cfg->minute0 / 1440;
    const int64_t span = (cfg->minute0 + last * cfg->bar_minutes + gap) / 1440 - first_day + 1;
    B200BT_REQUIRE(D >= span, B200BT_EINVAL, "daily_pnl: D = %lld columns do not cover the %lld calendar days of the series",
                   (long long)D, (long long)span);
    B200BT_REQUIRE((int64_t)pop * S <= INT64_MAX / D, B200BT_ELIMIT, "daily_pnl: pop * S * D must fit int64");
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t lanes = (int64_t)pop * S;
    rc = cuda_status(cudaMemsetAsync(lane_pnl, 0, (size_t)(lanes * D) * sizeof(double), st), "daily_pnl memset");
    if (rc) return rc;
    daily_pnl_kernel<<<(unsigned)((lanes + DP_WARPS - 1) / DP_WARPS), DP_WARPS * 32, 0, st>>>(
        price, ld_price, S, indiv, *cfg, lane_stats, events, event_cap, lane_pnl, D, (int)first_day, lanes);
    B200BT_LAUNCH_CHECK("daily_pnl");
    if (book_pnl_or_null) {
        const int64_t n = (int64_t)pop * D;
        book_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(lane_pnl, S, D, n, book_pnl_or_null);
        B200BT_LAUNCH_CHECK("daily_pnl book rows");
    }
    return B200BT_OK;
}

static int cscv_check(int N, int64_t T, int B) {
    B200BT_REQUIRE(N >= 2, B200BT_EINVAL, "cscv: need at least 2 trials (N = %d)", N);
    B200BT_REQUIRE(B >= 2 && B % 2 == 0, B200BT_EINVAL, "cscv: the block count must be even and >= 2 (B = %d)", B);
    B200BT_REQUIRE(B <= CS_MAX_BLOCKS, B200BT_ELIMIT, "cscv: at most %d blocks (B = %d)", CS_MAX_BLOCKS, B);
    B200BT_REQUIRE(T >= 0 && T / B >= 2, B200BT_EINVAL, "cscv: T = %lld days give blocks of fewer than 2 days at B = %d",
                   (long long)T, B);
    return B200BT_OK;
}

extern "C" int64_t b200bt_cscv_workspace_bytes(int N, int64_t T, int B) {
    if (N < 2 || B < 2 || B % 2 || B > CS_MAX_BLOCKS || T / B < 2) return 0;
    return cscv_layout(N, B, nullptr, nullptr);
}

extern "C" int b200bt_cscv(const double* pnl, int64_t ld, int N, int64_t T, int B, void* workspace, int64_t workspace_bytes,
                           int32_t* sel, double* is_sr, double* oos_sr, int32_t* n_below, int32_t* n_tied, double* mu,
                           double* m2, double* m3, double* m4, double* sr, b200bt_stream_t stream) {
    B200BT_REQUIRE(pnl && workspace && sel && is_sr && oos_sr && n_below && n_tied && mu && m2 && m3 && m4 && sr,
                   B200BT_EINVAL, "cscv: null pointer");
    int rc = cscv_check(N, T, B);
    if (rc) return rc;
    B200BT_REQUIRE(ld >= T, B200BT_EINVAL, "cscv: row stride %lld below T = %lld", (long long)ld, (long long)T);
    int64_t part_off = 0, n_part = 0;
    const int64_t need = cscv_layout(N, B, &part_off, &n_part);
    B200BT_REQUIRE(workspace_bytes >= need, B200BT_EINVAL, "cscv: workspace too small (%lld < %lld)",
                   (long long)workspace_bytes, (long long)need);
    B200BT_REQUIRE(((uintptr_t)workspace & 15) == 0, B200BT_EINVAL, "cscv: workspace must be 16-byte aligned");
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t L = T / B, r = T - (int64_t)B * L;
    const int C = (int)host_binom(B, B / 2);
    char* ws = (char*)workspace;
    CscvArgs A;
    A.ab = (const double*)ws;
    A.qb = (const double*)ws + (int64_t)B * N;
    A.mu = mu;
    A.N = N;
    A.C = C;
    A.tiles = (N + CS_THREADS - 1) / CS_THREADS;
    A.n_set = (double)((int64_t)(B / 2) * L);
    A.part_sr = (double*)(ws + part_off);
    A.part_n = (int*)(ws + part_off + n_part * 8);
    A.sel = sel;
    A.is_sr = is_sr;
    A.oos_sr = oos_sr;
    A.n_below = n_below;
    A.n_tied = n_tied;
    cscv_moments_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(pnl, ld, N, r, B, L, (double*)A.ab, (double*)A.qb, mu,
                                                                     m2, m3, m4, sr);
    B200BT_LAUNCH_CHECK("cscv moments");
    rc = cuda_status(cudaMemsetAsync(n_below, 0, (size_t)C * 4, st), "cscv memset");
    if (rc) return rc;
    rc = cuda_status(cudaMemsetAsync(n_tied, 0, (size_t)C * 4, st), "cscv memset");
    if (rc) return rc;
    switch (B) {
        case 2: return cscv_passes<2>(A, st);
        case 4: return cscv_passes<4>(A, st);
        case 6: return cscv_passes<6>(A, st);
        case 8: return cscv_passes<8>(A, st);
        case 10: return cscv_passes<10>(A, st);
        case 12: return cscv_passes<12>(A, st);
        case 14: return cscv_passes<14>(A, st);
        case 16: return cscv_passes<16>(A, st);
        case 18: return cscv_passes<18>(A, st);
        default: return cscv_passes<20>(A, st);
    }
}

extern "C" int b200bt_spa_moments(const double* d, int64_t ld, int N, int T, double q, double* mean, double* omega2,
                                  b200bt_stream_t stream) {
    B200BT_REQUIRE(mean && omega2, B200BT_EINVAL, "spa_moments: null pointer");
    int rc = spa_check(d, ld, N, T, "spa_moments");
    if (rc) return rc;
    B200BT_REQUIRE(q > 0.0 && q <= 1.0, B200BT_EINVAL, "spa_moments: q = %g outside (0, 1]", q);
    rc = check_device();
    if (rc) return rc;
    const size_t smem = (size_t)(3 * T + 1) * sizeof(double);
    rc = cuda_status(cudaFuncSetAttribute(spa_moments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                     "spa_moments: cudaFuncSetAttribute");
    if (rc) return rc;
    spa_moments_kernel<<<(unsigned)N, SPA_MOM_THREADS, smem, (cudaStream_t)stream>>>(d, ld, T, q, mean, omega2);
    B200BT_LAUNCH_CHECK("spa_moments");
    return B200BT_OK;
}

extern "C" int b200bt_spa_bootstrap(const double* d, int64_t ld, int N, int T, uint64_t q32, int64_t n_boot, uint64_t seed,
                                    uint64_t boot_offset, int n_stats, const double* shift, const double* scale, double* out,
                                    b200bt_stream_t stream) {
    B200BT_REQUIRE(shift && scale && out, B200BT_EINVAL, "spa_bootstrap: null pointer");
    int rc = spa_check(d, ld, N, T, "spa_bootstrap");
    if (rc) return rc;
    B200BT_REQUIRE(q32 >= 1 && q32 <= (1ull << 32), B200BT_EINVAL, "spa_bootstrap: q32 = %llu outside [1, 2^32]",
                   (unsigned long long)q32);
    B200BT_REQUIRE(n_boot >= 1, B200BT_EINVAL, "spa_bootstrap: n_boot = %lld", (long long)n_boot);
    B200BT_REQUIRE(n_stats >= 1, B200BT_EINVAL, "spa_bootstrap: n_stats = %d", n_stats);
    B200BT_REQUIRE(n_stats <= SPA_MAX_STATS, B200BT_ELIMIT, "spa_bootstrap: at most %d statistics (n_stats = %d)",
                   SPA_MAX_STATS, n_stats);
    B200BT_REQUIRE(n_boot <= (INT64_MAX >> 3) / n_stats, B200BT_ELIMIT, "spa_bootstrap: n_stats * n_boot too large");
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n_out = (int64_t)n_stats * n_boot;
    unsigned long long* o = reinterpret_cast<unsigned long long*>(out);
    spa_fill_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, st>>>(o, n_out);
    B200BT_LAUNCH_CHECK("spa_bootstrap fill");
    const int64_t tiles = ((int64_t)N + SPA_TILE - 1) / SPA_TILE;
    const int64_t want = (8 * (int64_t)device_sm_count() + tiles - 1) / tiles;
    const int64_t ny = std::max<int64_t>(1, std::min<int64_t>({want, (n_boot + SPA_WARPS - 1) / SPA_WARPS, 65535}));
    const int64_t per_cta = (n_boot + ny - 1) / ny;
    const dim3 grid((unsigned)tiles, (unsigned)((n_boot + per_cta - 1) / per_cta));
    if (T <= SPA_STAGE_T) {
        const size_t smem = (size_t)SPA_TILE * T * sizeof(double);
        rc = cuda_status(cudaFuncSetAttribute(spa_bootstrap_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)smem), "spa_bootstrap: cudaFuncSetAttribute");
        if (rc) return rc;
        spa_bootstrap_kernel<true><<<grid, SPA_WARPS * 32, smem, st>>>(d, ld, N, T, q32, n_boot, per_cta, seed, boot_offset,
                                                                       n_stats, shift, scale, o);
    } else {
        spa_bootstrap_kernel<false><<<grid, SPA_WARPS * 32, 0, st>>>(d, ld, N, T, q32, n_boot, per_cta, seed, boot_offset,
                                                                     n_stats, shift, scale, o);
    }
    B200BT_LAUNCH_CHECK("spa_bootstrap");
    spa_decode_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, st>>>(o, n_out);
    B200BT_LAUNCH_CHECK("spa_bootstrap decode");
    return B200BT_OK;
}

extern "C" int b200bt_boot_means(const double* d, int64_t ld, int N, int T, uint64_t q32, int64_t n_boot, uint64_t seed,
                                 uint64_t boot_offset, const double* center_or_null, double* out, int64_t ld_out,
                                 int64_t max_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(out, B200BT_EINVAL, "boot_means: null pointer");
    int rc = spa_check(d, ld, N, T, "boot_means");
    if (rc) return rc;
    B200BT_REQUIRE(N <= MCS_MAX_N, B200BT_ELIMIT, "boot_means: at most %d trials (N = %d)", MCS_MAX_N, N);
    B200BT_REQUIRE(q32 >= 1 && q32 <= (1ull << 32), B200BT_EINVAL, "boot_means: q32 = %llu outside [1, 2^32]",
                   (unsigned long long)q32);
    B200BT_REQUIRE(n_boot >= 1, B200BT_EINVAL, "boot_means: n_boot = %lld", (long long)n_boot);
    B200BT_REQUIRE(ld_out >= N, B200BT_EINVAL, "boot_means: ld_out = %lld below N = %d", (long long)ld_out, N);
    rc = mcs_check_budget(mcs_bytes(n_boot, ld_out), max_bytes, "boot_means");
    if (rc) return rc;
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t tiles = ((int64_t)N + SPA_TILE - 1) / SPA_TILE;
    const int64_t want = (8 * (int64_t)device_sm_count() + tiles - 1) / tiles;
    const int64_t ny = std::max<int64_t>(1, std::min<int64_t>({want, (n_boot + SPA_WARPS - 1) / SPA_WARPS, 65535}));
    const int64_t per_cta = (n_boot + ny - 1) / ny;
    const dim3 grid((unsigned)tiles, (unsigned)((n_boot + per_cta - 1) / per_cta));
    if (T <= SPA_STAGE_T) {
        const size_t smem = (size_t)SPA_TILE * T * sizeof(double);
        rc = cuda_status(cudaFuncSetAttribute(boot_means_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)smem), "boot_means: cudaFuncSetAttribute");
        if (rc) return rc;
        boot_means_kernel<true><<<grid, SPA_WARPS * 32, smem, st>>>(d, ld, N, T, q32, n_boot, per_cta, seed, boot_offset,
                                                                    center_or_null, out, ld_out);
    } else {
        boot_means_kernel<false><<<grid, SPA_WARPS * 32, 0, st>>>(d, ld, N, T, q32, n_boot, per_cta, seed, boot_offset,
                                                                  center_or_null, out, ld_out);
    }
    B200BT_LAUNCH_CHECK("boot_means");
    return B200BT_OK;
}

extern "C" int b200bt_autocov(const double* d, int64_t ld, int N, int T, int K, double* out, double* mean_or_null,
                              b200bt_stream_t stream) {
    B200BT_REQUIRE(out, B200BT_EINVAL, "autocov: null pointer");
    int rc = spa_check(d, ld, N, T, "autocov");
    if (rc) return rc;
    B200BT_REQUIRE(K >= 0 && K < T, B200BT_EINVAL, "autocov: lags 0..K need 0 <= K < T (K = %d, T = %d)", K, T);
    rc = check_device();
    if (rc) return rc;
    const size_t smem = (size_t)T * sizeof(double);
    rc = cuda_status(cudaFuncSetAttribute(autocov_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                     "autocov: cudaFuncSetAttribute");
    if (rc) return rc;
    autocov_kernel<<<(unsigned)N, SPA_MOM_THREADS, smem, (cudaStream_t)stream>>>(d, ld, T, K, out, mean_or_null);
    B200BT_LAUNCH_CHECK("autocov");
    return B200BT_OK;
}

extern "C" int b200bt_mcs_pairwise(const double* zeta, int64_t ld_z, int N, int64_t n_boot, double* s2,
                                   int64_t max_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(zeta && s2, B200BT_EINVAL, "mcs_pairwise: null pointer");
    int rc = mcs_check_n(N, "mcs_pairwise");
    if (rc) return rc;
    B200BT_REQUIRE(n_boot >= 1, B200BT_EINVAL, "mcs_pairwise: n_boot = %lld", (long long)n_boot);
    B200BT_REQUIRE(ld_z >= N, B200BT_EINVAL, "mcs_pairwise: ld_z = %lld below N = %d", (long long)ld_z, N);
    rc = mcs_check_budget(mcs_sum(mcs_bytes(n_boot, ld_z), mcs_bytes(N, N)), max_bytes, "mcs_pairwise");
    if (rc) return rc;
    rc = check_device();
    if (rc) return rc;
    const int tiles = (N + MCS_TILE - 1) / MCS_TILE;
    mcs_pairwise_kernel<<<(unsigned)(tiles * (tiles + 1) / 2), MCS_THREADS, 0, (cudaStream_t)stream>>>(zeta, ld_z, N,
                                                                                                      n_boot, tiles, s2);
    B200BT_LAUNCH_CHECK("mcs_pairwise");
    return B200BT_OK;
}

extern "C" int b200bt_mcs_range_stats(const double* mean, int N, int64_t n_boot_total, double* w, double* t,
                                      int64_t max_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(mean && w && t, B200BT_EINVAL, "mcs_range_stats: null pointer");
    int rc = mcs_check_n(N, "mcs_range_stats");
    if (rc) return rc;
    B200BT_REQUIRE(n_boot_total >= 1, B200BT_EINVAL, "mcs_range_stats: n_boot_total = %lld", (long long)n_boot_total);
    rc = mcs_check_budget(mcs_bytes(2 * (int64_t)N, N), max_bytes, "mcs_range_stats");
    if (rc) return rc;
    rc = check_device();
    if (rc) return rc;
    const int64_t n = (int64_t)N * N;
    mcs_range_stats_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(mean, N, (double)n_boot_total,
                                                                                        w, t);
    B200BT_LAUNCH_CHECK("mcs_range_stats");
    return B200BT_OK;
}

extern "C" int b200bt_mcs_range_order(const double* t, const double* rho, int N, int32_t* order, double* stat,
                                      double* rho_rank, int64_t max_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(t && rho && order && stat && rho_rank, B200BT_EINVAL, "mcs_range_order: null pointer");
    int rc = mcs_check_n(N, "mcs_range_order");
    if (rc) return rc;
    B200BT_REQUIRE(rho_rank != rho, B200BT_EINVAL, "mcs_range_order: rho_rank may alias t but not rho");
    rc = mcs_check_budget(mcs_bytes((rho_rank == t ? 2 : 3) * (int64_t)N, N), max_bytes, "mcs_range_order");
    if (rc) return rc;
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)N * 13;
    rc = cuda_status(cudaFuncSetAttribute(mcs_range_order_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                     "mcs_range_order: cudaFuncSetAttribute");
    if (rc) return rc;
    mcs_range_order_kernel<<<1, MCS_ORDER_THREADS, smem, st>>>(t, N, order, stat);
    B200BT_LAUNCH_CHECK("mcs_range_order");
    const int64_t n = (int64_t)N * N;
    mcs_rank_rho_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(rho, order, N, rho_rank);
    B200BT_LAUNCH_CHECK("mcs_range_order rank rho");
    return B200BT_OK;
}

extern "C" int b200bt_mcs_range_boot(const double* zeta, int64_t ld_z, int N, int64_t n_boot, const int32_t* order,
                                     const double* rho_rank, const double* stat, double* rmax, uint64_t* count,
                                     int64_t max_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(zeta && order && rho_rank && stat && rmax && count, B200BT_EINVAL, "mcs_range_boot: null pointer");
    int rc = mcs_check_n(N, "mcs_range_boot");
    if (rc) return rc;
    B200BT_REQUIRE(n_boot >= 1, B200BT_EINVAL, "mcs_range_boot: n_boot = %lld", (long long)n_boot);
    B200BT_REQUIRE(ld_z >= N, B200BT_EINVAL, "mcs_range_boot: ld_z = %lld below N = %d", (long long)ld_z, N);
    rc = mcs_check_budget(mcs_sum(mcs_sum(mcs_bytes(n_boot, ld_z), mcs_bytes(n_boot, N)), mcs_bytes(N, N)), max_bytes,
                          "mcs_range_boot");
    if (rc) return rc;
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t slab = (int64_t)65535 * MCS_TILE;           // resamples per launch (grid.y)
    for (int64_t lo = 0; lo < n_boot; lo += slab) {
        const int64_t nb = std::min(slab, n_boot - lo);
        const dim3 grid((unsigned)((N + MCS_TILE - 1) / MCS_TILE), (unsigned)((nb + MCS_TILE - 1) / MCS_TILE));
        mcs_range_boot_kernel<<<grid, MCS_THREADS, 0, st>>>(zeta + lo * ld_z, ld_z, N, nb, order, rho_rank, rmax + lo * N);
        B200BT_LAUNCH_CHECK("mcs_range_boot");
    }
    const size_t smem = (size_t)N * sizeof(int);
    rc = cuda_status(cudaFuncSetAttribute(mcs_range_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                     "mcs_range_boot: cudaFuncSetAttribute");
    if (rc) return rc;
    const int64_t ctas = std::min<int64_t>(2 * (int64_t)device_sm_count(), (n_boot + 7) / 8);
    mcs_range_count_kernel<<<(unsigned)ctas, MCS_THREADS, smem, st>>>(rmax, N, n_boot, stat,
                                                                     reinterpret_cast<unsigned long long*>(count));
    B200BT_LAUNCH_CHECK("mcs_range_boot count");
    return B200BT_OK;
}

extern "C" int64_t b200bt_mcs_max_workspace_bytes(int N, int64_t n_boot) {
    if (N < 2 || N > MCS_MAX_N || n_boot < 1 || n_boot > (INT64_MAX >> 4)) return 0;
    return mcs_max_ws_layout(N, n_boot, nullptr, nullptr);
}

extern "C" int b200bt_mcs_max(const double* zeta, int64_t ld_z, int N, int64_t n_boot, const double* mean, void* workspace,
                              int64_t workspace_bytes, int32_t* order, double* stat, uint64_t* count, int64_t max_bytes,
                              b200bt_stream_t stream) {
    B200BT_REQUIRE(zeta && mean && workspace && order && stat && count, B200BT_EINVAL, "mcs_max: null pointer");
    int rc = mcs_check_n(N, "mcs_max");
    if (rc) return rc;
    B200BT_REQUIRE(n_boot >= 1, B200BT_EINVAL, "mcs_max: n_boot = %lld", (long long)n_boot);
    B200BT_REQUIRE(ld_z >= N, B200BT_EINVAL, "mcs_max: ld_z = %lld below N = %d", (long long)ld_z, N);
    rc = mcs_check_budget(mcs_bytes(n_boot, ld_z), max_bytes, "mcs_max");
    if (rc) return rc;
    const int64_t need = b200bt_mcs_max_workspace_bytes(N, n_boot);
    B200BT_REQUIRE(workspace_bytes >= need, B200BT_EINVAL, "mcs_max: workspace too small (%lld < %lld)",
                   (long long)workspace_bytes, (long long)need);
    B200BT_REQUIRE(((uintptr_t)workspace & 15) == 0, B200BT_EINVAL, "mcs_max: workspace must be 16-byte aligned");
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    McsMaxWs w;
    mcs_max_ws_layout(N, n_boot, &w, (char*)workspace);
    unsigned long long* cnt = reinterpret_cast<unsigned long long*>(count);
    const unsigned rows_grid = (unsigned)((n_boot + MCS_ROWS_THREADS - 1) / MCS_ROWS_THREADS);
    mcs_max_init_kernel<<<1, 1024, 0, st>>>(mean, N, w);
    B200BT_LAUNCH_CHECK("mcs_max init");
    mcs_max_rows_kernel<<<rows_grid, MCS_ROWS_THREADS, 0, st>>>(zeta, ld_z, n_boot, w.list0, N, w, nullptr, nullptr);
    B200BT_LAUNCH_CHECK("mcs_max rows");
    for (int k = 0; k + 1 < N; ++k) {
        const int m = N - k;
        int* cur = (k & 1) ? w.list1 : w.list0;
        int* nxt = (k & 1) ? w.list0 : w.list1;
        mcs_max_var_kernel<<<(unsigned)((m + MCS_VAR_THREADS - 1) / MCS_VAR_THREADS), MCS_VAR_THREADS, 0, st>>>(
            zeta, ld_z, n_boot, cur, m, mean, w);
        B200BT_LAUNCH_CHECK("mcs_max var");
        mcs_max_step_kernel<<<1, MCS_ORDER_THREADS, 0, st>>>(cur, m, mean, w, k, nxt, order, stat);
        B200BT_LAUNCH_CHECK("mcs_max step");
        mcs_max_rows_kernel<<<rows_grid, MCS_ROWS_THREADS, 0, st>>>(zeta, ld_z, n_boot, cur, m, w, stat + k, cnt + k);
        B200BT_LAUNCH_CHECK("mcs_max rows");
    }
    return B200BT_OK;
}
