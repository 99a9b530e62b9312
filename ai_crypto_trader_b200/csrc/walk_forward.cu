// Walk-forward evaluation (sm_90a): a lane that trades a SCHEDULE of bar segments, each with its own individual, and the
// device decode of a GA parameter matrix into individuals.
//
// Reference semantics: services/strategy_evaluation.py:746-878 (_simulate_trades) called once per segment, the records of
// all segments concatenated in segment order and scored as one list by calculate_metrics (:32-228) and
// _calculate_strategy_score (:579-633).  Each segment starts flat and force-closes at its last bar; equity, peak, drawdown,
// the calendar-day buckets and the trade hash run on across segments.
//
// Mapping: ONE WARP PER LANE (schedule j, symbol s), sweep_kernel's bar scan and metrics (sweep_dev.cuh) run segment by
// segment.  At a segment boundary the warp reloads the scan constants, the machine and the individual's take-profit /
// stop-loss / size / fees, restarts the cp.async ring at the segment's first bar, and adds the segment's first bar to the
// queued (segment-local) event words before they reach the metrics, so records carry global bars and fall on the series'
// own calendar.  The ring copies 16 bytes per thread when the segment's price and RSI rows start on 16-byte boundaries,
// 4 bytes otherwise (a warp-uniform choice per segment).
#include <math.h>
#include <stddef.h>
#include "common.cuh"

#include "sweep_dev.cuh"

namespace b200bt {

constexpr int DECODE_MAX_PERIODS = 256;     // entries of the period -> bank row table of b200bt_decode_individuals

// One segment record of b200bt_sweep_segments' table (include/b200bt.h, B200BT_SEGMENT_*).
struct Segment {
    int64_t start;        // first bar
    int64_t end;          // one past the last bar
    int32_t individual;   // row of indiv that trades the segment
    int32_t reserved;     // 0
};
static_assert(sizeof(Segment) == B200BT_SEGMENT_BYTES, "segment record size");
static_assert(offsetof(Segment, start) == B200BT_SEGMENT_START && offsetof(Segment, end) == B200BT_SEGMENT_END &&
              offsetof(Segment, individual) == B200BT_SEGMENT_INDIVIDUAL &&
              offsetof(Segment, reserved) == B200BT_SEGMENT_RESERVED, "segment record layout");

// One segment of a lane: bars [0, n) of the rows pr / rr (the segment's first bar at index 0), whose first bar is global
// bar `off`.  Starts flat, force-closes at its last bar; every record goes through the metrics in `ws->acc`.
template <bool VEC16>
__device__ __forceinline__ void trade_segment(WarpShared* __restrict__ ws, const float* __restrict__ pr,
                                              const float* __restrict__ rr, int n, unsigned off, const ScanConst& c,
                                              const b200bt_individual& iv, long long minute0, int bar_minutes,
                                              int64_t ev_cap) {
    const int n_groups = (n + SW_GROUP - 1) / SW_GROUP;
    GroupRing<VEC16> ring(ws, pr, rr, n, 0, n_groups);
    Machine m = flat_machine(iv);
    unsigned qtail = 0;
    // bars below 2^30 (checked on the host): adding the offset never carries into the EXIT / SELL bits
    auto batch = [&](unsigned at, int cnt) {
        const uint2 evt = ws->evq[(at + (threadIdx.x & 31)) & (SW_EVQ - 1)];
        batch_core(&ws->acc, cnt, evt.x + off, __uint_as_float(evt.y), 0u, 0.f, minute0, bar_minutes, ev_cap);
    };
    for (int g = 0; g < n_groups; ++g) {
        scan_group(ring.land(), g * SW_GROUP, ws, c, m, qtail, true, batch);
        ring.release();
    }
    finish_scan(ws, m, qtail, pr, n, true, batch);
}

// True when schedule [b, e) of `segments` is invalid (include/b200bt.h, b200bt_sweep_segments); warp-uniform.
__device__ __forceinline__ bool bad_schedule(const Segment* __restrict__ segments, int64_t b, int64_t e, int64_t N,
                                             const b200bt_individual* __restrict__ indiv, int n_indiv, int P) {
    if (e <= b) return true;
    bool bad = false;
    for (int64_t k = b + (threadIdx.x & 31); k < e; k += 32) {
        const Segment sg = segments[k];
        const int32_t ind = sg.individual;
        bad |= sg.start < 0 || sg.end <= sg.start || sg.end > N || sg.reserved != 0;
        bad |= k > b && sg.start < segments[k - 1].end;
        if (ind < 0 || ind >= n_indiv) bad = true;
        else bad |= indiv[ind].rsi_row < 0 || indiv[ind].rsi_row >= P;
    }
    return __any_sync(FULL, bad);
}

__global__ void __launch_bounds__(SW_WARPS * 32, SW_MIN_BLOCKS)
segment_sweep_kernel(const float* __restrict__ price, int64_t ld_price, const float* __restrict__ rsi, int64_t ld_rsi,
                     int P, int S, int64_t N, const b200bt_individual* __restrict__ indiv, int n_indiv,
                     const Segment* __restrict__ segments, const int32_t* __restrict__ seg_begin, int J,
                     const b200bt_sweep_config cfg,   // by value, as sweep_kernel takes it
                     b200bt_lane_stats* __restrict__ stats, uint32_t* __restrict__ events, int64_t ev_cap) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int lane = threadIdx.x & 31;
    const int sym = (int)(blockIdx.x % (unsigned)S);
    const int j = (int)(blockIdx.x / (unsigned)S) * SW_WARPS + (threadIdx.x >> 5);
    if (j >= J) return;
    const int64_t w = (int64_t)j * S + sym;
    const int64_t b = seg_begin[j], e = seg_begin[j + 1];
    if (bad_schedule(segments, b, e, N, indiv, n_indiv, P)) {
        if (lane == 0) stats[w] = lost_lane_stats();
        return;
    }
    WarpShared* ws = reinterpret_cast<WarpShared*>(s_raw) + (threadIdx.x >> 5);
    if (lane == 0) {
        WarpAcc a0;
        init_acc(a0, indiv[segments[b].individual], cfg, events ? events + w * ev_cap : nullptr);
        ws->acc = a0;
    }
    const float* __restrict__ prow = price + (int64_t)sym * ld_price;
    const long long minute0 = cfg.minute0;
    const int bar_minutes = cfg.bar_minutes;

    for (int64_t k = b; k < e; ++k) {
        const int64_t start = segments[k].start, end = segments[k].end;
        const b200bt_individual iv = indiv[segments[k].individual];
        __syncwarp();                      // the previous segment's last batch is done with ws->acc / ws->sc
        if (lane == 0) {
            ScanConst sc0;
            init_scan_const(sc0, iv);
            ws->sc = sc0;
            WarpAcc& a = ws->acc;
            a.tp = iv.take_profit; a.sl = iv.stop_loss; a.size = iv.position_size;
            a.fee1 = __dmul_rn(a.size, 0.001); a.fee2 = __dmul_rn(a.size, 0.002);
        }
        __syncwarp();
        const ScanConst c = ws->sc;
        const float* pr = prow + start;
        const float* rr = rsi + ((int64_t)sym * P + iv.rsi_row) * ld_rsi + start;
        if ((((uintptr_t)pr | (uintptr_t)rr) & 15) == 0)
            trade_segment<true>(ws, pr, rr, (int)(end - start), (unsigned)start, c, iv, minute0, bar_minutes, ev_cap);
        else
            trade_segment<false>(ws, pr, rr, (int)(end - start), (unsigned)start, c, iv, minute0, bar_minutes, ev_cap);
    }

    if (lane == 0) {
        b200bt_lane_stats o;
        finalize_lane(ws->acc, cfg, o);
        stats[w] = o;
    }
}

// decode_population (ai_crypto_trader_b200/sweep.py) of one row of the GA matrix.
struct DecodeTable {
    int32_t col[6];                         // rsi_period, rsi_oversold, rsi_overbought, take_profit, stop_loss, max_position_size
    int32_t n_rows;
    int32_t row[DECODE_MAX_PERIODS];        // period -> bank row, -1 = not in the bank
};

__global__ void decode_individuals_kernel(const double* __restrict__ params, int64_t ld, int n, const DecodeTable T,
                                          b200bt_individual* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* p = params + (int64_t)i * ld;
    const double dflt[6] = {14.0, 30.0, 70.0, 3.0, 2.0, 5.0};
    double v[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) v[k] = T.col[k] >= 0 ? p[T.col[k]] : dflt[k];
    b200bt_individual o;
    // the period is truncated towards zero (numpy astype(int64)); outside the table: no bank row
    const double period = trunc(v[0]);
    o.rsi_row = (period >= 0.0 && period < (double)T.n_rows) ? T.row[(int)period] : -1;
    // thresholds rounded towards the side that keeps `rsi < oversold` / `rsi > overbought` exact in fp32
    float lo = __double2float_rn(v[1]), hi = __double2float_rn(v[2]);
    if (!((double)lo >= v[1])) lo = nextafterf(lo, INFINITY);
    if (!((double)hi <= v[2])) hi = nextafterf(hi, -INFINITY);
    o.rsi_lo = lo;
    o.rsi_hi = hi;
    o.reserved = 0;
    // strategy_evaluation.py:762-764, :773-774 (same float64 expressions; np.minimum keeps a NaN)
    o.take_profit = __ddiv_rn(v[3], 100.0);
    o.stop_loss = __ddiv_rn(v[4], 100.0);
    const double size = v[5] > 20.0 ? 20.0 : v[5];
    o.position_size = __dmul_rn(10000.0, __ddiv_rn(size, 100.0));
    out[i] = o;
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_sweep_segments(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S,
                                     int64_t N, const b200bt_individual* indiv, int n_indiv, const int64_t* segments,
                                     const int32_t* seg_begin, int J, const b200bt_sweep_config* cfg_host,
                                     b200bt_lane_stats* stats, uint32_t* events, int64_t event_cap,
                                     b200bt_stream_t stream) {
    B200BT_REQUIRE(indiv && segments && seg_begin && stats, B200BT_EINVAL, "sweep_segments: null pointer");
    B200BT_REQUIRE(n_indiv > 0 && J > 0, B200BT_EINVAL, "sweep_segments: bad sizes");
    int rc = check_sweep_args("sweep_segments", price, ld_price, rsi, ld_rsi, P, S, N, cfg_host, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE(cfg_host->gap_bar == 0, B200BT_EINVAL, "sweep_segments: gap_bar must be 0 (segments of a glued series)");
    const int64_t blocks = (int64_t)((J + SW_WARPS - 1) / SW_WARPS) * S;
    B200BT_REQUIRE(blocks < (1ll << 31), B200BT_ELIMIT, "sweep_segments: too many lanes");
    if ((rc = check_device())) return rc;
    if ((rc = allow_sw_smem(segment_sweep_kernel, "sweep_segments: cudaFuncSetAttribute"))) return rc;
    segment_sweep_kernel<<<(unsigned)blocks, SW_WARPS * 32, SW_SMEM, (cudaStream_t)stream>>>(
        price, ld_price, rsi, ld_rsi, P, S, N, indiv, n_indiv, reinterpret_cast<const Segment*>(segments), seg_begin, J,
        *cfg_host, stats, events, event_cap);
    B200BT_LAUNCH_CHECK("sweep_segments launch");
    return B200BT_OK;
}

extern "C" int b200bt_decode_individuals(const double* params, int64_t ld, int n, const int* gene_cols_host,
                                         const int32_t* period_row_host, int n_period_row, b200bt_individual* out,
                                         b200bt_stream_t stream) {
    B200BT_REQUIRE(params && gene_cols_host && period_row_host && out, B200BT_EINVAL, "decode_individuals: null pointer");
    B200BT_REQUIRE(n > 0 && ld > 0 && n_period_row > 0, B200BT_EINVAL, "decode_individuals: bad sizes");
    B200BT_REQUIRE(n_period_row <= DECODE_MAX_PERIODS, B200BT_ELIMIT, "decode_individuals: at most %d periods in the table",
                   DECODE_MAX_PERIODS);
    DecodeTable T;
    for (int k = 0; k < 6; ++k) {
        B200BT_REQUIRE(gene_cols_host[k] >= -1 && gene_cols_host[k] < ld, B200BT_EINVAL,
                       "decode_individuals: gene column %d outside [-1, ld)", k);
        T.col[k] = gene_cols_host[k];
    }
    T.n_rows = n_period_row;
    for (int k = 0; k < n_period_row; ++k) T.row[k] = period_row_host[k];
    int rc = check_device();
    if (rc) return rc;
    decode_individuals_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(params, ld, n, T, out);
    B200BT_LAUNCH_CHECK("decode_individuals launch");
    return B200BT_OK;
}
