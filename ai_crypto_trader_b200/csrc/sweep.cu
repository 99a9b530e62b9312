// Family 2: the per-bar entry/exit/stop/PnL state machine over
// (GA-individual x symbol) lanes, with calculate_metrics and the strategy score
// reduced in-kernel (sm_90a).
//
// Reference semantics: services/strategy_evaluation.py:746-878 (_simulate_trades),
// :32-228 (calculate_metrics), :579-633 (_calculate_strategy_score).
//
// Mapping: ONE WARP PER LANE.  The 32 threads of a warp look at 32 consecutive
// bars of the lane's (price, rsi) streams at once; the machine's state
// (flat / long / short + entry price) is warp-uniform.  A ballot finds the
// first bar in the window at which the current state has an event (entry
// signal, or take-profit / stop-loss / RSI exit), the state is advanced, and
// the remaining bars of the window are re-tested under the new state.  Quiet
// stretches therefore cost two coalesced 128-byte loads and four compares per
// 32 bars, and the time axis -- serial in the reference -- is consumed 32 bars
// per step.
//
// Exactness (bit-exact entry/exit bars against the float64 reference):
//  * RSI tests compare the fp32 bank value with thresholds the host rounded so
//    that the fp32 compare decides like the float64 one.
//  * The price exits `(p-e)/e >= tp`, `<= -sl` are screened with fp32 bounds
//    that are provably conservative (relative margin 1e-6); a bar that is not
//    a definite exit is decided by the float64 expression itself.
//  * PnL, equity, drawdown, daily buckets and the score are float64, evaluated
//    from the queued events 32 at a time with warp scans.
#include <math.h>
#include "common.cuh"

#include "sweep_dev.cuh"

namespace b200bt {

template <bool VEC16>
__global__ void __launch_bounds__(SW_WARPS * 32, SW_MIN_BLOCKS)
sweep_kernel(const float* __restrict__ price, int64_t ld_price,
             const float* __restrict__ rsi, int64_t ld_rsi, int P, int S, int64_t N,
             const b200bt_individual* __restrict__ indiv, const int32_t* __restrict__ order, int pop,
             const int* __restrict__ pop_dev,   // optional: number of entries of `order` to evaluate, on the device (<= pop)
             const b200bt_sweep_config cfg,  // NOT __grid_constant__: nvcc 12.9 miscompiled a loop-carried value with it
             b200bt_lane_stats* __restrict__ stats, uint32_t* __restrict__ events, int64_t ev_cap) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int lane = threadIdx.x & 31;
    // CTA b evaluates SW_WARPS consecutive individuals of the host's evaluation order on one symbol;
    // all symbols of the first (most expensive) individuals are dispatched first, so the grid drains
    // in longest-processing-time-first order and the tail consists of cheap lanes.
    const int sym = (int)(blockIdx.x % (unsigned)S);
    const int k = (int)(blockIdx.x / (unsigned)S) * SW_WARPS + (threadIdx.x >> 5);
    if (k >= (pop_dev ? min(pop, *pop_dev) : pop)) return;
    const int ind = order ? order[k] : k;
    const b200bt_individual iv = indiv[ind];
    WarpShared* ws = reinterpret_cast<WarpShared*>(s_raw) + (threadIdx.x >> 5);

    if (lane == 0) {
        ScanConst sc0;
        init_scan_const(sc0, iv);
        ws->sc = sc0;
        WarpAcc a0;
        init_acc(a0, iv, cfg, events ? events + ((int64_t)ind * S + sym) * ev_cap : nullptr);
        ws->acc = a0;
    }
    __syncwarp();

    const float* __restrict__ pr = price + (int64_t)sym * ld_price;
    const float* __restrict__ rr = rsi + ((int64_t)sym * P + iv.rsi_row) * ld_rsi;
    const long long minute0 = cfg.minute0;
    const int bar_minutes = cfg.bar_minutes;

    // the whole series, group by group through the warp's cp.async ring
    const int n = (int)N;
    const int n_groups = (n + SW_GROUP - 1) / SW_GROUP;
    GroupRing<VEC16> ring(ws, pr, rr, n, 0, n_groups);
    const ScanConst c = ws->sc;                // warp-uniform constants of the scan, kept in registers
    Machine m = flat_machine(iv);
    unsigned qtail = 0;
    auto batch = [&](unsigned at, int cnt) { process_batch(ws, at, cnt, minute0, bar_minutes, ev_cap); };
    for (int g = 0; g < n_groups; ++g) {
        scan_group(ring.land(), g * SW_GROUP, ws, c, m, qtail, true, batch);
        ring.release();
    }
    finish_scan(ws, m, qtail, pr, N, true, batch);

    if (lane == 0) {
        b200bt_lane_stats o;
        finalize_lane(ws->acc, cfg, o);
        stats[(int64_t)ind * S + sym] = o;
    }
}

__global__ void fitness_reduce_kernel(const b200bt_lane_stats* __restrict__ stats, int pop, int S,
                                      double* __restrict__ fitness) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pop) return;
    double acc = 0.0;
    for (int s = 0; s < S; ++s) acc += stats[(int64_t)i * S + s].score;
    fitness[i] = acc / (double)S;
}

}  // namespace b200bt

using namespace b200bt;

namespace b200bt {
int check_sweep_clock(const char* who, const b200bt_sweep_config* cfg, int64_t N) {
    B200BT_REQUIRE(cfg->bar_minutes > 0 && cfg->minute0 >= 0 && cfg->gap_minutes >= 0, B200BT_EINVAL,
                   "%s: bar_minutes must be > 0, minute0 and gap_minutes >= 0", who);
    // (minute0 is compared against the rest: no int64 overflow for any minute0)
    B200BT_REQUIRE(cfg->minute0 < (1ll << 32) - 1440 - N * (int64_t)cfg->bar_minutes - cfg->gap_minutes, B200BT_ELIMIT,
                   "%s: minute0 + N*bar_minutes + gap_minutes must stay below 2^32 - 1440 minutes", who);
    return B200BT_OK;
}

int check_sweep_args(const char* who, const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S,
                     int64_t N, const b200bt_sweep_config* cfg_host, const uint32_t* events, int64_t event_cap) {
    B200BT_REQUIRE(price && rsi && cfg_host, B200BT_EINVAL, "%s: null pointer", who);
    B200BT_REQUIRE(S > 0 && N > 0 && P > 0, B200BT_EINVAL, "%s: bad sizes", who);
    B200BT_REQUIRE(ld_price >= N && ld_rsi >= N, B200BT_EINVAL, "%s: row stride shorter than N", who);
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "%s: N must be < 2^30 bars", who);
    const int rc = check_sweep_clock(who, cfg_host, N);
    if (rc) return rc;
    B200BT_REQUIRE(events == nullptr || event_cap > 0, B200BT_EINVAL, "%s: event buffer without capacity", who);
    return B200BT_OK;
}

int check_record_args(const char* who, const float* price, int64_t ld_price, int S, int64_t N,
                      const b200bt_individual* indiv, int pop, const b200bt_sweep_config* cfg,
                      const b200bt_lane_stats* lane_stats, const uint32_t* events, int64_t event_cap) {
    B200BT_REQUIRE(price && indiv && lane_stats, B200BT_EINVAL, "%s: null pointer", who);
    B200BT_REQUIRE(S >= 1 && pop >= 1 && N >= 1 && ld_price >= N, B200BT_EINVAL, "%s: bad sizes", who);
    B200BT_REQUIRE(event_cap >= 0 && (events || event_cap == 0), B200BT_EINVAL, "%s: bad event buffer", who);
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "%s: N must be < 2^30 bars", who);
    return cfg ? check_sweep_clock(who, cfg, N) : B200BT_OK;
}

bool vec16_rows(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi) {
    return (((uintptr_t)price | (uintptr_t)rsi) & 15) == 0 && ld_price % 4 == 0 && ld_rsi % 4 == 0;
}

// The fused sweep over the first *pop_dev (<= pop) entries of `order`: the grid covers `pop` entries and warps beyond the
// device-side count leave at once.  The exact fallback of the time-chunked sweeps: the list of individuals to re-run and its
// length never leave the device.
int launch_sweep(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                 const b200bt_individual* indiv, const int32_t* order, int pop, const int* pop_dev,
                 const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats, uint32_t* events, int64_t event_cap,
                 cudaStream_t stream) {
    const int64_t blocks = (int64_t)((pop + SW_WARPS - 1) / SW_WARPS) * S;
    B200BT_REQUIRE(blocks < (1ll << 31), B200BT_ELIMIT, "sweep: too many lanes");
    auto kern = vec16_rows(price, ld_price, rsi, ld_rsi) ? sweep_kernel<true> : sweep_kernel<false>;
    const int rc = allow_sw_smem(kern, "sweep: cudaFuncSetAttribute");
    if (rc) return rc;
    kern<<<(unsigned)blocks, SW_WARPS * 32, SW_SMEM, stream>>>(
        price, ld_price, rsi, ld_rsi, P, S, N, indiv, order, pop, pop_dev, *cfg_host, stats, events, event_cap);
    B200BT_LAUNCH_CHECK("sweep launch");
    return B200BT_OK;
}
}  // namespace b200bt

extern "C" int b200bt_sweep(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P,
                            int S, int64_t N, const b200bt_individual* indiv, const int32_t* order, int pop,
                            const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats,
                            uint32_t* events, int64_t event_cap, b200bt_stream_t stream) {
    B200BT_REQUIRE(indiv && stats, B200BT_EINVAL, "sweep: null pointer");
    B200BT_REQUIRE(pop > 0, B200BT_EINVAL, "sweep: bad sizes");
    int rc = check_sweep_args("sweep", price, ld_price, rsi, ld_rsi, P, S, N, cfg_host, events, event_cap);
    if (rc) return rc;
    rc = check_device();
    if (rc) return rc;
    return launch_sweep(price, ld_price, rsi, ld_rsi, P, S, N, indiv, order, pop, nullptr, cfg_host, stats, events, event_cap,
                        (cudaStream_t)stream);
}

extern "C" int b200bt_fitness_reduce(const b200bt_lane_stats* stats, int pop, int S, double* fitness,
                                     b200bt_stream_t stream) {
    B200BT_REQUIRE(stats && fitness && pop > 0 && S > 0, B200BT_EINVAL, "fitness_reduce: bad argument");
    int rc = check_device();
    if (rc) return rc;
    fitness_reduce_kernel<<<(pop + 127) / 128, 128, 0, (cudaStream_t)stream>>>(stats, pop, S, fitness);
    B200BT_LAUNCH_CHECK("fitness_reduce launch");
    return B200BT_OK;
}
