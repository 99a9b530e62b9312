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

    Machine m;
    m.pos = 0; m.e = 0.f;
    m.rlo = iv.rsi_lo; m.rhi = iv.rsi_hi; m.plo = -INFINITY; m.phi = INFINITY;
    m.qhead = 0; m.entry_bar = 0;
    const ScanConst c = ws->sc;                // warp-uniform constants of the scan, kept in registers
    unsigned qtail = 0;

    // Streams are staged through a per-warp shared-memory ring filled with cp.async
    // (16 B per thread = 128 bars per instruction when the rows are 16-byte aligned):
    // SW_STAGES-1 groups are always in flight, no registers are tied up by prefetch.
    constexpr int G = SW_GROUP;               // bars per group
    float* const sp = &ws->ring[0][0][0];
    const int n = (int)N;
    const int n_full = n / G;                 // groups copied without bounds checks
    const int n_groups = (n + G - 1) / G;
    // running producer state: next group to issue, its ring slot, its source pointers
    int issued = 0;
    float* idst = sp + (VEC16 ? lane * 4 : lane);
    const float* ip = pr + (VEC16 ? lane * 4 : lane);
    const float* ir = rr + (VEC16 ? lane * 4 : lane);
    auto issue = [&]() {
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
        } else if (issued < n_groups) {
            // ragged last group: guarded loads, NaN beyond the series (NaN never fires an event)
            const float qnan = __int_as_float(0x7fc00000);
            float* dst = sp + (issued % SW_STAGES) * (2 * G);
            for (int i = lane; i < G; i += 32) {
                const int t = issued * G + i;
                dst[i] = t < n ? __ldg(pr + t) : qnan;
                dst[G + i] = t < n ? __ldg(rr + t) : qnan;
            }
        }
        cp_async_commit();  // always commit (possibly empty) so the group accounting stays uniform
        ++issued;
        ip += G; ir += G;
        idst = (issued % SW_STAGES == 0) ? idst - (SW_STAGES - 1) * (2 * G) : idst + 2 * G;
    };
#pragma unroll
    for (int g = 0; g < SW_STAGES - 1; ++g) issue();
    const float* cur = sp + lane;
    int cstage = 0;
    for (int g = 0; g < n_groups; ++g) {
        issue();
        cp_async_wait<SW_STAGES - 1>();       // group g has landed
        __syncwarp();
        const float* w = cur;
        int t0 = g * G;
#pragma unroll 1
        for (int v = 0; v < G / 64; ++v, w += 64, t0 += 64) {
            // two windows per step: both ballots are issued before either is needed
            const float p0 = w[0], r0 = w[G];
            const float p1 = w[32], r1 = w[G + 32];
            const unsigned h0 = __ballot_sync(FULL, fires(m, p0, r0));
            const unsigned h1 = __ballot_sync(FULL, fires(m, p1, r1));
            if (h0 | h1) {
                if (h0) scan_window(p0, r0, w - lane, t0, ws, c, m);
                scan_window(p1, r1, w - lane + 32, t0 + 32, ws, c, m);
                while (m.qhead - qtail >= 32) {
                    __syncwarp();
                    process_batch(ws, qtail, 32, minute0, bar_minutes, ev_cap);
                    qtail += 32;
                }
            }
        }
        __syncwarp();                         // stage is refilled by the next iteration's issue
        if (++cstage == SW_STAGES) { cstage = 0; cur -= (SW_STAGES - 1) * (2 * G); } else cur += 2 * G;
    }
    cp_async_wait<0>();
    if (m.pos != 0) {
        // force-close at the last bar (:849-876)
        const float pl = __ldg(pr + (N - 1));
        const unsigned word = (unsigned)(N - 1) | B200BT_EVENT_EXIT | (m.pos > 0 ? B200BT_EVENT_SELL : 0u);
        if (lane == 0) ws->evq[m.qhead & (SW_EVQ - 1)] = make_uint2(word, __float_as_uint(pl));
        ++m.qhead;
    }
    __syncwarp();
    while (m.qhead != qtail) {
        const int cnt = min(32u, m.qhead - qtail);
        process_batch(ws, qtail, cnt, minute0, bar_minutes, ev_cap);
        qtail += cnt;
    }

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

// The fused sweep over the first *pop_dev (<= pop) entries of `order`: the grid covers `pop` entries and warps beyond the
// device-side count leave at once.  The exact fallback of the time-chunked sweeps: the list of individuals to re-run and its
// length never leave the device.
int launch_sweep(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                 const b200bt_individual* indiv, const int32_t* order, int pop, const int* pop_dev,
                 const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats, uint32_t* events, int64_t event_cap,
                 cudaStream_t stream) {
    const int64_t blocks = (int64_t)((pop + SW_WARPS - 1) / SW_WARPS) * S;
    B200BT_REQUIRE(blocks < (1ll << 31), B200BT_ELIMIT, "sweep: too many lanes");
    const size_t smem = sizeof(WarpShared) * SW_WARPS;
    // 16-byte cp.async needs every (symbol, period) row to start on a 16-byte boundary
    const bool vec16 = (((uintptr_t)price | (uintptr_t)rsi) & 15) == 0 && ld_price % 4 == 0 && ld_rsi % 4 == 0;
    auto kern = vec16 ? sweep_kernel<true> : sweep_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_status(e, "sweep: cudaFuncSetAttribute");
    kern<<<(unsigned)blocks, SW_WARPS * 32, smem, stream>>>(
        price, ld_price, rsi, ld_rsi, P, S, N, indiv, order, pop, pop_dev, *cfg_host, stats, events, event_cap);
    B200BT_LAUNCH_CHECK("sweep launch");
    return B200BT_OK;
}
}  // namespace b200bt

extern "C" int b200bt_sweep(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P,
                            int S, int64_t N, const b200bt_individual* indiv, const int32_t* order, int pop,
                            const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats,
                            uint32_t* events, int64_t event_cap, b200bt_stream_t stream) {
    B200BT_REQUIRE(price && rsi && indiv && cfg_host && stats, B200BT_EINVAL, "sweep: null pointer");
    B200BT_REQUIRE(S > 0 && N > 0 && P > 0 && pop > 0, B200BT_EINVAL, "sweep: bad sizes");
    B200BT_REQUIRE(ld_price >= N && ld_rsi >= N, B200BT_EINVAL, "sweep: row stride shorter than N");
    B200BT_REQUIRE(N < (1ll << 30), B200BT_ELIMIT, "sweep: N must be < 2^30 bars");
    int rc = check_sweep_clock("sweep", cfg_host, N);
    if (rc) return rc;
    B200BT_REQUIRE(events == nullptr || event_cap > 0, B200BT_EINVAL, "sweep: event buffer without capacity");
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
