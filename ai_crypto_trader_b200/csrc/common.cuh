// Shared helpers for the b200bt kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "b200bt.h"

namespace b200bt {

void set_error(const char* fmt, ...);
int check_device();
int device_sm_count();     // SMs of the current device (132 on an H100 SXM)
extern std::atomic<int64_t> g_launches;

inline int cuda_status(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return B200BT_OK;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return (int)e;
}

#define B200BT_REQUIRE(cond, code, ...)        \
    do {                                       \
        if (!(cond)) {                         \
            ::b200bt::set_error(__VA_ARGS__);  \
            return (code);                     \
        }                                      \
    } while (0)

// B200BT_TRACE_LAUNCHES=1 (debugging a stall): every launch is named on stderr and waited for, so the last name without a
// "done" is the kernel that does not finish.
inline bool trace_launches() {
    static const bool v = getenv("B200BT_TRACE_LAUNCHES") != nullptr;
    return v;
}

#define B200BT_LAUNCH_CHECK(what)                                       \
    do {                                                                \
        ::b200bt::g_launches.fetch_add(1, std::memory_order_relaxed);   \
        cudaError_t e__ = cudaGetLastError();                           \
        if (e__ != cudaSuccess) return ::b200bt::cuda_status(e__, what); \
        if (::b200bt::trace_launches()) {                               \
            fprintf(stderr, "[b200bt] %s ...", what); fflush(stderr);   \
            e__ = cudaDeviceSynchronize();                              \
            fprintf(stderr, " done (%d)\n", (int)e__); fflush(stderr);  \
        }                                                               \
    } while (0)

constexpr unsigned FULL = 0xffffffffu;

// Zone map of a sweep's price / RSI rows (b200bt_zone_map, csrc/sweep_chunked.cu): (min, max) per 32-bar block ("coarse")
// and per 4-bar group ("fine") of every row.  Layout: coarse [S][P + 1][zone_row_stride(N)] float2, then fine
// [S][P + 1][zone_fine_stride(N)] float2, row 0 = price; rows are 16-byte aligned and padded with (NaN, NaN).
constexpr int ZONE_BLOCK = 32;          // bars per coarse range
constexpr int ZONE_TILE = 128;          // bars per tile of the thread-per-lane scan (fine rows hold whole tiles)
__host__ __device__ constexpr int64_t zone_row_stride(int64_t N) { return (((N + ZONE_BLOCK - 1) / ZONE_BLOCK) + 1) & ~(int64_t)1; }
__host__ __device__ constexpr int64_t zone_fine_stride(int64_t N) { return ((N + ZONE_TILE - 1) / ZONE_TILE) * (ZONE_TILE / 4); }

// RSI from the two Wilder averages, ta.momentum.RSIIndicator: 100 if D == 0 else 100 - 100 / (1 + U / D), rounded to fp32.
// Evaluated as 100 U / (U + D) with ONE reciprocal: the two float64 divisions of the literal form were half of the RSI
// bank kernel's instructions.  The forms agree to ~2e-14 absolute (1.5 ulp each), so they round to the same fp32 value
// except on a ~1e-8 fraction of double-rounding ties -- below the 2e-6 the bank is tested at against float64 pandas.
// A sum in the denormal range (thousands of flat bars) takes the literal form.
__device__ __forceinline__ float rsi_value(double U, double D) {
    if (D == 0.0) return 100.0f;
    const double S = U + D;
    if (S < 1e-290) return (float)(100.0 - 100.0 / (1.0 + U / D));
    return (float)((100.0 * U) * __drcp_rn(S));
}

// Index of the last k-minute bar COMPLETED by the close of base bar t (bar_minutes long, the series starting at Unix minute
// minute0 >= 0): buckets are epoch-aligned, and bar t completes its bucket when the next bar starts in a later one.  -1
// before the first completed bar.  b200bt_align and b200bt_market_monitor share this rule.
__host__ __device__ __forceinline__ int64_t completed_bucket(int64_t t, int64_t minute0, int bar_minutes, int k) {
    const int64_t m = minute0 + t * bar_minutes;
    const int64_t b = m / k - minute0 / k;
    return (m + bar_minutes) / k != m / k ? b : b - 1;
}

__device__ __forceinline__ double shfl_up_d(double v, int d) {
    return __shfl_up_sync(FULL, v, d);
}
__device__ __forceinline__ double shfl_d(double v, int src) {
    return __shfl_sync(FULL, v, src);
}
__device__ __forceinline__ double shfl_xor_d(double v, int m) {
    return __shfl_xor_sync(FULL, v, m);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += shfl_xor_d(v, m);
    return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v = fmax(v, shfl_xor_d(v, m));
    return v;
}
__device__ __forceinline__ double warp_min_d(double v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v = fmin(v, shfl_xor_d(v, m));
    return v;
}

// Trade-hash contribution of one event (event index, event word): two 32-bit multiply-xorshift
// mixes; the lane hash is the xor over all events (oracle/sim_oracle.c computes the same).
__host__ __device__ __forceinline__ uint64_t event_hash(uint32_t index, uint32_t word) {
    uint32_t a = (index * 0x9E3779B1u) ^ word;
    a *= 0x85EBCA77u;
    a ^= a >> 15;
    uint32_t b = (word * 0xC2B2AE3Du) ^ ((index << 13) | (index >> 19));
    b *= 0x27D4EB2Fu;
    b ^= b >> 16;
    return ((uint64_t)b << 32) | a;
}

// The bar clock the strategy entry points accept: N bars of bar_minutes > 0 from Unix minute minute0 >= 0, every bar's
// minute below 2^62.
inline bool bar_clock_ok(int64_t minute0, int64_t N, int bar_minutes) {
    return bar_minutes > 0 && minute0 >= 0 && minute0 + N * (int64_t)bar_minutes < (1ll << 62);
}

// Calendar days from the day of bar 0 (day minute0 / 1440) to the day of bar N - 1: the length of a per-day row.
inline int64_t series_days(int64_t minute0, int64_t N, int bar_minutes) {
    return (minute0 + (N - 1) * (int64_t)bar_minutes) / 1440 - minute0 / 1440 + 1;
}

}  // namespace b200bt
