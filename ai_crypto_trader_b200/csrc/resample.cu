// Multi-timeframe support (BASELINE configs[3]; spec: services/market_monitor_service.py:219-301).
// The reference fetches each timeframe as its own kline series (:168-171); here the k-minute bars
// are derived on the device from the resident 1-minute OHLCV (open = first, high = max, low = min,
// close = last, volume = sum over each clock-aligned k-minute bucket, like an exchange kline /
// pandas resample), and a higher-timeframe indicator is brought back to the 1-minute clock by
// "last COMPLETED higher-timeframe bar" (no look-ahead).
//
// Buckets are aligned to the Unix epoch: bucket b covers the minutes [b*k, (b+1)*k) counted from 1970-01-01 00:00 UTC,
// i.e. pandas' resample(f"{k}min", origin="epoch"), not its default origin="start_day" (the two differ for a k that does
// not divide 1440).  A base bar starting at minute m belongs to the bucket of m; it completes its bucket when the next
// bar's start, m + bar_minutes, lies in a later bucket.  minute0 must be >= 0 (the entry points refuse a negative clock:
// the bucket arithmetic is C's truncating division).  Input is expected free of NaN: open / close take the first / last
// bar of a bucket and volume sums every bar, where pandas' first / last / sum would skip a NaN.
#include "common.cuh"

namespace b200bt {

// ohlcv [5][S][N] -> out [5][S][M];  bucket(t) = (minute0 + t*bar_minutes)/k - minute0/k
__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ in, int S, int64_t N, int64_t minute0, int bar_minutes, int k,
                float* __restrict__ out, int64_t M) {
    const int sym = blockIdx.y;
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= M) return;
    const int64_t base = minute0 / k;
    // first/last 1-minute bar of bucket b (clock aligned), clipped to the series
    const int64_t m_lo = (base + b) * k, m_hi = m_lo + k - 1;
    int64_t t_lo = (m_lo - minute0 + bar_minutes - 1) / bar_minutes;
    if (m_lo - minute0 < 0) t_lo = 0;
    int64_t t_hi = (m_hi - minute0) / bar_minutes;
    if (t_hi > N - 1) t_hi = N - 1;
    const int64_t plane = (int64_t)S * N, oplane = (int64_t)S * M;
    const float* o = in + 0 * plane + (int64_t)sym * N;
    const float* h = in + 1 * plane + (int64_t)sym * N;
    const float* l = in + 2 * plane + (int64_t)sym * N;
    const float* c = in + 3 * plane + (int64_t)sym * N;
    const float* v = in + 4 * plane + (int64_t)sym * N;
    float hi = -INFINITY, lo = INFINITY;
    double vol = 0.0;
    for (int64_t t = t_lo; t <= t_hi; ++t) {
        hi = fmaxf(hi, h[t]);
        lo = fminf(lo, l[t]);
        vol += (double)v[t];
    }
    const int64_t oi = (int64_t)sym * M + b;
    const bool any = t_lo <= t_hi;
    const float qn = __int_as_float(0x7fc00000);
    out[0 * oplane + oi] = any ? o[t_lo] : qn;
    out[1 * oplane + oi] = any ? hi : qn;
    out[2 * oplane + oi] = any ? lo : qn;
    out[3 * oplane + oi] = any ? c[t_hi] : qn;
    out[4 * oplane + oi] = any ? (float)vol : qn;
}

// out[s][t] = src[s][j(t)], j(t) = index of the last higher-timeframe bar COMPLETED at 1-minute bar t
__global__ void __launch_bounds__(256)
align_kernel(const float* __restrict__ src, int S, int64_t M, int64_t N, int64_t minute0, int bar_minutes, int k,
             float* __restrict__ out) {
    const int sym = blockIdx.y;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    const int64_t j = completed_bucket(t, minute0, bar_minutes, k);
    out[(int64_t)sym * N + t] = (j >= 0 && j < M) ? src[(int64_t)sym * M + j] : __int_as_float(0x7fc00000);
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int64_t b200bt_resample_bars(int64_t N, int64_t minute0, int bar_minutes, int k) {
    if (N <= 0 || minute0 < 0 || bar_minutes <= 0 || k <= 0) return 0;
    return (minute0 + (N - 1) * (int64_t)bar_minutes) / k - minute0 / k + 1;
}

extern "C" int b200bt_resample(const float* ohlcv, int S, int64_t N, int64_t minute0, int bar_minutes, int k,
                               float* out, int64_t M, b200bt_stream_t stream) {
    B200BT_REQUIRE(ohlcv && out, B200BT_EINVAL, "resample: null pointer");
    B200BT_REQUIRE(S > 0 && N > 0 && bar_minutes > 0 && k >= bar_minutes && k % bar_minutes == 0, B200BT_EINVAL,
                   "resample: k must be a positive multiple of bar_minutes");
    B200BT_REQUIRE(minute0 >= 0, B200BT_EINVAL, "resample: minute0 must be >= 0");
    B200BT_REQUIRE(M == b200bt_resample_bars(N, minute0, bar_minutes, k), B200BT_EINVAL, "resample: M must be b200bt_resample_bars()");
    int rc = check_device();
    if (rc) return rc;
    dim3 grid((unsigned)((M + 255) / 256), (unsigned)S);
    resample_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ohlcv, S, N, minute0, bar_minutes, k, out, M);
    B200BT_LAUNCH_CHECK("resample launch");
    return B200BT_OK;
}

extern "C" int b200bt_align(const float* src, int S, int64_t M, int64_t N, int64_t minute0, int bar_minutes, int k,
                            float* out, b200bt_stream_t stream) {
    B200BT_REQUIRE(src && out && S > 0 && M > 0 && N > 0 && bar_minutes > 0 && k > 0, B200BT_EINVAL, "align: bad argument");
    B200BT_REQUIRE(minute0 >= 0, B200BT_EINVAL, "align: minute0 must be >= 0");
    int rc = check_device();
    if (rc) return rc;
    dim3 grid((unsigned)((N + 255) / 256), (unsigned)S);
    align_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, S, M, N, minute0, bar_minutes, k, out);
    B200BT_LAUNCH_CHECK("align launch");
    return B200BT_OK;
}
