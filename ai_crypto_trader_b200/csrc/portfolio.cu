// Portfolio risk reductions (sm_90a): simple returns, tail statistics for historical VaR / CVaR,
// and the pairwise-complete Pearson correlation matrix of the asset return series.
//
// Reference: services/portfolio_risk_service.py
//   returns            df['close'].pct_change()                                   :208
//   calculate_var      np.percentile(returns.dropna(), 100 (1 - c))               :217-246
//   calculate_cvar     mean(returns[returns <= percentile])                       :248-284
//   asset correlation  pd.DataFrame(returns).corr()  (pairwise complete over finite values, Pearson) :286-326
// The percentile itself is b200bt_select (montecarlo.cu) + np.percentile's interpolation on the host.
#include "common.cuh"

namespace b200bt {

// out[s][0] = NaN, out[s][t] = close[t] / close[t-1] - 1 evaluated in float64, stored as fp32.
__global__ void __launch_bounds__(256)
pct_change_kernel(const float* __restrict__ close, int64_t ld, int64_t N, float* __restrict__ out, int64_t ld_out) {
    const int s = blockIdx.y;
    const float* __restrict__ c = close + (int64_t)s * ld;
    float* __restrict__ o = out + (int64_t)s * ld_out;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < N; t += (int64_t)gridDim.x * blockDim.x) {
        float r = __int_as_float(0x7fc00000);
        if (t > 0) r = (float)__dsub_rn(__ddiv_rn((double)c[t], (double)c[t - 1]), 1.0);
        o[t] = r;
    }
}

// out[0] = sum of x <= threshold, out[1] = their count, out[2] = number of non-NaN x, out[3] = sum of non-NaN x.
// Per-CTA partials are folded by the last CTA in block order, so the result does not depend on scheduling.
__global__ void __launch_bounds__(256)
tail_partial_kernel(const float* __restrict__ x, int64_t n, double threshold, double* __restrict__ partial) {
    double s_tail = 0.0, n_tail = 0.0, n_ok = 0.0, s_all = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double v = (double)x[i];
        if (v == v) {
            n_ok += 1.0; s_all += v;
            if (v <= threshold) { s_tail += v; n_tail += 1.0; }
        }
    }
    __shared__ double sm[4][8];
    s_tail = warp_sum_d(s_tail); n_tail = warp_sum_d(n_tail); n_ok = warp_sum_d(n_ok); s_all = warp_sum_d(s_all);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) { sm[0][w] = s_tail; sm[1][w] = n_tail; sm[2][w] = n_ok; sm[3][w] = s_all; }
    __syncthreads();
    if (threadIdx.x < 4) {
        double a = 0.0;
        for (int i = 0; i < 8; ++i) a += sm[threadIdx.x][i];
        partial[(int64_t)blockIdx.x * 4 + threadIdx.x] = a;
    }
}

__global__ void tail_final_kernel(const double* __restrict__ partial, int blocks, double* __restrict__ out4) {
    if (threadIdx.x < 4) {
        double a = 0.0;
        for (int b = 0; b < blocks; ++b) a += partial[(int64_t)b * 4 + threadIdx.x];
        out4[threadIdx.x] = a;
    }
}

// ---- correlation ------------------------------------------------------------------------------------
// An entry is an observation when it is finite: pandas' nancorr masks with np.isfinite, so a ±inf return (after a zero
// close) is missing data like NaN.
__device__ __forceinline__ bool observed(float v) { return isfinite(v); }

__device__ __forceinline__ void pair_of(int p, int S, int& i, int& j) {
    // p-th pair (i <= j) in row-major order of the upper triangle
    int row = 0, left = p;
    while (left >= S - row) { left -= S - row; ++row; }
    i = row; j = row + left;
}

constexpr int CORR_THREADS = 256;
constexpr int CORR_PARTIAL = 8;   // n, kx, ky, Su, Sv, Suu, Svv, Suv

// grid (time splits, pair blocks): each thread owns one (i, j) pair and accumulates, over the CTA's share of the time
// axis and over the bars where BOTH series are observed, n and the sums Su, Sv, Suu, Svv, Suv of u = x - kx, v = y - ky,
// shifted by the split's first joint observation (kx, ky).  The shift is exact in float64, so a series that is constant
// over the pair's joint observations gives u = 0 and a variance of exactly 0, and the cancellation in Suu - Su^2/n is
// bounded by the pair's own spread over the split, not by the row's level elsewhere.
// A tile of all S rows is staged through shared memory (row stride T+1 words: conflict-free column reads).
__global__ void __launch_bounds__(CORR_THREADS)
corr_partial_kernel(const float* __restrict__ x, int64_t ld, int S, int64_t N, int T, double* __restrict__ partial) {
    extern __shared__ float tile[];
    const int n_pairs = S * (S + 1) / 2;
    const int p = blockIdx.y * CORR_THREADS + threadIdx.x;
    int i = 0, j = 0;
    if (p < n_pairs) pair_of(p, S, i, j);
    int64_t n = 0;   // an integer count keeps the FP64 pipe for the sums
    double kx = 0.0, ky = 0.0, su = 0.0, sv = 0.0, suu = 0.0, svv = 0.0, suv = 0.0;
    const int64_t tiles = (N + T - 1) / T;
    for (int64_t tl = blockIdx.x; tl < tiles; tl += gridDim.x) {
        const int64_t t0 = tl * T;
        const int len = (int)min((int64_t)T, N - t0);
        __syncthreads();
        for (int e = threadIdx.x; e < S * T; e += CORR_THREADS) {
            const int r = e / T, c = e - r * T;
            tile[r * (T + 1) + c] = c < len ? x[(int64_t)r * ld + t0 + c] : __int_as_float(0x7fc00000);
        }
        __syncthreads();
        if (p < n_pairs) {
            const float* __restrict__ a = tile + i * (T + 1);
            const float* __restrict__ b = tile + j * (T + 1);
            int c = 0;
            if (n == 0) {   // until the split's first joint observation, which sets the shift
                for (; c < len; ++c) {
                    if (observed(a[c]) && observed(b[c])) { kx = (double)a[c]; ky = (double)b[c]; break; }
                }
            }
            for (; c < len; ++c) {
                const float fa = a[c], fb = b[c];
                if (observed(fa) && observed(fb)) {
                    const double u = (double)fa - kx, v = (double)fb - ky;
                    ++n; su += u; sv += v;
                    suu = fma(u, u, suu); svv = fma(v, v, svv); suv = fma(u, v, suv);
                }
            }
        }
    }
    if (p < n_pairs) {
        double* o = partial + ((int64_t)blockIdx.x * n_pairs + p) * CORR_PARTIAL;
        o[0] = (double)n; o[1] = kx; o[2] = ky; o[3] = su; o[4] = sv; o[5] = suu; o[6] = svv; o[7] = suv;
    }
}

// Folds the time splits in order with the pairwise update of mean, M2 and co-moment (Chan, Golub & LeVeque): a split's
// moments about its own mean, then merged by the difference of the means.  A constant run keeps M2 = 0 exactly.
__global__ void corr_final_kernel(const double* __restrict__ partial, int splits, int S, double* __restrict__ out) {
    const int n_pairs = S * (S + 1) / 2;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pairs) return;
    int i, j;
    pair_of(p, S, i, j);
    double n = 0.0, mx = 0.0, my = 0.0, m2x = 0.0, m2y = 0.0, cxy = 0.0;
    for (int s = 0; s < splits; ++s) {
        const double* q = partial + ((int64_t)s * n_pairs + p) * CORR_PARTIAL;
        const double nb = q[0];
        if (nb == 0.0) continue;
        const double du = q[3] / nb, dv = q[4] / nb;
        const double bmx = q[1] + du, bmy = q[2] + dv;
        const double bm2x = q[5] - q[3] * du, bm2y = q[6] - q[4] * dv, bcxy = q[7] - q[3] * dv;
        if (n == 0.0) {
            n = nb; mx = bmx; my = bmy; m2x = bm2x; m2y = bm2y; cxy = bcxy;
            continue;
        }
        const double nt = n + nb, ex = bmx - mx, ey = bmy - my, f = n * nb / nt;
        m2x += bm2x + ex * ex * f;
        m2y += bm2y + ey * ey * f;
        cxy += bcxy + ex * ey * f;
        mx += ex * (nb / nt);
        my += ey * (nb / nt);
        n = nt;
    }
    double r = __longlong_as_double(0x7ff8000000000000ll);
    if (n >= 1.0) {
        const double den = sqrt(m2x * m2y);
        if (den > 0.0) r = fmin(1.0, fmax(-1.0, cxy / den));
    }
    out[(int64_t)i * S + j] = r;
    out[(int64_t)j * S + i] = r;
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_pct_change(const float* close, int64_t ld, int S, int64_t N, float* out, int64_t ld_out,
                                 b200bt_stream_t stream) {
    B200BT_REQUIRE(close && out, B200BT_EINVAL, "pct_change: null pointer");
    B200BT_REQUIRE(S > 0 && N > 0 && ld >= N && ld_out >= N, B200BT_EINVAL, "pct_change: bad sizes");
    B200BT_REQUIRE(S <= 65535, B200BT_ELIMIT, "pct_change: at most 65535 rows (S = %d)", S);
    int rc = check_device();
    if (rc) return rc;
    const unsigned bx = (unsigned)min((int64_t)1184, (N + 255) / 256);
    pct_change_kernel<<<dim3(bx, (unsigned)S), 256, 0, (cudaStream_t)stream>>>(close, ld, N, out, ld_out);
    B200BT_LAUNCH_CHECK("pct_change launch");
    return B200BT_OK;
}

static int tail_blocks(int64_t n) { return (int)min((int64_t)592, (n + 255) / 256); }

extern "C" int64_t b200bt_tail_stats_workspace_bytes(int64_t n) { return (int64_t)tail_blocks(n) * 4 * 8; }

extern "C" int b200bt_tail_stats(const float* x, int64_t n, double threshold, double* out4, void* workspace,
                                 int64_t workspace_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(x && out4 && workspace, B200BT_EINVAL, "tail_stats: null pointer");
    B200BT_REQUIRE(n > 0, B200BT_EINVAL, "tail_stats: empty input");
    B200BT_REQUIRE(workspace_bytes >= b200bt_tail_stats_workspace_bytes(n), B200BT_EINVAL, "tail_stats: workspace too small");
    int rc = check_device();
    if (rc) return rc;
    const int blocks = tail_blocks(n);
    tail_partial_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, n, threshold, (double*)workspace);
    B200BT_LAUNCH_CHECK("tail_partial launch");
    tail_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((const double*)workspace, blocks, out4);
    B200BT_LAUNCH_CHECK("tail_final launch");
    return B200BT_OK;
}

static int corr_tile(int S) {
    int T = (int)(98304 / (4 * (int64_t)S)) - 1;
    if (T > 256) T = 256;
    return T & ~31;
}
static int corr_splits(int S, int64_t N) {
    const int pair_blocks = (S * (S + 1) / 2 + CORR_THREADS - 1) / CORR_THREADS;
    const int T = corr_tile(S);
    int splits = (296 + pair_blocks - 1) / pair_blocks;
    const int64_t tiles = (N + T - 1) / T;
    if (splits > tiles) splits = (int)tiles;
    return splits < 1 ? 1 : splits;
}

extern "C" int64_t b200bt_correlation_workspace_bytes(int S, int64_t N) {
    if (S <= 0 || S > 512 || N <= 0) return 0;
    return (int64_t)corr_splits(S, N) * (S * (S + 1) / 2) * CORR_PARTIAL * 8;
}

extern "C" int b200bt_correlation(const float* x, int64_t ld, int S, int64_t N, double* out, void* workspace,
                                  int64_t workspace_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(x && out && workspace, B200BT_EINVAL, "correlation: null pointer");
    B200BT_REQUIRE(S > 0 && S <= 512 && N > 0 && ld >= N, B200BT_EINVAL, "correlation: bad sizes (1 <= S <= 512)");
    B200BT_REQUIRE(workspace_bytes >= b200bt_correlation_workspace_bytes(S, N), B200BT_EINVAL, "correlation: workspace too small");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    double* partial = (double*)workspace;
    const int T = corr_tile(S), splits = corr_splits(S, N);
    const int n_pairs = S * (S + 1) / 2, pair_blocks = (n_pairs + CORR_THREADS - 1) / CORR_THREADS;
    const size_t smem = (size_t)S * (T + 1) * 4;
    cudaError_t e = cudaFuncSetAttribute(corr_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_status(e, "correlation: cudaFuncSetAttribute");
    corr_partial_kernel<<<dim3((unsigned)splits, (unsigned)pair_blocks), CORR_THREADS, smem, st>>>(x, ld, S, N, T, partial);
    B200BT_LAUNCH_CHECK("corr_partial launch");
    corr_final_kernel<<<(n_pairs + 127) / 128, 128, 0, st>>>(partial, splits, S, out);
    B200BT_LAUNCH_CHECK("corr_final launch");
    return B200BT_OK;
}
