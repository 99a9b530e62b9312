// Family 3: Monte-Carlo price paths (GBM / bootstrap) with a Philox4x32-10
// counter-based RNG, plus the exact order statistics the risk report needs (sm_90a).
//
// Reference semantics: MonteCarloService.run_monte_carlo_simulation,
// services/monte_carlo_service.py:197-394.
//   GBM        paths[t] = paths[t-1] * exp((mu - sigma^2/2) dt + sigma sqrt(dt) Z)   :266-273
//   historical iid bootstrap of the return sample, log or simple compounding        :277-298
//   per-path max drawdown = max_t (runmax_t - S_t)/runmax_t                         :327-336
//
// One thread per path.  The path lives in log space in registers
// (logS_t = logS_{t-1} + increment), so risk-only mode never exponentiates inside
// the time loop: the final price is s0*exp(logS_T) and the maximum drawdown is
// 1 - exp(min_t(logS_t - max_{s<=t} logS_s)).  Four steps (one Philox block) are
// accumulated in fp32 relative to an fp64 base that absorbs each block's sum, so
// 10^4 increments do not drift while the inner loop stays on the fp32 pipe.
// Randomness is a pure function of (seed, path index, step): results do not
// depend on the launch geometry or on how paths are sharded across GPUs.
#include <math.h>
#include <string.h>
#include "common.cuh"
#include "philox.cuh"

namespace b200bt {

// 24-bit uniform in (0,1]: (k + 0.5) * 2^-24 rounded to fp32 (for k >= 2^23 the half is absorbed by
// round-to-even, so the top value rounds to exactly 1; never 0).
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }

// Box-Muller: two uniforms -> two standard normals (r cos 2*pi*v, r sin 2*pi*v), all on the MUFU units.
// Radius: t = -2 ln u with the fast __logf (absolute error 2^-21 in ln u).  For u -> 1 that error exceeds -ln u
// itself and can make t slightly negative: t is clamped at 0, i.e. a radius below ~1e-3 (probability ~5e-7 per
// draw) is only known to ~1e-3 absolute -- far below the Monte-Carlo error of any statistic reported here, and
// checked against the float64 NumPy restatement (oracle/mc_ref.py) at 3e-5 relative on the final prices.
// Angle: taken in (-pi, pi) where __sincosf is accurate to 2^-21; the half-turn shift is undone by the sign flip.
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    const float t = fmaxf(-2.0f * __logf(u01(a)), 0.0f);
    const float r = t * rsqrtf(fmaxf(t, 1e-30f));
    float s, c;
    __sincosf(6.283185307179586f * u01(b) - 3.14159265358979f, &s, &c);
    z0 = -r * c;
    z1 = -r * s;
}

constexpr int MC_THREADS = 256;

// The n entries of a bootstrap table into shared memory as log returns: paths compound in log space either way.
__device__ __forceinline__ void stage_log_returns(float* s_ret, const float* __restrict__ returns, int n, int log_returns) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float r = returns[i];
        s_ret[i] = log_returns ? r : log1pf(r);
    }
    __syncthreads();
}

// mode 0: GBM.  mode 1: bootstrap of `returns` (R values, staged in shared memory),
// blocks of `block_len` consecutive returns (circular), log_returns selects compounding.
template <int MODE>
__global__ void __launch_bounds__(MC_THREADS)
mc_paths_kernel(double s0, double drift, double vol, const float* __restrict__ returns, int R, int block_len,
                int log_returns, int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset,
                float* __restrict__ finals, float* __restrict__ maxdd, float* __restrict__ paths) {
    extern __shared__ float s_ret[];
    if (MODE == 1) stage_log_returns(s_ret, returns, R, log_returns);
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_paths) return;

    // log-price relative to log(s0): block base `base` and running maximum `runmax` in fp64, the four
    // steps of a Philox block in fp32 relative to the base (their sum is folded into the base exactly)
    double base = 0.0, runmax = 0.0, worst = 0.0;
    const float fs0 = (float)s0, fdrift = (float)drift, fvol = (float)vol;
    if (paths) paths[p] = fs0;
    BlockBootstrap boot;
    for (int t0 = 0; t0 < steps; t0 += 4) {
        uint32_t x[4];
        philox_path(seed, path_offset, p, (uint32_t)(t0 >> 2), (uint32_t)MODE, x);
        float inc[4];
        if (MODE == 0) {
            float z[4];
            box_muller(x[0], x[1], z[0], z[1]);
            box_muller(x[2], x[3], z[2], z[3]);
#pragma unroll
            for (int j = 0; j < 4; ++j) inc[j] = fmaf(fvol, z[j], fdrift);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) inc[j] = s_ret[boot.next(x[j], R, block_len)];
        }
        const float d0 = (float)(runmax - base);   // running maximum seen from the block base (>= 0)
        float l = 0.f, mx = d0, wmin = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (t0 + j < steps) {
                l += inc[j];
                mx = fmaxf(mx, l);
                wmin = fminf(wmin, l - mx);
                if (paths) paths[(int64_t)(t0 + j + 1) * n_paths + p] = fs0 * expf((float)base + l);
            }
        }
        if (mx > d0) runmax = base + (double)mx;
        worst = fmin(worst, (double)wmin);
        base += (double)l;
    }
    const double logS = base;
    finals[p] = (float)(s0 * exp(logS));
    maxdd[p] = (float)(1.0 - exp(worst));
}

// ---- joint paths of S <= 32 assets (portfolio value V_t = sum_i q_i s0_i exp(logS_i,t)) ----------
// One thread per path.  Each asset's log-price is kept as in mc_paths_kernel (fp32 within a Philox block of four steps,
// relative to an fp64 base), so asset i of a joint run computes exactly what the single-asset kernel computes from the
// same increments.  Counter = (path lo, hi, step/4, (factor << 8) | MODE): GBM factor 0 is mc_paths_kernel<0>'s stream,
// the bootstrap's one day-index stream is mc_paths_kernel<1>'s.
// Per-asset constants live in the parameter space (constant bank) and are indexed with compile-time offsets after
// unrolling, so every FMA of the mat-vec reads its Cholesky entry as an operand.  The fp64 bases live in shared memory
// (thread-private columns, touched once per block of four steps), which leaves the registers to z, l and A.
constexpr int JOINT_THREADS = 128;
constexpr int JOINT_MAX_ASSETS = 32;
constexpr int JOINT_MAX_TABLE = 12288;   // R * S floats of the bootstrap table (48 KB, the single-asset table's limit)

template <int SMAX>
struct JointParams {
    float L[SMAX * (SMAX + 1) / 2];   // Cholesky factor of the correlation, lower triangle packed by rows (GBM)
    float drift[SMAX], vol[SMAX];     // per-step drift / volatility, rounded to fp32 as mc_paths_kernel rounds them
    float w[SMAX];                    // q_i s0_i / V_0: the portfolio value is tracked relative to V_0
    double a[SMAX];                   // q_i s0_i
    double s0[SMAX];
    int S;
};

// V_t / V_0 = sum_i A_i exp(l_i), A_i = w_i exp(base_i); four partial sums shorten the dependent chain
template <int SMAX>
__device__ __forceinline__ float joint_value(const float (&A)[SMAX], const float (&l)[SMAX], int S) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < SMAX; ++i)
        if (i < S) acc[i & 3] = fmaf(A[i], __expf(l[i]), acc[i & 3]);
    return (acc[0] + acc[1]) + (acc[2] + acc[3]);
}

// (min. 1 block per SM: without it ptxas caps the 16-asset instances a few registers short and spills)
template <int MODE, int SMAX>
__global__ void __launch_bounds__(JOINT_THREADS, 1)
mc_joint_kernel(const __grid_constant__ JointParams<SMAX> P, const float* __restrict__ returns, int R, int block_len,
                int log_returns, int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset,
                float* __restrict__ finals, float* __restrict__ maxdd, float* __restrict__ asset_finals) {
    extern __shared__ double s_joint[];
    double* s_base = s_joint;                                            // [SMAX][JOINT_THREADS]
    float* s_ret = reinterpret_cast<float*>(s_joint + SMAX * JOINT_THREADS);   // [R][S] bootstrap table
    const int S = P.S;
    if (MODE == 1) stage_log_returns(s_ret, returns, R * S, log_returns);
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_paths) return;

    float l[SMAX], A[SMAX];
#pragma unroll
    for (int i = 0; i < SMAX; ++i) {
        l[i] = 0.f;
        A[i] = P.w[i];
        if (i < S) s_base[i * JOINT_THREADS + threadIdx.x] = 0.0;
    }
    float runmax = joint_value<SMAX>(A, l, S), dd = 0.f;
    BlockBootstrap boot;
    for (int t0 = 0; t0 < steps; t0 += 4) {
        float z[SMAX][4];   // GBM: four normals per factor, then (L z) in place
        int day[4];         // bootstrap: one day (row of the table) per step
        if (MODE == 0) {
#pragma unroll
            for (int k = 0; k < SMAX; ++k) {
                if (k < S) {
                    uint32_t x[4];
                    philox_path(seed, path_offset, p, (uint32_t)(t0 >> 2), ((uint32_t)k << 8) | (uint32_t)MODE, x);
                    box_muller(x[0], x[1], z[k][0], z[k][1]);
                    box_muller(x[2], x[3], z[k][2], z[k][3]);
                }
            }
            // bottom row first: row i reads z_0..z_i, which rows above it have not overwritten yet
#pragma unroll
            for (int i = SMAX - 1; i >= 0; --i) {
                if (i < S) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        float y = P.L[i * (i + 1) / 2] * z[0][j];
#pragma unroll
                        for (int k = 1; k <= i; ++k) y = fmaf(P.L[i * (i + 1) / 2 + k], z[k][j], y);
                        z[i][j] = y;
                    }
                }
            }
        } else {
            uint32_t x[4];
            philox_path(seed, path_offset, p, (uint32_t)(t0 >> 2), (uint32_t)MODE, x);
#pragma unroll
            for (int j = 0; j < 4; ++j) day[j] = boot.next(x[j], R, block_len) * S;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (t0 + j < steps) {
#pragma unroll
                for (int i = 0; i < SMAX; ++i)
                    if (i < S) l[i] += MODE == 0 ? fmaf(P.vol[i], z[i][j], P.drift[i]) : s_ret[day[j] + i];
                const float v = joint_value<SMAX>(A, l, S);
                runmax = fmaxf(runmax, v);
                dd = fmaxf(dd, 1.0f - __fdividef(v, runmax));   // (runmax_t - V_t) / runmax_t
            }
        }
#pragma unroll
        for (int i = 0; i < SMAX; ++i) {
            if (i < S) {
                double& b = s_base[i * JOINT_THREADS + threadIdx.x];
                const double nb = b + (double)l[i];
                b = nb;
                const float hi = (float)nb;   // exp(nb) = exp(hi) (1 + (nb - hi)) to fp32 accuracy
                A[i] = P.w[i] * expf(hi) * (1.0f + (float)(nb - (double)hi));
                l[i] = 0.f;
            }
        }
    }
    double v = 0.0;
#pragma unroll
    for (int i = 0; i < SMAX; ++i) {
        if (i < S) {
            const double e = exp(s_base[i * JOINT_THREADS + threadIdx.x]);
            v += P.a[i] * e;
            if (asset_finals) asset_finals[(int64_t)i * n_paths + p] = (float)(P.s0[i] * e);
        }
    }
    finals[p] = (float)v;
    maxdd[p] = dd;
}

// ---- exact order statistics: two-level radix select over fp32 keys ----------
__device__ __forceinline__ uint32_t ordered_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
    const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}

__global__ void sel_hist_hi(const float* __restrict__ x, int64_t n, unsigned* __restrict__ hist) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t k = ordered_key(x[i]) >> 16;
        // warp-aggregate equal bins (finals cluster in a few hundred bins)
        const unsigned peers = __match_any_sync(__activemask(), k);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[k], __popc(peers));
    }
}

// one block: for every rank find the high-16 bin holding it and the rank inside the bin
__global__ void __launch_bounds__(1024) sel_find_hi(const unsigned* __restrict__ hist, const int64_t* __restrict__ ranks, int n_ranks,
                            unsigned* __restrict__ bin_of, unsigned* __restrict__ rem_of) {
    __shared__ unsigned long long s_part[1024];
    const int tid = threadIdx.x;  // 1024 threads x 64 bins
    unsigned long long loc = 0;
    for (int j = 0; j < 64; ++j) loc += hist[tid * 64 + j];
    s_part[tid] = loc;
    __syncthreads();
    if (tid == 0) {
        unsigned long long run = 0;
        for (int i = 0; i < 1024; ++i) { const unsigned long long v = s_part[i]; s_part[i] = run; run += v; }
    }
    __syncthreads();
    const unsigned long long base = s_part[tid];
    for (int r = 0; r < n_ranks; ++r) {
        const unsigned long long k = (unsigned long long)ranks[r];
        if (k >= base && k < base + loc) {
            unsigned long long run = base;
            for (int j = 0; j < 64; ++j) {
                const unsigned c = hist[tid * 64 + j];
                if (k < run + c) { bin_of[r] = tid * 64 + j; rem_of[r] = (unsigned)(k - run); break; }
                run += c;
            }
        }
    }
}

__global__ void sel_hist_lo(const float* __restrict__ x, int64_t n, const unsigned* __restrict__ bin_of, int n_ranks,
                            unsigned* __restrict__ hist_lo /*[n_ranks][65536]*/) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t k = ordered_key(x[i]);
        const uint32_t hi = k >> 16, lo = k & 0xffffu;
        for (int r = 0; r < n_ranks; ++r) {
            if (bin_of[r] == hi && (r == 0 || bin_of[r - 1] != hi))  // ranks sharing a bin share its histogram
                atomicAdd(&hist_lo[(int64_t)r * 65536 + lo], 1u);
        }
    }
}

__global__ void __launch_bounds__(1024) sel_find_lo(const unsigned* __restrict__ hist_lo, const unsigned* __restrict__ bin_of,
                            const unsigned* __restrict__ rem_of, int n_ranks, float* __restrict__ out) {
    __shared__ unsigned s_part[1024];
    const int r = blockIdx.x, tid = threadIdx.x;
    int owner = r;
    while (owner > 0 && bin_of[owner - 1] == bin_of[r]) --owner;  // histogram owner for this bin
    const unsigned* h = hist_lo + (int64_t)owner * 65536;
    unsigned loc = 0;
    for (int j = 0; j < 64; ++j) loc += h[tid * 64 + j];
    s_part[tid] = loc;
    __syncthreads();
    if (tid == 0) {
        unsigned run = 0;
        for (int i = 0; i < 1024; ++i) { const unsigned v = s_part[i]; s_part[i] = run; run += v; }
    }
    __syncthreads();
    const unsigned base = s_part[tid], k = rem_of[r];
    if (k >= base && k < base + loc) {
        unsigned run = base;
        for (int j = 0; j < 64; ++j) {
            const unsigned c = h[tid * 64 + j];
            if (k < run + c) { out[r] = key_to_float((bin_of[r] << 16) | (unsigned)(tid * 64 + j)); break; }
            run += c;
        }
    }
}

// ---- moments --------------------------------------------------------------
// out[0]=sum x, out[1]=sum pct, out[2]=count(x > s0), out[3]=sum dd, out[4]=max dd,
// out[5]=sum pct[pct<=var], out[6]=count(pct<=var)   (var_thresh may be +inf on the first pass)
__global__ void mc_moments(const float* __restrict__ finals, const float* __restrict__ maxdd, int64_t n, double s0,
                           double var_thresh, double* __restrict__ out) {
    double a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0, a5 = 0, a6 = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double f = (double)finals[i];
        const double pct = (f / s0 - 1.0) * 100.0;  // monte_carlo_service.py:312
        a0 += f;
        a1 += pct;
        a2 += f > s0 ? 1.0 : 0.0;
        if (maxdd) { const double d = (double)maxdd[i]; a3 += d; a4 = fmax(a4, d); }
        if (pct <= var_thresh) { a5 += pct; a6 += 1.0; }
    }
    a0 = warp_sum_d(a0); a1 = warp_sum_d(a1); a2 = warp_sum_d(a2); a3 = warp_sum_d(a3);
    a4 = warp_max_d(a4); a5 = warp_sum_d(a5); a6 = warp_sum_d(a6);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&out[0], a0); atomicAdd(&out[1], a1); atomicAdd(&out[2], a2); atomicAdd(&out[3], a3);
        atomicAdd(&out[5], a5); atomicAdd(&out[6], a6);
        // max of non-negative doubles via their ordered bit patterns
        atomicMax(reinterpret_cast<unsigned long long*>(&out[4]), (unsigned long long)__double_as_longlong(a4));
    }
}

}  // namespace b200bt

using namespace b200bt;

static int mc_launch(int mode, double s0, double drift, double vol, const float* returns, int R, int block_len,
                     int log_returns, int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset, float* finals,
                     float* maxdd, float* paths, b200bt_stream_t stream) {
    B200BT_REQUIRE(finals && maxdd, B200BT_EINVAL, "mc: null output");
    B200BT_REQUIRE(n_paths > 0 && steps >= 0, B200BT_EINVAL, "mc: bad sizes");
    B200BT_REQUIRE(s0 > 0.0, B200BT_EINVAL, "mc: initial price must be positive");
    if (mode == 1) {
        B200BT_REQUIRE(returns && R > 0 && block_len > 0, B200BT_EINVAL, "mc_bootstrap: bad return sample");
        B200BT_REQUIRE((size_t)R * 4 <= 48 * 1024, B200BT_ELIMIT, "mc_bootstrap: at most 12288 returns");
    }
    int rc = check_device();
    if (rc) return rc;
    const unsigned blocks = (unsigned)((n_paths + MC_THREADS - 1) / MC_THREADS);
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == 0) {
        mc_paths_kernel<0><<<blocks, MC_THREADS, 0, st>>>(s0, drift, vol, nullptr, 0, 1, 1, n_paths, steps, seed,
                                                           path_offset, finals, maxdd, paths);
    } else {
        mc_paths_kernel<1><<<blocks, MC_THREADS, (size_t)R * 4, st>>>(s0, 0.0, 0.0, returns, R, block_len, log_returns,
                                                                       n_paths, steps, seed, path_offset, finals, maxdd, paths);
    }
    B200BT_LAUNCH_CHECK("mc launch");
    return B200BT_OK;
}

extern "C" int b200bt_mc_gbm(double s0, double mu, double sigma, double dt, int64_t n_paths, int steps, uint64_t seed,
                             uint64_t path_offset, float* finals, float* maxdd, float* paths, b200bt_stream_t stream) {
    // monte_carlo_service.py:273: (mu - 0.5*sigma**2)*dt + sigma*sqrt(dt)*Z
    const double drift = (mu - 0.5 * sigma * sigma) * dt;
    const double vol = sigma * sqrt(dt);
    return mc_launch(0, s0, drift, vol, nullptr, 0, 1, 1, n_paths, steps, seed, path_offset, finals, maxdd, paths, stream);
}

extern "C" int b200bt_mc_bootstrap(const float* returns, int R, int block_len, int log_returns, double s0,
                                   int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset, float* finals,
                                   float* maxdd, float* paths, b200bt_stream_t stream) {
    return mc_launch(1, s0, 0.0, 0.0, returns, R, block_len, log_returns, n_paths, steps, seed, path_offset, finals, maxdd,
                     paths, stream);
}

extern "C" int b200bt_select(const float* x, int64_t n, const int64_t* ranks_dev, int n_ranks, float* out,
                             void* workspace, int64_t workspace_bytes, b200bt_stream_t stream) {
    B200BT_REQUIRE(x && ranks_dev && out && workspace, B200BT_EINVAL, "select: null pointer");
    B200BT_REQUIRE(n > 0 && n_ranks > 0 && n_ranks <= 64, B200BT_EINVAL, "select: bad sizes");
    const int64_t need = b200bt_select_workspace_bytes(n_ranks);
    B200BT_REQUIRE(workspace_bytes >= need, B200BT_EINVAL, "select: workspace too small (%lld < %lld)",
                   (long long)workspace_bytes, (long long)need);
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned* hist = (unsigned*)workspace;
    unsigned* bin_of = hist + 65536;
    unsigned* rem_of = bin_of + 64;
    unsigned* hist_lo = rem_of + 64;
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)need, st);
    if (e != cudaSuccess) return cuda_status(e, "select: memset");
    const int64_t grid = (int64_t)device_sm_count() * 8;
    const int blocks = (int)((n + 255) / 256 < grid ? (n + 255) / 256 : grid);
    sel_hist_hi<<<blocks, 256, 0, st>>>(x, n, hist);
    B200BT_LAUNCH_CHECK("select hist_hi");
    sel_find_hi<<<1, 1024, 0, st>>>(hist, ranks_dev, n_ranks, bin_of, rem_of);
    B200BT_LAUNCH_CHECK("select find_hi");
    sel_hist_lo<<<blocks, 256, 0, st>>>(x, n, bin_of, n_ranks, hist_lo);
    B200BT_LAUNCH_CHECK("select hist_lo");
    sel_find_lo<<<n_ranks, 1024, 0, st>>>(hist_lo, bin_of, rem_of, n_ranks, out);
    B200BT_LAUNCH_CHECK("select find_lo");
    return B200BT_OK;
}

extern "C" int64_t b200bt_select_workspace_bytes(int n_ranks) {
    return (int64_t)(65536 + 128 + (int64_t)n_ranks * 65536) * 4;
}

extern "C" int b200bt_mc_moments(const float* finals, const float* maxdd, int64_t n, double s0, double var_threshold,
                                 double* out7, b200bt_stream_t stream) {
    B200BT_REQUIRE(finals && out7 && n > 0 && s0 > 0.0, B200BT_EINVAL, "mc_moments: bad argument");
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(out7, 0, 7 * sizeof(double), st);
    if (e != cudaSuccess) return cuda_status(e, "mc_moments: memset");
    const int64_t grid = (int64_t)device_sm_count() * 4;
    const int blocks = (int)((n + 255) / 256 < grid ? (n + 255) / 256 : grid);
    mc_moments<<<blocks, 256, 0, st>>>(finals, maxdd, n, s0, var_threshold, out7);
    B200BT_LAUNCH_CHECK("mc_moments");
    return B200BT_OK;
}

// ---- joint (portfolio) paths -----------------------------------------------------------------------
template <int SMAX>
static int joint_launch_bucket(int mode, int S, const double* s0, const double* qty, const double* drift,
                               const double* vol, const float* chol, const float* returns, int R, int block_len,
                               int log_returns, int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset,
                               float* finals, float* maxdd, float* asset_finals, cudaStream_t st) {
    JointParams<SMAX> P;
    memset(&P, 0, sizeof(P));
    P.S = S;
    double v0 = 0.0;
    for (int i = 0; i < S; ++i) v0 += qty[i] * s0[i];
    for (int i = 0; i < S; ++i) {
        P.a[i] = qty[i] * s0[i];
        P.s0[i] = s0[i];
        P.w[i] = (float)(P.a[i] / v0);
        if (mode == 0) {
            P.drift[i] = (float)drift[i];
            P.vol[i] = (float)vol[i];
            for (int k = 0; k <= i; ++k) P.L[i * (i + 1) / 2 + k] = chol[i * S + k];
        }
    }
    const unsigned blocks = (unsigned)((n_paths + JOINT_THREADS - 1) / JOINT_THREADS);
    size_t smem = (size_t)SMAX * JOINT_THREADS * sizeof(double);
    if (mode == 0) {
        mc_joint_kernel<0, SMAX><<<blocks, JOINT_THREADS, smem, st>>>(P, nullptr, 0, 1, 1, n_paths, steps, seed,
                                                                       path_offset, finals, maxdd, asset_finals);
    } else {
        smem += (size_t)R * S * sizeof(float);
        cudaError_t e = cudaFuncSetAttribute(mc_joint_kernel<1, SMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return cuda_status(e, "mc_portfolio_bootstrap: shared memory attribute");
        mc_joint_kernel<1, SMAX><<<blocks, JOINT_THREADS, smem, st>>>(P, returns, R, block_len, log_returns, n_paths,
                                                                       steps, seed, path_offset, finals, maxdd,
                                                                       asset_finals);
    }
    B200BT_LAUNCH_CHECK(mode == 0 ? "mc_portfolio_gbm" : "mc_portfolio_bootstrap");
    return B200BT_OK;
}

// Checks shared by both entry points, then dispatch on the smallest bucket that holds S assets.
static int joint_launch(int mode, int S, const double* s0, const double* qty, const double* drift, const double* vol,
                        const float* chol, const float* returns, int R, int block_len, int log_returns, int64_t n_paths,
                        int steps, uint64_t seed, uint64_t path_offset, float* finals, float* maxdd, float* asset_finals,
                        b200bt_stream_t stream) {
    B200BT_REQUIRE(S >= 1, B200BT_EINVAL, "mc_portfolio: need at least one asset (S = %d)", S);
    B200BT_REQUIRE(S <= JOINT_MAX_ASSETS, B200BT_ELIMIT, "mc_portfolio: at most %d assets (S = %d)", JOINT_MAX_ASSETS, S);
    B200BT_REQUIRE(s0 && qty && finals && maxdd, B200BT_EINVAL, "mc_portfolio: null pointer");
    B200BT_REQUIRE(n_paths > 0 && steps >= 0, B200BT_EINVAL, "mc_portfolio: bad sizes");
    double v0 = 0.0;
    for (int i = 0; i < S; ++i) {
        B200BT_REQUIRE(s0[i] > 0.0 && isfinite(s0[i]), B200BT_EINVAL, "mc_portfolio: initial price %d must be positive", i);
        B200BT_REQUIRE(qty[i] >= 0.0 && isfinite(qty[i]), B200BT_EINVAL, "mc_portfolio: quantity %d must be >= 0", i);
        v0 += qty[i] * s0[i];
    }
    B200BT_REQUIRE(v0 > 0.0 && isfinite(v0), B200BT_EINVAL, "mc_portfolio: initial portfolio value must be positive");
    if (mode == 0) {
        B200BT_REQUIRE(drift && vol && chol, B200BT_EINVAL, "mc_portfolio_gbm: null pointer");
        for (int i = 0; i < S; ++i) {
            B200BT_REQUIRE(isfinite(drift[i]) && isfinite(vol[i]), B200BT_EINVAL, "mc_portfolio_gbm: drift / vol %d", i);
            for (int k = 0; k <= i; ++k)
                B200BT_REQUIRE(isfinite(chol[i * S + k]), B200BT_EINVAL, "mc_portfolio_gbm: Cholesky entry (%d, %d)", i, k);
        }
    } else {
        B200BT_REQUIRE(returns && R > 0 && block_len > 0, B200BT_EINVAL, "mc_portfolio_bootstrap: bad return table");
        B200BT_REQUIRE((int64_t)R * S <= JOINT_MAX_TABLE, B200BT_ELIMIT,
                       "mc_portfolio_bootstrap: at most %d table entries (R x S = %lld)", JOINT_MAX_TABLE,
                       (long long)R * S);
    }
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
#define B200BT_JOINT_BUCKET(N)                                                                                          \
    joint_launch_bucket<N>(mode, S, s0, qty, drift, vol, chol, returns, R, block_len, log_returns, n_paths, steps, seed, \
                           path_offset, finals, maxdd, asset_finals, st)
    if (S <= 4) return B200BT_JOINT_BUCKET(4);
    if (S <= 8) return B200BT_JOINT_BUCKET(8);
    if (S <= 16) return B200BT_JOINT_BUCKET(16);
    return B200BT_JOINT_BUCKET(32);
#undef B200BT_JOINT_BUCKET
}

extern "C" int b200bt_mc_portfolio_gbm(int S, const double* s0_host, const double* qty_host, const double* drift_host,
                                       const double* vol_host, const float* chol_host, int64_t n_paths, int steps,
                                       uint64_t seed, uint64_t path_offset, float* finals, float* maxdd,
                                       float* asset_finals_or_null, b200bt_stream_t stream) {
    return joint_launch(0, S, s0_host, qty_host, drift_host, vol_host, chol_host, nullptr, 0, 1, 1, n_paths, steps, seed,
                        path_offset, finals, maxdd, asset_finals_or_null, stream);
}

extern "C" int b200bt_mc_portfolio_bootstrap(int S, const float* returns, int R, int block_len, int log_returns,
                                             const double* s0_host, const double* qty_host, int64_t n_paths, int steps,
                                             uint64_t seed, uint64_t path_offset, float* finals, float* maxdd,
                                             float* asset_finals_or_null, b200bt_stream_t stream) {
    return joint_launch(1, S, s0_host, qty_host, nullptr, nullptr, nullptr, returns, R, block_len, log_returns, n_paths,
                        steps, seed, path_offset, finals, maxdd, asset_finals_or_null, stream);
}
