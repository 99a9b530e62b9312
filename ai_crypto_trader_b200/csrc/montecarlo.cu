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

// mode 0: GBM.  mode 1: bootstrap of `returns` (R values, staged in shared memory),
// blocks of `block_len` consecutive returns (circular), log_returns selects compounding.
template <int MODE>
__global__ void __launch_bounds__(MC_THREADS)
mc_paths_kernel(double s0, double drift, double vol, const float* __restrict__ returns, int R, int block_len,
                int log_returns, int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset,
                float* __restrict__ finals, float* __restrict__ maxdd, float* __restrict__ paths) {
    extern __shared__ float s_ret[];
    if (MODE == 1) {
        for (int i = threadIdx.x; i < R; i += blockDim.x) {
            const float r = returns[i];
            s_ret[i] = log_returns ? r : log1pf(r);  // compounding in log space either way
        }
        __syncthreads();
    }
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_paths) return;
    const uint64_t gid = path_offset + (uint64_t)p;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    const uint32_t c0 = (uint32_t)gid, c1 = (uint32_t)(gid >> 32);

    // log-price relative to log(s0): block base `base` and running maximum `runmax` in fp64, the four
    // steps of a Philox block in fp32 relative to the base (their sum is folded into the base exactly)
    double base = 0.0, runmax = 0.0, worst = 0.0;
    const float fs0 = (float)s0, fdrift = (float)drift, fvol = (float)vol;
    if (paths) paths[p] = fs0;
    int boot_idx = 0, boot_left = 0;
    for (int t0 = 0; t0 < steps; t0 += 4) {
        uint32_t x[4];
        philox4x32_10(c0, c1, (uint32_t)(t0 >> 2), (uint32_t)MODE, k0, k1, x);
        float inc[4];
        if (MODE == 0) {
            float z[4];
            box_muller(x[0], x[1], z[0], z[1]);
            box_muller(x[2], x[3], z[2], z[3]);
#pragma unroll
            for (int j = 0; j < 4; ++j) inc[j] = fmaf(fvol, z[j], fdrift);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (boot_left == 0) {
                    boot_idx = (int)__umulhi(x[j], (uint32_t)R);  // uniform start in [0, R)
                    boot_left = block_len;
                } else {
                    boot_idx = boot_idx + 1 == R ? 0 : boot_idx + 1;
                }
                --boot_left;
                inc[j] = s_ret[boot_idx];
            }
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
    int rc = check_device();
    if (rc) return rc;
    const unsigned blocks = (unsigned)((n_paths + MC_THREADS - 1) / MC_THREADS);
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == 0) {
        mc_paths_kernel<0><<<blocks, MC_THREADS, 0, st>>>(s0, drift, vol, nullptr, 0, 1, 1, n_paths, steps, seed,
                                                           path_offset, finals, maxdd, paths);
    } else {
        B200BT_REQUIRE(returns && R > 0 && block_len > 0, B200BT_EINVAL, "mc_bootstrap: bad return sample");
        B200BT_REQUIRE((size_t)R * 4 <= 48 * 1024, B200BT_ELIMIT, "mc_bootstrap: at most 12288 returns");
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
