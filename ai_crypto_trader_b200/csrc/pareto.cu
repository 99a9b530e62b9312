// Multi-objective ranking of a GA population (NSGA-II, Deb, Pratap, Agarwal, Meyarivan 2002): the objective matrix from
// the lane stats, non-dominated fronts, crowding distance and the crowded order.  Contract: include/b200bt.h; restated
// by tests/pareto_ref.py.
//
// Schedule of b200bt_pareto_rank (n points, M objectives, W = ceil(n / 32) words per bit row):
//   prep       v[j][p] = (maximize_j ? obj : -obj), NaN -> -inf, column-major so that the tiles below load coalesced
//   dominance  every (q, p) pair, p tiled through shared memory 1024 at a time: bit p of row q is set iff q dominates p
//              (rows [n][W] uint32), and count[q] += #{p dominating q} (one integer atomic per warp and tile)
//   peel       one cooperative launch, one grid sync per front: the members of front k walk their bit rows and decrement
//              the counts of the points they dominate; a count reaching 0 appends its point to front k + 1 of the member
//              list.  Integer atomics only: the counts, the fronts and each front's member SET do not depend on their
//              order (the order within a front's slice of the list does, and no output reads it)
//   crowding   one thread per member: predecessor, successor, min and max of its front per objective from a scan over the
//              front's slice of the list (O(sum m_f^2 M)), order-free reductions, so the result is exact and deterministic
//   order      one thread per member: its position inside its front = #{front members before it in (crowding desc,
//              index asc)}; order[fstart + position] = p, key[p] = -(fstart + position)
#include <cooperative_groups.h>
#include <math.h>
#include "common.cuh"

namespace cg = cooperative_groups;

namespace b200bt {

constexpr int PR_MAX_N = 65536;
constexpr int PR_MAX_M = 8;
constexpr int OBJ_FIELDS = 19;           // b200bt_lane_stats fields 0..18 (trade_hash is not a number)
constexpr int DOM_TILE_WORDS = 32;       // a dominance tile: 32 words = 1024 points, one word per lane
constexpr int DOM_ROWS = 64;             // rows q per dominance block (8 warps x 8 rows)
constexpr int PEEL_THREADS = 512;

struct ObjFields { int f[PR_MAX_M]; };
struct ObjSense { int maximize[PR_MAX_M]; };

__global__ void objective_matrix_kernel(const b200bt_lane_stats* __restrict__ stats, int pop, int S, ObjFields F, int M,
                                        double* __restrict__ out, int64_t ld_out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)pop * M) return;
    const int i = (int)(t / M), j = (int)(t % M);
    const double* row = reinterpret_cast<const double*>(stats + (int64_t)i * S);
    const int field = F.f[j];
    double acc = 0.0;                    // fitness_reduce_kernel's expression (csrc/sweep.cu)
    for (int s = 0; s < S; ++s) acc += row[(int64_t)s * (sizeof(b200bt_lane_stats) / 8) + field];
    out[(int64_t)i * ld_out + j] = acc / (double)S;
}

__global__ void pareto_prep_kernel(const double* __restrict__ obj, int64_t ld, int n, int M, ObjSense D,
                                   double* __restrict__ v) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)n * M) return;
    const int j = (int)(t / n), p = (int)(t % n);
    const double x = obj[(int64_t)p * ld + j];
    const double y = D.maximize[j] ? x : -x;
    v[t] = isnan(y) ? -INFINITY : y;
}

// Block: 8 warps, lane = word of the tile, warp = row q (8 rows each).  Shared: the tile's values as sv[j][b * 33 + w]
// for point tile0 + 32 w + b, so that the 32 lanes read 32 consecutive doubles.  Points past n are NaN: no comparison
// with them is true, so they set no bit.
template <int M>
__global__ void __launch_bounds__(256) pareto_dominance_kernel(const double* __restrict__ v, int n, int W,
                                                               uint32_t* __restrict__ dom, int* __restrict__ count) {
    extern __shared__ double sv[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile0 = blockIdx.x * DOM_TILE_WORDS * 32;
    for (int t = threadIdx.x; t < 1024 * M; t += blockDim.x) {
        const int j = t >> 10, pl = t & 1023;
        const int p = tile0 + pl;
        sv[j * 1056 + (pl & 31) * 33 + (pl >> 5)] = p < n ? v[(int64_t)j * n + p] : NAN;
    }
    __syncthreads();
    const int w = blockIdx.x * DOM_TILE_WORDS + lane;
    for (int r = warp; r < DOM_ROWS; r += 8) {
        const int q = blockIdx.y * DOM_ROWS + r;
        if (q >= n) break;
        double vq[M];
#pragma unroll
        for (int j = 0; j < M; ++j) vq[j] = v[(int64_t)j * n + q];
        uint32_t word = 0;
        int dominated_by = 0;
#pragma unroll 4
        for (int b = 0; b < 32; ++b) {
            bool qp = true, pq = true;           // v[q] >= v[p] in every objective / v[p] >= v[q] in every objective
#pragma unroll
            for (int j = 0; j < M; ++j) {
                const double x = sv[j * 1056 + b * 33 + lane];
                qp &= vq[j] >= x;
                pq &= x >= vq[j];
            }
            word |= (uint32_t)(qp && !pq) << b;
            dominated_by += (pq && !qp);
        }
        if (w < W) dom[(int64_t)q * W + w] = word;
#pragma unroll
        for (int m = 16; m > 0; m >>= 1) dominated_by += __shfl_xor_sync(FULL, dominated_by, m);
        if (lane == 0 && dominated_by) atomicAdd(count + q, dominated_by);
    }
}

// ctr[0..2]: sizes of the fronts k, k + 1, k + 2 (mod 3) as they fill; ctr[3]: number of fronts.  fstart[k]: first slot of
// front k in `members`, fstart[#fronts] = n.
__global__ void __launch_bounds__(PEEL_THREADS) pareto_peel_kernel(const uint32_t* __restrict__ dom, int n, int W,
                                                                    int* count, int* members, int* fstart, int* ctr,
                                                                    int32_t* __restrict__ front) {
    cg::grid_group grid = cg::this_grid();
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = tid; p < n; p += stride)
        if (__ldcg(count + p) == 0) {
            front[p] = 0;
            members[atomicAdd(ctr, 1)] = (int)p;
        }
    grid.sync();
    int b = 0;
    for (int k = 0;; ++k) {
        const int e = b + __ldcg(ctr + k % 3);
        if (tid == 0) {
            fstart[k] = b;
            ctr[(k + 2) % 3] = 0;              // front k + 2's counter; its last reader passed the previous grid sync
        }
        if (e >= n || e == b) {                // every point has its front (e == b cannot happen: a DAG has a source)
            if (tid == 0) {
                fstart[k + 1] = e;
                ctr[3] = k + 1;
            }
            return;
        }
        const int64_t items = (int64_t)(e - b) * W;
        int* next = ctr + (k + 1) % 3;
        for (int64_t it = tid; it < items; it += stride) {
            const int q = __ldcg(members + b + it / W);
            const int w = (int)(it % W);
            uint32_t word = dom[(int64_t)q * W + w];
            while (word) {
                const int p = w * 32 + __ffs(word) - 1;
                word &= word - 1;
                if (atomicSub(count + p, 1) == 1) {
                    front[p] = k + 1;
                    members[e + atomicAdd(next, 1)] = p;
                }
            }
        }
        grid.sync();
        b = e;
    }
}

// Member slot -> its values in slot order (vc [M][n]).
__global__ void pareto_compact_kernel(const double* __restrict__ v, const int* __restrict__ members, int n, int M,
                                      double* __restrict__ vc) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)n * M) return;
    const int j = (int)(t / n), slot = (int)(t % n);
    vc[t] = v[(int64_t)j * n + members[slot]];
}

__global__ void pareto_crowding_kernel(const double* __restrict__ vc, const int* __restrict__ members,
                                       const int* __restrict__ fstart, const int32_t* __restrict__ front, int n, int M,
                                       double* __restrict__ crowding, double* __restrict__ crowd_slot) {
    const int slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n) return;
    const int p = members[slot];
    const int f = front[p];
    const int lo = fstart[f], hi = fstart[f + 1];
    double d = 0.0;
    for (int j = 0; j < M; ++j) {
        const double* col = vc + (int64_t)j * n;
        const double x = col[slot];
        bool has_prev = false, has_next = false;
        double prev = 0.0, next = 0.0, vmin = x, vmax = x;
        int iprev = -1, inext = -1;
        for (int s = lo; s < hi; ++s) {
            const double y = col[s];
            const int q = members[s];
            vmin = fmin(vmin, y);
            vmax = fmax(vmax, y);
            if (y < x || (y == x && q < p)) {              // before p in (value, index): keep the last such
                if (!has_prev || y > prev || (y == prev && q > iprev)) { prev = y; iprev = q; has_prev = true; }
            } else if (y > x || (y == x && q > p)) {       // after p: keep the first such
                if (!has_next || y < next || (y == next && q < inext)) { next = y; inext = q; has_next = true; }
            }
        }
        if (!has_prev || !has_next) {
            d = INFINITY;
        } else {
            const double r = __dsub_rn(vmax, vmin);
            if (r != 0.0 && isfinite(r)) d = __dadd_rn(d, __ddiv_rn(__dsub_rn(next, prev), r));
        }
    }
    crowding[p] = d;
    crowd_slot[slot] = d;
}

__global__ void pareto_order_kernel(const double* __restrict__ crowd_slot, const int* __restrict__ members,
                                    const int* __restrict__ fstart, const int32_t* __restrict__ front, int n,
                                    int32_t* __restrict__ order, double* __restrict__ key) {
    const int slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n) return;
    const int p = members[slot];
    const int f = front[p];
    const int lo = fstart[f], hi = fstart[f + 1];
    const double c = crowd_slot[slot];
    int pos = lo;
    for (int s = lo; s < hi; ++s) {
        const double y = crowd_slot[s];
        pos += (y > c || (y == c && members[s] < p));
    }
    order[pos] = p;
    if (key) key[p] = (double)(-pos);      // +0.0 for the first
}

struct ParetoLayout {
    int64_t v, vc, crowd, dom, count, members, fstart, ctr, total;
};

static int64_t align256(int64_t x) { return (x + 255) & ~(int64_t)255; }

static ParetoLayout pareto_layout(int n, int M) {
    const int64_t W = (n + 31) / 32;
    ParetoLayout L;
    int64_t o = 0;
    L.v = o;        o = align256(o + (int64_t)n * M * 8);
    L.vc = o;       o = align256(o + (int64_t)n * M * 8);
    L.crowd = o;    o = align256(o + (int64_t)n * 8);
    L.dom = o;      o = align256(o + (int64_t)n * W * 4);
    L.count = o;    o = align256(o + (int64_t)n * 4);
    L.members = o;  o = align256(o + (int64_t)n * 4);
    L.fstart = o;   o = align256(o + ((int64_t)n + 1) * 4);
    L.ctr = o;      o = align256(o + 4 * 4);
    L.total = o;
    return L;
}

template <int M>
static int launch_dominance(const double* v, int n, int W, uint32_t* dom, int* count, cudaStream_t st) {
    const size_t smem = (size_t)M * 1056 * 8;
    const int rc = cuda_status(cudaFuncSetAttribute(pareto_dominance_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                    (int)smem), "pareto dominance smem");
    if (rc) return rc;
    dim3 grid((unsigned)((W + DOM_TILE_WORDS - 1) / DOM_TILE_WORDS), (unsigned)((n + DOM_ROWS - 1) / DOM_ROWS));
    pareto_dominance_kernel<M><<<grid, 256, smem, st>>>(v, n, W, dom, count);
    B200BT_LAUNCH_CHECK("pareto dominance");
    return B200BT_OK;
}

}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_objective_matrix(const b200bt_lane_stats* stats, int pop, int S, const int* fields_host, int M,
                                       double* out, int64_t ld_out, b200bt_stream_t stream) {
    B200BT_REQUIRE(stats && fields_host && out, B200BT_EINVAL, "objective_matrix: null pointer");
    B200BT_REQUIRE(pop >= 1 && S >= 1 && M >= 1, B200BT_EINVAL, "objective_matrix: pop, S and M must be >= 1");
    B200BT_REQUIRE(M <= PR_MAX_M, B200BT_ELIMIT, "objective_matrix: at most %d objectives (M = %d)", PR_MAX_M, M);
    B200BT_REQUIRE(ld_out >= M, B200BT_EINVAL, "objective_matrix: row stride %lld below M = %d", (long long)ld_out, M);
    ObjFields F;
    for (int j = 0; j < PR_MAX_M; ++j) F.f[j] = 0;
    for (int j = 0; j < M; ++j) {
        B200BT_REQUIRE(fields_host[j] >= 0 && fields_host[j] < OBJ_FIELDS, B200BT_EINVAL,
                       "objective_matrix: field %d of objective %d is not a lane-stat number (0..%d)", fields_host[j], j,
                       OBJ_FIELDS - 1);
        F.f[j] = fields_host[j];
    }
    int rc = check_device();
    if (rc) return rc;
    const int64_t t = (int64_t)pop * M;
    objective_matrix_kernel<<<(unsigned)((t + 255) / 256), 256, 0, (cudaStream_t)stream>>>(stats, pop, S, F, M, out, ld_out);
    B200BT_LAUNCH_CHECK("objective_matrix");
    return B200BT_OK;
}

extern "C" int64_t b200bt_pareto_workspace_bytes(int n, int M) {
    if (n < 1 || n > PR_MAX_N || M < 1 || M > PR_MAX_M) return 0;
    return pareto_layout(n, M).total;
}

extern "C" int b200bt_pareto_rank(const double* obj, int64_t ld, int n, int M, const int* maximize_host, void* workspace,
                                  int64_t workspace_bytes, int32_t* front, double* crowding, int32_t* order,
                                  double* key_or_null, b200bt_stream_t stream) {
    B200BT_REQUIRE(obj && maximize_host && workspace && front && crowding && order, B200BT_EINVAL,
                   "pareto_rank: null pointer");
    B200BT_REQUIRE(n >= 1 && M >= 1, B200BT_EINVAL, "pareto_rank: n and M must be >= 1");
    B200BT_REQUIRE(n <= PR_MAX_N, B200BT_ELIMIT, "pareto_rank: at most %d points (n = %d)", PR_MAX_N, n);
    B200BT_REQUIRE(M <= PR_MAX_M, B200BT_ELIMIT, "pareto_rank: at most %d objectives (M = %d)", PR_MAX_M, M);
    B200BT_REQUIRE(ld >= M, B200BT_EINVAL, "pareto_rank: row stride %lld below M = %d", (long long)ld, M);
    const ParetoLayout L = pareto_layout(n, M);
    B200BT_REQUIRE(workspace_bytes >= L.total, B200BT_EINVAL, "pareto_rank: workspace too small (%lld < %lld)",
                   (long long)workspace_bytes, (long long)L.total);
    B200BT_REQUIRE(((uintptr_t)workspace & 255) == 0, B200BT_EINVAL, "pareto_rank: workspace must be 256-byte aligned");
    ObjSense D;
    for (int j = 0; j < PR_MAX_M; ++j) D.maximize[j] = j < M ? (maximize_host[j] != 0) : 1;
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    double* v = (double*)(ws + L.v);
    double* vc = (double*)(ws + L.vc);
    double* crowd_slot = (double*)(ws + L.crowd);
    uint32_t* dom = (uint32_t*)(ws + L.dom);
    int* count = (int*)(ws + L.count);
    int* members = (int*)(ws + L.members);
    int* fstart = (int*)(ws + L.fstart);
    int* ctr = (int*)(ws + L.ctr);
    const int W = (n + 31) / 32;
    const int64_t nm = (int64_t)n * M;

    pareto_prep_kernel<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(obj, ld, n, M, D, v);
    B200BT_LAUNCH_CHECK("pareto prep");
    if ((rc = cuda_status(cudaMemsetAsync(count, 0, (size_t)n * 4, st), "pareto_rank memset"))) return rc;
    if ((rc = cuda_status(cudaMemsetAsync(ctr, 0, 4 * 4, st), "pareto_rank memset"))) return rc;
    switch (M) {
        case 1: rc = launch_dominance<1>(v, n, W, dom, count, st); break;
        case 2: rc = launch_dominance<2>(v, n, W, dom, count, st); break;
        case 3: rc = launch_dominance<3>(v, n, W, dom, count, st); break;
        case 4: rc = launch_dominance<4>(v, n, W, dom, count, st); break;
        case 5: rc = launch_dominance<5>(v, n, W, dom, count, st); break;
        case 6: rc = launch_dominance<6>(v, n, W, dom, count, st); break;
        case 7: rc = launch_dominance<7>(v, n, W, dom, count, st); break;
        default: rc = launch_dominance<8>(v, n, W, dom, count, st); break;
    }
    if (rc) return rc;

    // the peel: as many co-resident blocks as the work can use, at most two per SM (a grid sync per front costs more with
    // more blocks, and the chain of n fronts is nothing but grid syncs)
    int per_sm = 0;
    if ((rc = cuda_status(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pareto_peel_kernel, PEEL_THREADS, 0),
                          "pareto peel occupancy")))
        return rc;
    per_sm = per_sm < 2 ? per_sm : 2;
    B200BT_REQUIRE(per_sm >= 1, B200BT_ELIMIT, "pareto_rank: the peel kernel cannot be resident");
    int64_t blocks = (int64_t)device_sm_count() * per_sm;
    const int64_t want = ((int64_t)n * W + PEEL_THREADS - 1) / PEEL_THREADS;
    if (blocks > want) blocks = want;
    if (blocks < 1) blocks = 1;
    int n_ = n, W_ = W;
    void* args[] = {(void*)&dom, (void*)&n_, (void*)&W_, (void*)&count, (void*)&members, (void*)&fstart, (void*)&ctr,
                    (void*)&front};
    if ((rc = cuda_status(cudaLaunchCooperativeKernel((const void*)pareto_peel_kernel, dim3((unsigned)blocks),
                                                      dim3(PEEL_THREADS), args, 0, st), "pareto peel")))
        return rc;
    B200BT_LAUNCH_CHECK("pareto peel");

    pareto_compact_kernel<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(v, members, n, M, vc);
    B200BT_LAUNCH_CHECK("pareto compact");
    pareto_crowding_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(vc, members, fstart, front, n, M, crowding,
                                                                        crowd_slot);
    B200BT_LAUNCH_CHECK("pareto crowding");
    pareto_order_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(crowd_slot, members, fstart, front, n, order,
                                                                     key_or_null);
    B200BT_LAUNCH_CHECK("pareto order");
    return B200BT_OK;
}
