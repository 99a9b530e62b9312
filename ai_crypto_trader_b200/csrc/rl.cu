// Reinforcement-learning agents of the strategy-evolution service (sm_90a): services/reinforcement_learning.py's
// TradingRLAgent (NumPy path) trained by optimize_with_reinforcement_learning over market history, for a population of
// agents at once.  Contract and the rules restated: include/b200bt.h (b200bt_rl_*); design: DESIGN.md section 3.15.
//
// rl_states_kernel  one thread per (symbol, bar): the 16 features of _convert_market_data_to_state as float64.
// rl_train_kernel   one warp (one CTA) per agent.  The online and target networks live in shared memory (W2 rows padded
//                   to 25 doubles so that the lane-per-unit passes read them without bank conflicts).  The forward passes
//                   of a replay that do not depend on each other -- current_q and next_q of the minibatch, the loss pass --
//                   run one sample per lane; the per-sample SGD steps run one hidden unit per lane (lanes 0..23), one
//                   sample after the other.  Replay memory is a ring of 8-byte words (point, action, done) in the agent
//                   state; states and rewards are re-derived from the state table.
// Every float64 operation is an explicit _rn intrinsic (no contraction) and every sum runs in index order from its first
// term, so tests/rl_ref.py restates the kernel exactly.
#include <math.h>
#include "common.cuh"
#include "philox.cuh"

namespace b200bt {
namespace {

constexpr int IN = B200BT_RL_FEATURES, HID = 24, OUT = 3;
constexpr int W1 = 0, B1 = W1 + IN * HID, W2 = B1 + HID, B2 = W2 + HID * HID, W3 = B2 + HID, B3 = W3 + HID * OUT;
static_assert(B3 + OUT == B200BT_RL_PARAMS, "parameter layout");
constexpr int W2_LD = HID + 1;                                  // shared-memory row stride of W2
constexpr int SW2 = W2, SB2 = SW2 + HID * W2_LD, SW3 = SB2 + HID, SB3 = SW3 + HID * OUT, SNET = SB3 + OUT + 1;
constexpr int MAX_BATCH = B200BT_RL_MAX_BATCH;
constexpr uint32_t STREAM_INIT = 0, STREAM_ACT = 1, STREAM_SAMPLE = 2;
constexpr int T_BITS = 40;

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double relu(double z) { return z <= 0.0 ? 0.0 : z; }       // np.maximum(0, z): NaN stays

// canonical parameter index -> shared-memory index
__device__ __forceinline__ int sidx(int e) {
    if (e < W2) return e;
    if (e < B2) { const int r = e - W2; return SW2 + (r / HID) * W2_LD + r % HID; }
    return e - B2 + SB2;
}

// ---- states ---------------------------------------------------------------------------------------------------------
__global__ void rl_states_kernel(const float* __restrict__ cols, const float* __restrict__ close,
                                 const float* __restrict__ volume, int64_t ld, int S, int64_t N, int h1, int h24,
                                 double* __restrict__ out) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (int64_t)S * N) return;
    const int s = (int)(g / N);
    const int64_t t = g % N;
    const int64_t SN = (int64_t)S * N;
    auto col = [&](int c) { return (double)cols[c * SN + g]; };
    const float* cr = close + (int64_t)s * ld;
    const double p = (double)cr[t];
    double f[IN];
    f[0] = __ddiv_rn(col(B200BT_COL_RSI), 100.0);
    f[1] = __ddiv_rn(dadd(col(B200BT_COL_MACD), 1.0), 2.0);
    f[2] = __ddiv_rn(dadd(col(B200BT_COL_MACD_SIGNAL), 1.0), 2.0);
    if (p > 0.0) {
        const double up = col(B200BT_COL_BB_HIGH), mid = col(B200BT_COL_BB_MID), lo = col(B200BT_COL_BB_LOW);
        const double range = dsub(up, lo);
        f[3] = range > 0.0 ? __ddiv_rn(dsub(up, p), range) : 0.5;
        f[4] = range > 0.0 ? __ddiv_rn(dsub(p, lo), range) : 0.5;
        f[5] = __ddiv_rn(dsub(p, mid), p);
        f[6] = __ddiv_rn(col(B200BT_COL_EMA_12), p);
        f[7] = __ddiv_rn(col(B200BT_COL_EMA_26), p);
        f[8] = __ddiv_rn(col(B200BT_COL_ATR), p);
    } else {
        f[3] = f[4] = f[5] = 0.5;
        f[6] = f[7] = 1.0;
        f[8] = 0.0;
    }
    const double v = __ddiv_rn((double)volume[(int64_t)s * ld + t], 1000000.0);
    f[9] = 1.0 < v ? 1.0 : v;                                    // min(v, 1)
    double pc1 = 0.0, pc24 = 0.0;
    if (t >= h1) { const double c0 = (double)cr[t - h1]; pc1 = __ddiv_rn(dmul(100.0, dsub(p, c0)), c0); }
    if (t >= h24) { const double c0 = (double)cr[t - h24]; pc24 = __ddiv_rn(dmul(100.0, dsub(p, c0)), c0); }
    f[10] = __ddiv_rn(dadd(pc1, 10.0), 20.0);
    f[11] = __ddiv_rn(dadd(pc24, 30.0), 60.0);
    f[12] = 0.5;                                                 // social defaults 50, 0, 0
    f[13] = 0.0;
    f[14] = 0.0;
    const double sma20 = col(B200BT_COL_SMA_20), sma50 = col(B200BT_COL_SMA_50);
    f[15] = (p > sma20 && sma20 > sma50) ? 0.8 : (p < sma20 && sma20 < sma50) ? 0.2 : 0.5;
    double* o = out + g * IN;
#pragma unroll
    for (int i = 0; i < IN; ++i) o[i] = f[i];
}

// ---- training -------------------------------------------------------------------------------------------------------
// _calculate_reward (strategy_evolution_service.py:849-899) from the state of point t and of its next point
__device__ double reward(int a, const double* __restrict__ s, const double* __restrict__ ns) {
    const double pc = dmul(dsub(ns[10], 0.5), 2.0);
    double r;
    if (a == 0) {
        r = pc;
        if (s[0] < 0.3) r = dadd(r, 0.2);
        if (s[12] > 0.6) r = dadd(r, 0.1);
        if (s[4] < 0.2) r = dadd(r, 0.2);
    } else if (a == 2) {
        r = -pc;
        if (s[0] > 0.7) r = dadd(r, 0.2);
        if (s[12] < 0.4) r = dadd(r, 0.1);
        if (s[3] > 0.8) r = dadd(r, 0.2);
    } else {
        r = fabs(pc) < 0.01 ? 0.05 : (0.4 <= s[0] && s[0] <= 0.6) ? 0.05 : -0.05;
    }
    return r;
}

// sum(rewards) from the int 0 as Python 3.12 adds floats: Neumaier's compensated sum, the compensation added at the end
// when it is nonzero and finite
struct PySum {
    double f = 0.0, c = 0.0;
    bool first = true;
    __device__ void add(double x) {
        if (first) { f = dadd(0.0, x); first = false; return; }
        const double t = dadd(f, x);
        c = fabs(f) >= fabs(x) ? dadd(c, dadd(dsub(f, t), x)) : dadd(c, dadd(dsub(x, t), f));
        f = t;
    }
    __device__ double value() const { return (c != 0.0 && isfinite(c)) ? dadd(f, c) : f; }
};

__device__ __forceinline__ double max3(const double* q) {
    double m = q[0];
    if (q[1] > m) m = q[1];
    if (q[2] > m) m = q[2];
    return m;
}

// one forward pass by one thread (weights in shared memory: every lane reads the same word, a broadcast)
__device__ __forceinline__ void forward_lane(const double* __restrict__ W, const double* __restrict__ s, double q[OUT]) {
    double x[IN], a2[HID];
#pragma unroll
    for (int i = 0; i < IN; ++i) x[i] = s[i];
#pragma unroll
    for (int j = 0; j < HID; ++j) {
        double h = dmul(x[0], W[W1 + j]);
#pragma unroll
        for (int i = 1; i < IN; ++i) h = dadd(h, dmul(x[i], W[W1 + i * HID + j]));
        h = relu(dadd(h, W[B1 + j]));
#pragma unroll
        for (int k = 0; k < HID; ++k) {
            const double p = dmul(h, W[SW2 + j * W2_LD + k]);
            a2[k] = j == 0 ? p : dadd(a2[k], p);
        }
    }
#pragma unroll
    for (int k = 0; k < HID; ++k) {
        const double h2 = relu(dadd(a2[k], W[SB2 + k]));
#pragma unroll
        for (int o = 0; o < OUT; ++o) {
            const double p = dmul(h2, W[SW3 + k * OUT + o]);
            q[o] = k == 0 ? p : dadd(q[o], p);
        }
    }
#pragma unroll
    for (int o = 0; o < OUT; ++o) q[o] = dadd(q[o], W[SB3 + o]);
}

struct Scratch {                     // per-agent shared scratch next to the two networks
    double target[MAX_BATCH][OUT];
    double maxq[MAX_BATCH];
    double err[MAX_BATCH];
    double s[IN], h1[HID], h2[HID], d_out[4], d_h2[HID], d_h1[HID], q[4];
    uint64_t word[MAX_BATCH];
    int32_t pick[MAX_BATCH];
};

// forward pass of one state with one hidden unit per lane; q -> sc.q (all lanes see it after the call)
__device__ void forward_warp(const double* __restrict__ W, const double* __restrict__ s, Scratch& sc, int lane) {
    if (lane < HID) {
        double h = dmul(s[0], W[W1 + lane]);
#pragma unroll
        for (int i = 1; i < IN; ++i) h = dadd(h, dmul(s[i], W[W1 + i * HID + lane]));
        sc.h1[lane] = relu(dadd(h, W[B1 + lane]));
    }
    __syncwarp();
    if (lane < HID) {
        double h = dmul(sc.h1[0], W[SW2 + lane]);
#pragma unroll
        for (int j = 1; j < HID; ++j) h = dadd(h, dmul(sc.h1[j], W[SW2 + j * W2_LD + lane]));
        sc.h2[lane] = relu(dadd(h, W[SB2 + lane]));
    }
    __syncwarp();
    if (lane < OUT) {
        double o = dmul(sc.h2[0], W[SW3 + lane]);
#pragma unroll
        for (int k = 1; k < HID; ++k) o = dadd(o, dmul(sc.h2[k], W[SW3 + k * OUT + lane]));
        sc.q[lane] = dadd(o, W[SB3 + lane]);
    }
    __syncwarp();
}

// one SGD step of _numpy_train (reinforcement_learning.py:204-235) on the state in sc.s towards target tg
__device__ void sgd_step(double* __restrict__ W, const double* __restrict__ tg, double alpha, Scratch& sc, int lane) {
    forward_warp(W, sc.s, sc, lane);
    if (lane < OUT) sc.d_out[lane] = dsub(sc.q[lane], tg[lane]);
    __syncwarp();
    if (lane < HID) {                                             // d_hidden2 = d_output . W3^T, masked where hidden2 <= 0
        double d = dmul(sc.d_out[0], W[SW3 + lane * OUT]);
        d = dadd(d, dmul(sc.d_out[1], W[SW3 + lane * OUT + 1]));
        d = dadd(d, dmul(sc.d_out[2], W[SW3 + lane * OUT + 2]));
        sc.d_h2[lane] = sc.h2[lane] <= 0.0 ? 0.0 : d;
    }
    __syncwarp();
    if (lane < HID) {                                             // d_hidden1 = d_hidden2 . W2^T, masked, pre-update W2
        double d = dmul(sc.d_h2[0], W[SW2 + lane * W2_LD]);
#pragma unroll
        for (int k = 1; k < HID; ++k) d = dadd(d, dmul(sc.d_h2[k], W[SW2 + lane * W2_LD + k]));
        sc.d_h1[lane] = sc.h1[lane] <= 0.0 ? 0.0 : d;
    }
    __syncwarp();
    // w -= alpha * d for every parameter (each is updated once, so the reference's W3, b3, W2, ... order is moot)
    for (int e = lane; e < IN * HID; e += 32)
        W[W1 + e] = dsub(W[W1 + e], dmul(alpha, dmul(sc.s[e / HID], sc.d_h1[e % HID])));
    for (int e = lane; e < HID * HID; e += 32) {
        const int j = e / HID, k = e % HID;
        W[SW2 + j * W2_LD + k] = dsub(W[SW2 + j * W2_LD + k], dmul(alpha, dmul(sc.h1[j], sc.d_h2[k])));
    }
    for (int e = lane; e < HID * OUT; e += 32)
        W[SW3 + e] = dsub(W[SW3 + e], dmul(alpha, dmul(sc.h2[e / OUT], sc.d_out[e % OUT])));
    if (lane < HID) {
        W[B1 + lane] = dsub(W[B1 + lane], dmul(alpha, sc.d_h1[lane]));
        W[SB2 + lane] = dsub(W[SB2 + lane], dmul(alpha, sc.d_h2[lane]));
    }
    if (lane < OUT) W[SB3 + lane] = dsub(W[SB3 + lane], dmul(alpha, sc.d_out[lane]));
    __syncwarp();
}

__device__ __forceinline__ uint64_t rl_word(int64_t t, int a, bool done) {
    return (uint64_t)t | ((uint64_t)a << T_BITS) | ((uint64_t)done << (T_BITS + 2));
}
__device__ __forceinline__ int64_t word_t(uint64_t w) { return (int64_t)(w & ((1ull << T_BITS) - 1)); }
__device__ __forceinline__ int word_a(uint64_t w) { return (int)((w >> T_BITS) & 3u); }
__device__ __forceinline__ bool word_done(uint64_t w) { return (w >> (T_BITS + 2)) & 1u; }

// GaRng of (agent, stream) positioned after `pos` words
__device__ GaRng rng_at(uint64_t seed, uint64_t gid, uint32_t stream, uint64_t pos) {
    GaRng r(seed, (uint32_t)(gid >> 32), (uint32_t)gid, stream);
    r.blk = (uint32_t)(pos >> 2);
    if (pos & 3u) {
        philox4x32_10(r.c0, r.c1, r.c2, r.blk++, r.k0, r.k1, r.x);
        r.have = 4u - (uint32_t)(pos & 3u);
    }
    return r;
}
__device__ __forceinline__ uint64_t rng_pos(const GaRng& r) { return 4ull * r.blk - r.have; }

__global__ void __launch_bounds__(32) rl_train_kernel(
        const double* __restrict__ states, int64_t N, const b200bt_rl_agent* __restrict__ agents, int64_t agent_offset,
        int64_t stride, unsigned char* __restrict__ agent_state, const int64_t* __restrict__ call_end, int n_calls,
        int points, const double* __restrict__ init_weights, double* __restrict__ avg_reward, double* __restrict__ q_out,
        double* __restrict__ history, int64_t history_rows) {
    extern __shared__ __align__(16) double smem[];
    double* Wo = smem;                    // online network
    double* Wt = smem + SNET;             // target network
    Scratch& sc = *reinterpret_cast<Scratch*>(smem + 2 * SNET);
    const int lane = threadIdx.x;
    const int64_t a_idx = blockIdx.x;
    const b200bt_rl_agent ag = agents[a_idx];
    const uint64_t gid = (uint64_t)agent_offset + (uint64_t)a_idx;
    unsigned char* base = agent_state + a_idx * stride;
    b200bt_rl_agent_state* hdr = reinterpret_cast<b200bt_rl_agent_state*>(base);
    double* g_online = reinterpret_cast<double*>(base + sizeof(b200bt_rl_agent_state));
    double* g_target = g_online + B200BT_RL_PARAMS;
    uint64_t* ring = reinterpret_cast<uint64_t*>(g_target + B200BT_RL_PARAMS);
    const double* S0 = states + (int64_t)ag.symbol * N * IN;

    b200bt_rl_agent_state st = *hdr;
    if (!st.initialized) {
        if (init_weights) {
            for (int e = lane; e < B200BT_RL_PARAMS; e += 32) Wo[sidx(e)] = init_weights[a_idx * B200BT_RL_PARAMS + e];
        } else {
            // randn * 0.1 for W1, W2, W3 in that order, biases 0 (reinforcement_learning.py:142-147): normal pair p is
            // Box-Muller of INIT block p (u1 from words 3, 2; u2 from words 1, 0)
            for (int e = lane; e < B200BT_RL_PARAMS; e += 32) Wo[sidx(e)] = 0.0;
            __syncwarp();
            constexpr int NW = IN * HID + HID * HID + HID * OUT;
            for (int p = lane; p < NW / 2; p += 32) {
                uint32_t x[4];
                philox4x32_10((uint32_t)gid, (uint32_t)(gid >> 32), STREAM_INIT, (uint32_t)p, (uint32_t)ag.seed,
                              (uint32_t)(ag.seed >> 32), x);
                const double u1 = dadd(dmul((double)(x[3] >> 5), 67108864.0), (double)(x[2] >> 6)) * (1.0 / 9007199254740992.0);
                const double u2 = dadd(dmul((double)(x[1] >> 5), 67108864.0), (double)(x[0] >> 6)) * (1.0 / 9007199254740992.0);
                const double r = sqrt(dmul(-2.0, log(dsub(1.0, u1))));
                const double ang = dmul(6.283185307179586, u2);
                const double z[2] = {dmul(r, cos(ang)), dmul(r, sin(ang))};
                for (int h = 0; h < 2; ++h) {
                    const int n = 2 * p + h;
                    const int e = n < IN * HID ? W1 + n : n < IN * HID + HID * HID ? W2 + (n - IN * HID) : W3 + (n - IN * HID - HID * HID);
                    Wo[sidx(e)] = dmul(z[h], 0.1);
                }
            }
        }
        __syncwarp();
        for (int e = lane; e < SNET; e += 32) Wt[e] = Wo[e];
        st.initialized = 1;
        st.n_transitions = 0;
        st.replays = 0;
        st.epsilon = ag.epsilon_start;
        st.act_words = 0;
        st.sample_words = 0;
        st.mean_q = NAN;
    } else {
        for (int e = lane; e < B200BT_RL_PARAMS; e += 32) {
            Wo[sidx(e)] = g_online[e];
            Wt[sidx(e)] = g_target[e];
        }
    }
    __syncwarp();

    GaRng act = rng_at(ag.seed, gid, STREAM_ACT, st.act_words);
    GaRng smp = rng_at(ag.seed, gid, STREAM_SAMPLE, st.sample_words);
    const int B = ag.batch_size, M = ag.memory_size;
    int64_t row = 0;
    for (int c = 0; c < n_calls; ++c) {
        const int64_t end = call_end[c];
        const int64_t lo = end - points + 1 > 0 ? end - points + 1 : 0;
        PySum rsum;
        for (int64_t t = lo; t <= end; ++t) {
            const double* s = S0 + t * IN;
            // act (:292-318)
            int a;
            if (act.uniform() < st.epsilon) {
                a = (int)act.below(3u);
            } else {
                forward_warp(Wo, s, sc, lane);
                a = 0;
                if (sc.q[1] > sc.q[a]) a = 1;
                if (sc.q[2] > sc.q[a]) a = 2;
            }
            const bool done = t == end;
            rsum.add(reward(a, s, S0 + (done ? t : t + 1) * IN));
            // remember (:320-333): a deque of maxlen M as a ring
            if (lane == 0) ring[st.n_transitions % M] = rl_word(t, a, done);
            ++st.n_transitions;
            const int64_t fill = st.n_transitions < M ? st.n_transitions : M;
            if (fill < B) continue;
            __syncwarp();
            // replay (:335-419). 1. random.sample: B distinct deque positions, in draw order
            for (int i = 0; i < B; ++i) {
                uint32_t cand;
                while (true) {
                    cand = smp.below((uint32_t)fill);
                    bool dup = false;
                    for (int u = lane; u < i; u += 32) dup = dup || sc.pick[u] == (int32_t)cand;
                    if (!__any_sync(FULL, dup)) break;
                }
                if (lane == 0) sc.pick[i] = (int32_t)cand;
                __syncwarp();
            }
            const int64_t oldest = st.n_transitions - fill;
            for (int i = lane; i < B; i += 32) sc.word[i] = ring[(oldest + sc.pick[i]) % M];
            __syncwarp();
            // 2-3. current_q (online), next_q (target), targets; one sample per lane
            for (int i = lane; i < B; i += 32) {
                const uint64_t w = sc.word[i];
                const int64_t ti = word_t(w);
                const bool di = word_done(w);
                const int ai = word_a(w);
                const double* si = S0 + ti * IN;
                const double* ni = S0 + (di ? ti : ti + 1) * IN;
                double cq[OUT], nq[OUT];
                forward_lane(Wo, si, cq);
                forward_lane(Wt, ni, nq);
                const double r = reward(ai, si, ni);
#pragma unroll
                for (int o = 0; o < OUT; ++o) sc.target[i][o] = cq[o];
                sc.target[i][ai] = di ? r : dadd(r, dmul(ag.gamma, max3(nq)));
                sc.maxq[i] = max3(cq);
            }
            __syncwarp();
            // 4. one SGD step per sample in minibatch order
            for (int i = 0; i < B; ++i) {
                if (lane < IN) sc.s[lane] = S0[word_t(sc.word[i]) * IN + lane];
                __syncwarp();
                sgd_step(Wo, sc.target[i], ag.learning_rate, sc, lane);
            }
            // 5. loss of the post-update outputs (only the history reports it)
            double loss = NAN;
            if (history) {
                for (int i = lane; i < B; i += 32) {
                    double q[OUT];
                    forward_lane(Wo, S0 + word_t(sc.word[i]) * IN, q);
                    double e = 0.0;
#pragma unroll
                    for (int o = 0; o < OUT; ++o) {
                        const double d = dsub(q[o], sc.target[i][o]);
                        e = o == 0 ? dmul(d, d) : dadd(e, dmul(d, d));
                    }
                    sc.err[i] = e;
                }
                __syncwarp();
                double acc = sc.err[0];
                for (int i = 1; i < B; ++i) acc = dadd(acc, sc.err[i]);
                loss = __ddiv_rn(acc, (double)(B * OUT));
            }
            // 6-8. step counter, target copy, epsilon decay, mean_q
            ++st.replays;
            if (st.replays % ag.update_target_every == 0) {
                for (int e = lane; e < SNET; e += 32) Wt[e] = Wo[e];
            }
            if (st.epsilon > ag.epsilon_end) st.epsilon = dmul(st.epsilon, ag.epsilon_decay);
            double mq = sc.maxq[0];
            for (int i = 1; i < B; ++i) mq = dadd(mq, sc.maxq[i]);
            st.mean_q = __ddiv_rn(mq, (double)B);
            if (history && lane == 0 && row < history_rows) {
                double* hr = history + (a_idx * history_rows + row) * 4;
                hr[0] = loss;
                hr[1] = st.mean_q;
                hr[2] = st.epsilon;
                hr[3] = (double)st.replays;
            }
            ++row;
            __syncwarp();
        }
        // the call's record (:760-779): Q-values of its last point, average reward
        forward_warp(Wo, S0 + end * IN, sc, lane);
        if (lane == 0) {
            const int64_t k = a_idx * n_calls + c;
            avg_reward[k] = __ddiv_rn(rsum.value(), (double)(end - lo + 1));
            for (int o = 0; o < OUT; ++o) q_out[k * OUT + o] = sc.q[o];
        }
        __syncwarp();
    }

    for (int e = lane; e < B200BT_RL_PARAMS; e += 32) {
        g_online[e] = Wo[sidx(e)];
        g_target[e] = Wt[sidx(e)];
    }
    if (lane == 0) {
        st.act_words = rng_pos(act);
        st.sample_words = rng_pos(smp);
        *hdr = st;
    }
}

}  // namespace
}  // namespace b200bt

using namespace b200bt;

extern "C" int b200bt_rl_states(const float* cols, const float* close, const float* volume, int64_t ld, int S, int64_t N,
                                int bar_minutes, double* states, b200bt_stream_t stream) {
    B200BT_REQUIRE(cols && close && volume && states, B200BT_EINVAL, "rl_states: null pointer");
    B200BT_REQUIRE(S >= 1 && N >= 1 && ld >= N, B200BT_EINVAL, "rl_states: bad sizes");
    B200BT_REQUIRE(N < (1ll << T_BITS), B200BT_ELIMIT, "rl_states: N must be < 2^40 bars");
    B200BT_REQUIRE(bar_minutes > 0 && 60 % bar_minutes == 0, B200BT_EINVAL,
                   "rl_states: bar_minutes = %d does not divide 60 (the 1-hour price change)", bar_minutes);
    int rc = check_device();
    if (rc) return rc;
    const int64_t n = (int64_t)S * N;
    rl_states_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(cols, close, volume, ld, S, N,
                                                                                     60 / bar_minutes, 1440 / bar_minutes,
                                                                                     states);
    B200BT_LAUNCH_CHECK("rl_states launch");
    return B200BT_OK;
}

static int64_t rl_stride(int memory_max) {
    return (int64_t)sizeof(b200bt_rl_agent_state) + 2 * 8 * (int64_t)B200BT_RL_PARAMS + 8 * (int64_t)memory_max;
}

extern "C" int64_t b200bt_rl_workspace_bytes(int A, int memory_max) {
    if (A < 1 || memory_max < 1 || memory_max > B200BT_RL_MAX_MEMORY) return 0;
    return (int64_t)A * rl_stride(memory_max);
}

extern "C" int b200bt_rl_train(const double* states, int S, int64_t N, const b200bt_rl_agent* agents_host, int A,
                               int64_t agent_offset, int memory_max, void* agent_state, int64_t agent_state_bytes,
                               const int64_t* call_end_host, int n_calls, int points_per_call,
                               const double* init_weights_or_null, double* avg_reward, double* q_values,
                               double* history_or_null, int64_t history_rows, b200bt_stream_t stream) {
    B200BT_REQUIRE(states && agents_host && agent_state && call_end_host && avg_reward && q_values, B200BT_EINVAL,
                   "rl_train: null pointer");
    B200BT_REQUIRE(S >= 1 && N >= 1 && A >= 1 && n_calls >= 1 && agent_offset >= 0, B200BT_EINVAL, "rl_train: bad sizes");
    B200BT_REQUIRE(N < (1ll << T_BITS), B200BT_ELIMIT, "rl_train: N must be < 2^40 bars");
    B200BT_REQUIRE(points_per_call >= 1, B200BT_EINVAL, "rl_train: points_per_call = %d < 1", points_per_call);
    B200BT_REQUIRE(memory_max >= 1 && memory_max <= B200BT_RL_MAX_MEMORY, B200BT_EINVAL,
                   "rl_train: memory_max = %d outside [1, %d]", memory_max, B200BT_RL_MAX_MEMORY);
    B200BT_REQUIRE(agent_state_bytes >= b200bt_rl_workspace_bytes(A, memory_max), B200BT_EINVAL,
                   "rl_train: agent state of %lld bytes, %lld needed", (long long)agent_state_bytes,
                   (long long)b200bt_rl_workspace_bytes(A, memory_max));
    for (int a = 0; a < A; ++a) {
        const b200bt_rl_agent& g = agents_host[a];
        B200BT_REQUIRE(g.symbol >= 0 && g.symbol < S, B200BT_EINVAL, "rl_train: agent %d: symbol %d outside [0, %d)", a,
                       g.symbol, S);
        B200BT_REQUIRE(g.batch_size >= 1 && g.batch_size <= B200BT_RL_MAX_BATCH, B200BT_EINVAL,
                       "rl_train: agent %d: batch_size %d outside [1, %d]", a, g.batch_size, B200BT_RL_MAX_BATCH);
        B200BT_REQUIRE(g.memory_size >= g.batch_size && g.memory_size <= memory_max, B200BT_EINVAL,
                       "rl_train: agent %d: memory_size %d outside [batch_size = %d, memory_max = %d]", a, g.memory_size,
                       g.batch_size, memory_max);
        B200BT_REQUIRE(g.update_target_every >= 1, B200BT_EINVAL, "rl_train: agent %d: update_target_every < 1", a);
    }
    int64_t rows = 0;
    for (int c = 0; c < n_calls; ++c) {
        const int64_t e = call_end_host[c];
        B200BT_REQUIRE(e >= 0 && e < N, B200BT_EINVAL, "rl_train: call %d ends at bar %lld outside [0, N = %lld)", c,
                       (long long)e, (long long)N);
        rows += e + 1 < points_per_call ? e + 1 : points_per_call;
    }
    B200BT_REQUIRE(!history_or_null || history_rows >= rows, B200BT_EINVAL,
                   "rl_train: history of %lld rows per agent, the calls hold %lld points", (long long)history_rows,
                   (long long)rows);
    int rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t agent_bytes = sizeof(b200bt_rl_agent) * (size_t)A, end_bytes = sizeof(int64_t) * (size_t)n_calls;
    void* dev = nullptr;
    if ((rc = cuda_status(cudaMallocAsync(&dev, agent_bytes + end_bytes, st), "rl_train: cudaMallocAsync"))) return rc;
    b200bt_rl_agent* d_agents = (b200bt_rl_agent*)dev;
    int64_t* d_end = (int64_t*)((char*)dev + agent_bytes);
    rc = cuda_status(cudaMemcpyAsync(d_agents, agents_host, agent_bytes, cudaMemcpyHostToDevice, st), "rl_train: copy");
    if (!rc) rc = cuda_status(cudaMemcpyAsync(d_end, call_end_host, end_bytes, cudaMemcpyHostToDevice, st), "rl_train: copy");
    if (!rc) {
        const size_t smem = (2 * SNET) * sizeof(double) + sizeof(Scratch);
        rl_train_kernel<<<A, 32, smem, st>>>(states, N, d_agents, agent_offset, rl_stride(memory_max),
                                             (unsigned char*)agent_state, d_end, n_calls, points_per_call,
                                             init_weights_or_null, avg_reward, q_values, history_or_null, history_rows);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        rc = cuda_status(cudaGetLastError(), "rl_train launch");
    }
    const int rc_free = cuda_status(cudaFreeAsync(dev, st), "rl_train: cudaFreeAsync");
    return rc ? rc : rc_free;
}
