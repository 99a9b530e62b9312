// GA operators on the device (SURVEY 8-f2): tournament selection with elitism, uniform crossover, per-gene mutation
// -- the operators of services/genetic_algorithm.py:135-252 as three small kernels over a [pop][genes] float64
// matrix, driven by Philox4x32-10 keyed by (seed; generation, slot, stream).
//
// Parity with the reference is DISTRIBUTIONAL, not draw-for-draw: the reference consumes Python's global Mersenne
// twister in program order (ai_crypto_trader_b200/genetic_algorithm.py reproduces that stream exactly on the host);
// here every slot draws from its own counter, so a generation is one launch.  Same operators, same probabilities:
//   selection (:135-161)  elites = the max(1, int(elitism * pop)) best (stable by index), every other slot the winner
//                         of a tournament among `tournament` DISTINCT individuals (random.sample; first maximum wins)
//   breeding  (:225-252)  parents = two uniform draws from the selected list; with probability crossover_rate a
//                         uniform crossover (one coin per gene, :180-186); then per gene with probability
//                         mutation_rate (:191-223): integer genes +-max(1, int(0.1 (hi - lo))), float genes either
//                         x U(0.8, 1.2) or + U(-0.1 span, 0.1 span), clamped to the range.
//
// The stream is a function of the source alone, so tests/ga_ref.py restates it draw for draw:
//   words      counter = (slot or pair index, generation, stream id, block index), key = (seed low, seed high); a block's
//              words are handed out x[3], x[2], x[1], x[0], and one (slot, stream) is one continuous word stream, so a
//              uniform() after an odd number of words takes its two words from two blocks
//   uniform()  53 bits: the high 27 from the first word drawn, the low 26 from the second (sequenced statements, not
//              one expression whose operand order the compiler picks)
//   arithmetic the three products that are fused are written as fma() -- init lo + (hi - lo) u, the x U(0.8, 1.2)
//              factor and the + U(-0.1 span, 0.1 span) step -- so the results do not depend on --fmad; every other
//              float64 operation is rounded on its own
#include <math.h>
#include "common.cuh"
#include "philox.cuh"

namespace b200bt {

constexpr int GA_MAX_GENES = 64;
constexpr int GA_MAX_TOURNAMENT = 8;

struct GaRanges {
    double lo[GA_MAX_GENES], hi[GA_MAX_GENES];
    int is_int[GA_MAX_GENES];
};

// sel[j] = index of the individual copied into slot j of the "selected" list
__global__ void ga_select_kernel(const double* __restrict__ fitness, const int32_t* __restrict__ ranked, int pop, int n_elite,
                                 int tournament, uint64_t seed, uint32_t generation, int32_t* __restrict__ sel) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= pop) return;
    if (j < n_elite) { sel[j] = ranked[j]; return; }
    GaRng rng(seed, generation, (uint32_t)j, 0u);
    int pick[GA_MAX_TOURNAMENT];
    int best = -1;
    double best_fit = 0.0;
    for (int t = 0; t < tournament; ++t) {
        int cand;
        bool fresh;
        do {                                           // random.sample: distinct contenders
            cand = (int)rng.below((uint32_t)pop);
            fresh = true;
            for (int u = 0; u < t; ++u) fresh = fresh && pick[u] != cand;
        } while (!fresh);
        pick[t] = cand;
        const double f = fitness[cand];
        if (best < 0 || f > best_fit) { best = cand; best_fit = f; }      // first maximum wins (:158)
    }
    sel[j] = best;
}

// one thread per PAIR of offspring slots (n_elite + 2q, n_elite + 2q + 1); the first n_elite threads copy the elites
__global__ void ga_breed_kernel(const double* __restrict__ params, const int32_t* __restrict__ sel, int pop, int genes,
                                int n_elite, const GaRanges R, double crossover_rate, double mutation_rate, uint64_t seed,
                                uint32_t generation, double* __restrict__ out) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_pairs = (pop - n_elite + 1) / 2;
    if (q < n_elite) {
        const double* src = params + (int64_t)sel[q] * genes;
        for (int g = 0; g < genes; ++g) out[(int64_t)q * genes + g] = src[g];
    }
    if (q >= n_pairs) return;
    GaRng rng(seed, generation, (uint32_t)q, 1u);
    const double* p1 = params + (int64_t)sel[rng.below((uint32_t)pop)] * genes;      // random.choice(selected) twice (:233-234)
    const double* p2 = params + (int64_t)sel[rng.below((uint32_t)pop)] * genes;
    const bool cross = !(rng.uniform() > crossover_rate);                             // (:168)
    const int slot_a = n_elite + 2 * q, slot_b = slot_a + 1;
    for (int child = 0; child < 2; ++child) {
        const int slot = child == 0 ? slot_a : slot_b;
        if (slot >= pop) break;
        GaRng coin(seed, generation, (uint32_t)q, 2u);                                 // the SAME coins for both children:
        GaRng mut(seed, generation, (uint32_t)slot, 3u);                               // a gets what b does not (:180-186)
        for (int g = 0; g < genes; ++g) {
            const bool first = coin.uniform() < 0.5;
            double v = !cross ? (child == 0 ? p1[g] : p2[g]) : ((first == (child == 0)) ? p1[g] : p2[g]);
            const double lo = R.lo[g], hi = R.hi[g];
            if (mut.uniform() < mutation_rate) {
                if (R.is_int[g]) {
                    const double step = fmax(1.0, floor((hi - lo) * 0.1));
                    v += (mut.next() & 1u) ? step : -step;
                } else if (mut.uniform() < 0.5) {
                    v *= fma(mut.uniform(), 0.4, 0.8);
                } else {
                    const double span = hi - lo;
                    v = fma((2.0 * mut.uniform() - 1.0) * 0.1, span, v);
                }
                v = fmax(lo, fmin(hi, v));
            }
            out[(int64_t)slot * genes + g] = v;
        }
    }
}

// initial population (:83-117): integer genes uniform on {lo..hi}, float genes uniform on [lo, hi]; rows < n_seeded are
// the caller's seeded individuals, clamped
__global__ void ga_init_kernel(int pop, int genes, int n_seeded, const GaRanges R, uint64_t seed, double* __restrict__ params) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= pop) return;
    GaRng rng(seed, 0u, (uint32_t)j, 4u);
    for (int g = 0; g < genes; ++g) {
        const double lo = R.lo[g], hi = R.hi[g];
        double v;
        if (j < n_seeded) v = fmax(lo, fmin(hi, params[(int64_t)j * genes + g]));
        else if (R.is_int[g]) v = lo + (double)rng.below((uint32_t)(hi - lo) + 1u);
        else v = fma(hi - lo, rng.uniform(), lo);
        params[(int64_t)j * genes + g] = v;
    }
}

}  // namespace b200bt

using namespace b200bt;

static int fill_ranges(const double* lo, const double* hi, const int* is_int, int genes, GaRanges& R, const char* who) {
    B200BT_REQUIRE(lo && hi && is_int && genes > 0 && genes <= GA_MAX_GENES, B200BT_EINVAL, "%s: 1..%d genes", who, GA_MAX_GENES);
    for (int g = 0; g < genes; ++g) {
        B200BT_REQUIRE(hi[g] >= lo[g], B200BT_EINVAL, "%s: empty range for gene %d", who, g);
        B200BT_REQUIRE(!is_int[g] || hi[g] - lo[g] < 4.0e9, B200BT_ELIMIT, "%s: integer range of gene %d too wide", who, g);
        R.lo[g] = lo[g]; R.hi[g] = hi[g]; R.is_int[g] = is_int[g];
    }
    return B200BT_OK;
}

extern "C" int b200bt_ga_init(double* params, int pop, int genes, int n_seeded, const double* lo_host, const double* hi_host,
                              const int* is_int_host, uint64_t seed, b200bt_stream_t stream) {
    B200BT_REQUIRE(params && pop > 0 && n_seeded >= 0 && n_seeded <= pop, B200BT_EINVAL, "ga_init: bad argument");
    GaRanges R;
    int rc = fill_ranges(lo_host, hi_host, is_int_host, genes, R, "ga_init");
    if (rc) return rc;
    if ((rc = check_device())) return rc;
    ga_init_kernel<<<(pop + 127) / 128, 128, 0, (cudaStream_t)stream>>>(pop, genes, n_seeded, R, seed, params);
    B200BT_LAUNCH_CHECK("ga_init launch");
    return B200BT_OK;
}

extern "C" int b200bt_ga_next_generation(const double* params, const double* fitness, const int32_t* ranked, int pop, int genes,
                                         const double* lo_host, const double* hi_host, const int* is_int_host,
                                         double elitism_pct, int tournament, double crossover_rate, double mutation_rate,
                                         uint64_t seed, uint32_t generation, int32_t* selected_workspace, double* params_out,
                                         b200bt_stream_t stream) {
    B200BT_REQUIRE(params && fitness && ranked && selected_workspace && params_out && params != params_out, B200BT_EINVAL,
                   "ga_next_generation: null or aliased pointer");
    B200BT_REQUIRE(pop > 0 && tournament >= 1 && tournament <= GA_MAX_TOURNAMENT && tournament <= pop, B200BT_EINVAL,
                   "ga_next_generation: 1 <= tournament <= min(pop, %d)", GA_MAX_TOURNAMENT);
    B200BT_REQUIRE(isfinite(elitism_pct), B200BT_EINVAL, "ga_next_generation: elitism_pct is not finite");
    GaRanges R;
    int rc = fill_ranges(lo_host, hi_host, is_int_host, genes, R, "ga_next_generation");
    if (rc) return rc;
    if ((rc = check_device())) return rc;
    // min(pop, max(1, int(elitism_pct * pop))) (:142), clamped in double so that no out-of-range value is cast to int
    const double elite_count = elitism_pct * pop;
    const int n_elite = elite_count >= (double)pop ? pop : elite_count < 1.0 ? 1 : (int)elite_count;
    cudaStream_t st = (cudaStream_t)stream;
    ga_select_kernel<<<(pop + 127) / 128, 128, 0, st>>>(fitness, ranked, pop, n_elite, tournament, seed, generation, selected_workspace);
    B200BT_LAUNCH_CHECK("ga_select launch");
    const int n_pairs = (pop - n_elite + 1) / 2;
    const int threads = n_pairs > n_elite ? n_pairs : n_elite;
    ga_breed_kernel<<<(threads + 127) / 128, 128, 0, st>>>(params, selected_workspace, pop, genes, n_elite, R, crossover_rate,
                                                            mutation_rate, seed, generation, params_out);
    B200BT_LAUNCH_CHECK("ga_breed launch");
    return B200BT_OK;
}
