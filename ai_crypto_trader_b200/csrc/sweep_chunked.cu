// Family 2, time-parallel form: the population sweep with every expensive lane split into
// TIME CHUNKS that are scanned concurrently (sm_90a).
//
// The trade state machine (strategy_evaluation.py:746-878) is serial in time, and the lanes of a
// GA population differ by two to three orders of magnitude in trade count, so at moderate
// population sizes the fused kernel (sweep.cu) is bounded by the serial event chain of its few
// heaviest lanes.  The machine, however, forgets: whenever it is flat, its future does not depend
// on its past.  A chunk [T_c, T_{c+1}) is therefore scanned by its own warp, which starts `warm`
// bars early in the flat state without recording, and records from T_c on.  Two trajectories that
// are ever flat at the same bar coincide from then on, so after the warm-up the chunk's assumed
// state (position side + entry bar) is almost always the true one.  It is VERIFIED, not trusted:
//   scan kernels    chunk_scan_kernel: one WARP per (individual, symbol, chunk) of the expensive lanes
//                   (b200bt_sweep_chunked), or lane_scan_kernel: every lane cut into the same K chunks and one
//                   THREAD per (individual, symbol, chunk) (b200bt_sweep_tiled, see "thread-per-lane scan").
//                   Events -> blocks of a global pool (bump allocator, singly linked per chunk), plus the
//                   chunk's assumed state at T_c and its end state.
//   verify / repair lane_repair_kernel: one warp per lane walks the chunk boundaries in time order and re-scans a chunk
//                   whose assumed state differs from its predecessor's end state (chunk_scan_item<REPAIR>: from the true
//                   state, until the trajectory meets the recorded one; the rest of the recorded chain is spliced on).
//                   A bounded pass on the critical path, an unbounded one beside the metrics kernels (finish_chunks).
//   metrics kernels one warp per (individual, symbol, chunk) again (see "metrics, chunk-parallel" below), then
//                   one thread per (individual, symbol) checks end state of chunk c-1 == assumed state
//                   of chunk c for every boundary and merges the chunks' partial metrics.
// A lane with any mismatching boundary is flagged; the host re-evaluates flagged lanes with the
// fused (serial) kernel, so results never depend on the speculation being right.
#include <stddef.h>
#include "sweep_dev.cuh"

namespace b200bt {

constexpr int CK_BLOCK = 256;   // events per pool block
constexpr unsigned SEG_LOST = 0xffffffffu;   // seg_count of a chunk whose events were lost (full pool, tile given up, unpacked warp)

// Device-side counters of one sweep (a workspace section, zeroed at the start of the sweep); the first five are the flags
// the caller reads back, in the order of the C-ABI's overflow_host int[5].  The scan and repair kernels are given pointers
// to the fields they use: an address computed from the struct's base stays in registers the scan loops cannot spare.
struct SweepCounters {
    int overflow;            // [0] the event pool ran out
    int fallback_lanes;      // [1] (individual, symbol) lanes re-run by the exact fallback
    unsigned alloc;          // [2] pool blocks handed out (the pool's bump allocator)
    int stalls;              // [3] tiles of the thread-per-lane scan that did not arrive in time
    unsigned peak_chunks;    // [4] chunks that set a new equity peak (length of the peak list)
    int stall[8];            // the first stall: block, warp, item, tile, tiles, stage * 2 + parity, first tile, rows
    unsigned scan_work, chunk_repair_work, lane_repair_work;   // work counters of the persistent grids
    int n_fix_items;         // fix-up work items (individuals the overlapped repair touched)
    int n_redo;              // individuals listed for the exact fallback
};
constexpr int SWEEP_FLAGS = 5;
static_assert(offsetof(SweepCounters, peak_chunks) == (SWEEP_FLAGS - 1) * sizeof(int), "flags are the ABI's int[5]");

// The event pool and the per-chunk tables the scan kernels write and the repair / metrics kernels read.  Events live in
// blocks of CK_BLOCK (event word, price bits) pairs, bump-allocated; a chunk's blocks are linked from seg_first[seg]
// through next[].
struct ChunkTables {
    uint2* pool; int pool_blocks; int* next;
    unsigned* alloc; int* overflow;        // &SweepCounters::alloc, ::overflow
    int* seg_first; unsigned* seg_count;   // first block, number of events (SEG_LOST: dropped)
    int2* seg_in; int2* seg_out;           // assumed state at the chunk's start, state at its end: (side, entry bar or -1)
};

struct ChunkScanArgs : ChunkTables {
    const float* price; int64_t ld_price;
    const float* rsi; int64_t ld_rsi;
    int P, S; int64_t N;
    const b200bt_individual* indiv;
    const b200bt_chunk_item* items; int n_items; int n_seg;   // n_seg = segments per symbol
    int warm;
    const int32_t* n_chunks;
    unsigned char* redo;  // repair pass of the overlapped tail: individuals whose metrics must be recomputed
};

__device__ __forceinline__ unsigned seg_records(unsigned count) { return count == SEG_LOST ? 0u : count; }

// links a new pool block behind chunk `seg`'s last one, `block` (-1: none yet), and moves `block` to it; false when the
// pool is full (flagged)
__device__ __forceinline__ bool pool_take_block(const ChunkTables& T, const int seg, int& block) {
    const int b = (int)atomicAdd(T.alloc, 1u);
    if (b >= T.pool_blocks) { atomicExch(T.overflow, 1); return false; }
    T.next[b] = -1;
    if (block < 0) T.seg_first[seg] = b; else T.next[block] = b;
    block = b;
    return true;
}

// the chunk is not scanned: it is marked as having lost its events, which sends it to a repair pass or its lane to the
// exact fallback
__device__ __forceinline__ void mark_lost(const ChunkTables& T, const int seg) {
    T.seg_in[seg] = make_int2(0, -1);
    T.seg_out[seg] = make_int2(0, -1);
    T.seg_count[seg] = SEG_LOST;
}

__device__ __forceinline__ int64_t chunk_begin(int64_t N, int c, int K) {
    if (c >= K) return N;
    return ((N * c) / K) & ~(int64_t)(SW_GROUP - 1);   // group aligned
}

// REPAIR = false: speculative pass over every (work item, symbol), warm-up from the flat state.
// REPAIR = true : re-scan of chunks whose assumed state was wrong, started AT T_c from the now known
//                 true state (end state of the preceding chunk); one work item per listed chunk.
template <bool VEC16, bool REPAIR>
__device__ __forceinline__ bool chunk_scan_item(const ChunkScanArgs& A, const b200bt_chunk_item item, const int sym, WarpShared* ws) {
    const int lane = threadIdx.x & 31;
    const b200bt_individual iv = A.indiv[item.individual];
    if (lane == 0) {
        ScanConst sc0;
        init_scan_const(sc0, iv);
        ws->sc = sc0;
        ws->acc.tp = iv.take_profit;   // only the screening-band decision reads these here
        ws->acc.sl = iv.stop_loss;
    }
    __syncwarp();
    const ScanConst c = ws->sc;
    const float* __restrict__ pr = A.price + (int64_t)sym * A.ld_price;
    const float* __restrict__ rr = A.rsi + ((int64_t)sym * A.P + iv.rsi_row) * A.ld_rsi;

    const int n = (int)A.N;
    const int T0 = (int)chunk_begin(A.N, item.chunk, item.n_chunks);       // first recorded bar
    const int T1 = (int)chunk_begin(A.N, item.chunk + 1, item.n_chunks);   // end (exclusive)
    int s0 = REPAIR ? T0 : T0 - A.warm;
    if (s0 < 0 || item.chunk == 0) s0 = 0;
    s0 &= ~(SW_GROUP - 1);
    const int seg = sym * A.n_seg + item.segment;

    Machine m = flat_machine(iv);
    unsigned qtail = 0;
    if (REPAIR) {
        // true state at T0 = end state of the preceding chunk (position side, entry bar -> entry price)
        const int2 z = A.seg_out[seg - 1];
        if (z.x != 0) set_open(m, c, z.x > 0, __ldg(pr + z.y), z.y);
    }

    // REPAIR: the chain the speculative scan recorded for this chunk and the state it assumed at T0.  Two trajectories that
    // are in the same state at the same bar coincide from there on, so the re-scan stops at the first group boundary at
    // which its state equals the recorded trajectory's and splices the rest of the recorded events (below).
    int old_block = -1, old_idx = 0, old_pos = 0, old_ebar = -1;
    unsigned old_left = 0;
    bool old_ok = false, spliced = false;
    if (REPAIR) {
        const unsigned oc = A.seg_count[seg];
        const int2 oin = A.seg_in[seg];
        old_ok = oc != SEG_LOST;     // (a chunk whose events were dropped has no chain to splice)
        old_left = seg_records(oc);
        old_block = A.seg_first[seg];
        old_pos = oin.x; old_ebar = oin.x != 0 ? oin.y : -1;
    }

    // event sink: 32 queued events -> one coalesced 256-byte store into the chunk's current pool block
    int cur_block = -1, fill = CK_BLOCK, dead = 0;
    auto flush = [&](unsigned at, int cnt) {
        if (fill == CK_BLOCK && !dead) {
            int b = cur_block;
            if (lane == 0 && !pool_take_block(A, seg, b)) b = -1;
            b = __shfl_sync(FULL, b, 0);
            if (b < 0) dead = 1; else { cur_block = b; fill = 0; }
        }
        if (!dead) {
            if (lane < cnt) A.pool[(int64_t)cur_block * CK_BLOCK + fill + lane] = ws->evq[(at + lane) & (SW_EVQ - 1)];
            fill += 32;   // only the last flush of a chunk is partial
        }
    };

    constexpr int G = SW_GROUP;
    const int g_begin = s0 / G, g_end = (T1 + G - 1) / G;
    GroupRing<VEC16> ring(ws, pr, rr, n, g_begin, g_end);
    for (int g = g_begin; g < g_end; ++g) {
        const float* w = ring.land();
        const bool emit = g * G >= T0;
        if (g * G == T0 && lane == 0) A.seg_in[seg] = make_int2(m.pos, m.pos != 0 ? m.entry_bar : -1);
        if (REPAIR && old_ok && g > g_begin) {
            // state of the recorded trajectory before bar tb = g * G: consume its events with bar < tb
            const unsigned tb = (unsigned)(g * G);
            while (old_left) {
                const int n_here = (int)min(min(32u, old_left), (unsigned)(CK_BLOCK - old_idx));
                const unsigned word = lane < n_here ? A.pool[(int64_t)old_block * CK_BLOCK + old_idx + lane].x : 0xffffffffu;
                const int k = __popc(__ballot_sync(FULL, lane < n_here && (word & B200BT_EVENT_BAR_MASK) < tb));    // (bars ascend: a prefix)
                if (k) {
                    const unsigned last = __shfl_sync(FULL, word, k - 1);
                    old_pos = (last & B200BT_EVENT_EXIT) ? 0 : ((last & B200BT_EVENT_SELL) ? -1 : 1);
                    old_ebar = (last & B200BT_EVENT_EXIT) ? -1 : (int)(last & B200BT_EVENT_BAR_MASK);
                    old_idx += k; old_left -= (unsigned)k;
                    if (old_idx == CK_BLOCK && old_left) { old_block = A.next[old_block]; old_idx = 0; }
                }
                if (k < n_here) break;
            }
            if (m.pos == old_pos && (m.pos == 0 || m.entry_bar == old_ebar)) {
                // same state at the same bar: the rest of the recorded chain is this trajectory's; copy it behind the
                // re-scanned events (the chunk's end state, and with it every later chunk, stands as recorded)
                while (old_left) {
                    const int n_here = (int)min(min(32u, old_left), (unsigned)(CK_BLOCK - old_idx));
                    if (lane < n_here) ws->evq[(m.qhead + lane) & (SW_EVQ - 1)] = A.pool[(int64_t)old_block * CK_BLOCK + old_idx + lane];
                    m.qhead += (unsigned)n_here;
                    old_idx += n_here; old_left -= (unsigned)n_here;
                    if (old_idx == CK_BLOCK && old_left) { old_block = A.next[old_block]; old_idx = 0; }
                    __syncwarp();
                    // (inline rather than drain_full: the splice synchronises once per copied block, and drain_full's
                    // __syncwarp per batch makes the repair kernels' code larger)
                    while (m.qhead - qtail >= 32) { flush(qtail, 32); qtail += 32; }
                    __syncwarp();
                }
                spliced = true;
                break;
            }
        }
        scan_group(w, g * G, ws, c, m, qtail, emit, flush);
        ring.release();
    }
    if (lane == 0 && !spliced) {
        const int2 st = make_int2(m.pos, m.pos != 0 ? m.entry_bar : -1);
        A.seg_out[seg] = st;
        if (T0 >= T1) A.seg_in[seg] = st;   // empty chunk: its assumed state is the state after the warm-up
    }
    finish_scan(ws, m, qtail, pr, A.N, !spliced && item.chunk == item.n_chunks - 1, flush);
    if (lane == 0) A.seg_count[seg] = dead ? SEG_LOST : m.qhead;
    __syncwarp();
    return spliced;      // REPAIR: the chunk's recorded end state stands
}

template <bool VEC16>
__global__ void __launch_bounds__(SW_WARPS * 32, 3)
chunk_scan_kernel(const ChunkScanArgs A) {   // by value, not __grid_constant__ (see sweep.cu)
    extern __shared__ __align__(16) unsigned char s_raw[];
    WarpShared* ws = reinterpret_cast<WarpShared*>(s_raw) + (threadIdx.x >> 5);
    const int sym = (int)(blockIdx.x % (unsigned)A.S);
    const int it = (int)(blockIdx.x / (unsigned)A.S) * SW_WARPS + (threadIdx.x >> 5);
    if (it >= A.n_items) return;
    chunk_scan_item<VEC16, false>(A, A.items[it], sym, ws);
}

// Verification and repair.  Two kernels share chunk_scan_item<REPAIR> (re-scan from the true state until the trajectory
// meets the recorded one, then splice the recorded chain on); neither needs a work list or anything read by the host.
//
// chunk_repair_kernel (critical path): one warp per (chunk, symbol), handed out by a counter.  The warp compares its chunk's
// assumed start state with the predecessor's recorded end state and re-scans on a mismatch.  All wrong chunks of a lane are
// repaired CONCURRENTLY, each trusting its predecessor's recorded end state -- which stands whenever the predecessor's own
// re-scan finds its way back to the recorded trajectory, i.e. almost always.  (A predecessor that is being rewritten at
// the same moment is a benign race on an aligned 8-byte word: whichever value is read becomes the chunk's published start
// state, and the boundary is checked again below and in lane_combine_kernel.)
template <bool VEC16>
__global__ void __launch_bounds__(SW_WARPS * 32, 3)
chunk_repair_kernel(const ChunkScanArgs A, unsigned* __restrict__ work) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    WarpShared* ws = reinterpret_cast<WarpShared*>(s_raw) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int64_t total = (int64_t)A.n_items * A.S;
    for (;;) {
        unsigned t = 0;
        if (lane == 0) t = atomicAdd(work, 1u);
        t = __shfl_sync(FULL, t, 0);
        if ((int64_t)t >= total) break;
        const int it = (int)(t / (unsigned)A.S), sym = (int)(t - (unsigned)it * (unsigned)A.S);
        const b200bt_chunk_item item = A.items[it];
        if (item.chunk == 0) continue;
        const int seg = sym * A.n_seg + item.segment;
        const int2 a = A.seg_in[seg], z = A.seg_out[seg - 1];
        if ((a.x != z.x || a.y != z.y) && A.seg_count[seg - 1] != SEG_LOST) chunk_scan_item<VEC16, true>(A, item, sym, ws);
    }
}

// lane_repair_kernel (beside the metrics kernels): one warp per (individual, symbol) lane walks the lane's boundaries in
// time order and re-scans where a chunk does not follow from its predecessor, checking the next boundary against the end
// state it has just produced -- so the lane is consistent when the warp leaves it, however many chunks in a row a re-scan
// runs through without meeting its recorded trajectory (lanes that hold one position across many chunks).  After
// chunk_repair_kernel only those cascades are left.  Individuals it touches are flagged in A.redo (metrics recomputed).
template <bool VEC16>
__global__ void __launch_bounds__(SW_WARPS * 32, 3)
lane_repair_kernel(const ChunkScanArgs A, const int pop, const int32_t* __restrict__ seg_base, unsigned* __restrict__ work) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    WarpShared* ws = reinterpret_cast<WarpShared*>(s_raw) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int lanes = pop * A.S;
    for (;;) {
        int t = 0;
        if (lane == 0) t = (int)atomicAdd(work, 1u);
        t = __shfl_sync(FULL, t, 0);
        if (t >= lanes) break;
        const int ind = t / A.S, sym = t - ind * A.S;
        const int K = A.n_chunks[ind];
        const int sb = seg_base[ind];
        const int base = sym * A.n_seg + sb;
        int2 prev = A.seg_out[base];
        bool usable = A.seg_count[base] != SEG_LOST;      // (a chunk that lost events to a full pool ends the walk: the lane is flagged later)
        for (int c = 1; c < K && usable; ++c) {
            const int2 a = A.seg_in[base + c];
            if (a.x != prev.x || a.y != prev.y) {
                b200bt_chunk_item item;
                item.individual = ind; item.chunk = c; item.segment = sb + c; item.n_chunks = K;
                if (A.redo && lane == 0) A.redo[ind] = 1;
                chunk_scan_item<VEC16, true>(A, item, sym, ws);      // (ends with a __syncwarp: its stores are visible to the warp)
            }
            prev = A.seg_out[base + c];
            usable = A.seg_count[base + c] != SEG_LOST;
        }
    }
}

// ---- thread-per-lane scan ---------------------------------------------------------------------------
// The warp-per-lane scan above spends a full warp on the scalar event chain of one lane.  With every lane cut
// into the SAME K time chunks there are pop x S x K independent machines -- enough to give each one a THREAD:
// a CTA owns (symbol, chunk, 256 individuals), streams tiles of the price row and the whole RSI bank of that
// symbol through shared memory (cp.async, two stages) and every thread steps its own machine through the tile,
// four bars per step.  The event path then runs in SIMT fashion for up to 32 lanes at once, all threads walk
// the same bars (no tail), and the bank is fetched once per 256 lanes.  Events go to the same pool / segment
// tables as the warp scan, so verification, repair and the metrics kernels are shared.
#ifndef B200BT_LS_T
#define B200BT_LS_T 128
#endif
constexpr int LS_T = B200BT_LS_T;       // bars per tile
constexpr int LS_STRIDE = LS_T + 4;     // row stride in floats (16-byte aligned rows, rows 8 apart share banks)
#ifndef B200BT_LS_THREADS
#define B200BT_LS_THREADS 256
#endif
constexpr int LS_THREADS = B200BT_LS_THREADS;

constexpr int LS_ZONE = 32;             // bars per zone-map block

// Zone map: (min, max) of every 32-bar block ("coarse") and of every 4-bar group ("fine") of the price row and of each
// RSI row, NaNs ignored.  A machine whose thresholds lie outside a range cannot fire inside it: the scan skips a 32-bar
// block after four compares when no machine of the warp can fire in it, and inside a block it tests each 4-bar group
// against the group's precomputed range (two 8-byte loads, four compares) instead of folding the eight values itself.
// Layout: coarse [S][P + 1][zone_row_stride(N)] float2, then fine [S][P + 1][zone_fine_stride(N)] float2; row 0 = price;
// both strides keep rows 16-byte aligned and pad with (NaN, NaN) (every compare false).
__global__ void __launch_bounds__(256)
zone_map_kernel(const float* __restrict__ price, int64_t ld_price, const float* __restrict__ rsi, int64_t ld_rsi, int P,
                int64_t N, int64_t row_stride, int64_t fine_stride, float2* __restrict__ zones, float2* __restrict__ fine) {
    const int row = blockIdx.y % (P + 1), sym = blockIdx.y / (P + 1);
    const float* __restrict__ src = row == 0 ? price + (int64_t)sym * ld_price : rsi + ((int64_t)sym * P + row - 1) * ld_rsi;
    float2* __restrict__ dst = zones + ((int64_t)sym * (P + 1) + row) * row_stride;
    float2* __restrict__ fdst = fine + ((int64_t)sym * (P + 1) + row) * fine_stride;
    const int lane = threadIdx.x & 31;
    // (fine_stride covers whole 128-bar tiles and is >= 8 * row_stride - 8: one pass writes both)
    for (int64_t blk = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); blk * (LS_ZONE / 4) < fine_stride || blk < row_stride;
         blk += (int64_t)gridDim.x * 8) {
        const int64_t t = blk * LS_ZONE + lane;
        const float v = t < N ? __ldg(src + t) : __int_as_float(0x7fc00000);
        float lo = v, hi = v;
#pragma unroll
        for (int m = 1; m < 4; m <<= 1) {
            lo = fminf(lo, __shfl_xor_sync(FULL, lo, m));
            hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, m));
        }
        if ((lane & 3) == 0 && blk * (LS_ZONE / 4) + (lane >> 2) < fine_stride) fdst[blk * (LS_ZONE / 4) + (lane >> 2)] = make_float2(lo, hi);
#pragma unroll
        for (int m = 4; m < 32; m <<= 1) {
            lo = fminf(lo, __shfl_xor_sync(FULL, lo, m));
            hi = fmaxf(hi, __shfl_xor_sync(FULL, hi, m));
        }
        if (lane == 0 && blk < row_stride) dst[blk] = make_float2(lo, hi);
    }
}

struct LaneScanArgs : ChunkTables {
    const float* price; int64_t ld_price;
    const float* rsi; int64_t ld_rsi;
    const float2* zones; int64_t n_zone_blocks;   // zone map (coarse part; n_zone_blocks = its row stride) or NULL
    const float2* fine; int64_t n_fine;           // 4-bar ranges and their row stride
    int P, S; int64_t N;
    const b200bt_individual* indiv; const int32_t* slots; int n_slots; int pop; int K; int warm;
    unsigned* work;          // &SweepCounters::scan_work
    SweepCounters* ctr;      // (stalls, stall)
    long long wait_cycles;   // bound of a tile wait in SM clocks (LS_WAIT_CYCLES; b200bt_sweep_scan_wait_cycles overrides, for tests)
};

__device__ __forceinline__ int sym_of_block(unsigned bx, int S) { return (int)(bx % (unsigned)S); }

// device-side tables the shared kernels expect: uniform K chunks per individual.  Work items are listed in dispatch
// order (`order`: individuals by predicted cost, a lane's chunks adjacent), so that the 32 chunks a warp of the
// thread-per-chunk metrics kernels folds hold similar numbers of records; segments stay indexed by individual.
__global__ void lane_tables_kernel(int pop, int K, const int32_t* __restrict__ order, b200bt_chunk_item* __restrict__ items,
                                   int32_t* __restrict__ seg_base, int32_t* __restrict__ n_chunks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pop * K) return;
    const int k = i / K, c = i - k * K;
    const int ind = order ? order[k] : k;
    b200bt_chunk_item it;
    it.individual = ind; it.chunk = c; it.n_chunks = K; it.segment = ind * K + c;
    items[i] = it;
    if (c == 0) { seg_base[ind] = ind * K; n_chunks[ind] = K; }
}

#ifndef B200BT_LS_MIN_BLOCKS
#define B200BT_LS_MIN_BLOCKS 3      // 80 registers, 0 / 16 B spilled without / with zones (nvcc 12.9); at 4 CTAs/SM (64) 3 % slower
#endif
#ifndef B200BT_LS_STAGES
#define B200BT_LS_STAGES 2
#endif
// 4-bar groups per iteration of the scan loop, chosen per launch from the event density the pool was sized for.  The scan
// is issue-bound and its group body holds four inlined copies of the event step: unrolled twice the kernel has 2704 SASS
// instructions with zones, not unrolled 2144.  On the H100 the smaller loop scans the random configs[1] population ~7 %
// faster, while a population with ~7x the events (generation 3 of a GA run) is ~1 % faster unrolled.  (A rolled loop over
// the four bars -- one step copy, bars read back from the stage -- is ~45 % slower: the group's float4 registers and the
// straight-line selects are what make the step cheap.)
constexpr int LS_UNROLL_SPARSE = 1, LS_UNROLL_DENSE = 2;
constexpr double LS_DENSE_EVENTS = 0.05;      // pool events per machine and bar from which the dense form is launched
constexpr int LS_STAGES = B200BT_LS_STAGES;   // tiles in flight per warp (ring depth)
constexpr int LS_WARPS = LS_THREADS / 32;
constexpr int LS_RSI_ROWS = 2;                // distinct RSI rows the 32 machines of a warp may read (host packing)
constexpr int LS_ROWS = 1 + LS_RSI_ROWS;      // staged rows per warp: price + its RSI rows

static_assert(LS_ZONE == ZONE_BLOCK && LS_T == ZONE_TILE, "zone map layout (common.cuh) follows the scan's tile");

// Tile movement.  The 32 machines of a warp read the price row and (the host packs them so) at most LS_RSI_ROWS RSI rows.
// Every WARP owns a private ring of LS_STAGES shared-memory stages, each holding one 128-bar tile of those rows plus the
// tile's zone ranges; a stage is filled by bulk async copies (cp.async.bulk, one per row, issued by LS_ROWS lanes,
// completion counted on the stage's mbarrier) LS_STAGES - 1 tiles ahead of the scan and refilled by the warp itself the
// moment it has scanned it.  No warp ever waits for another one -- ncu on the round-1 form (one tile of all P + 1 rows per
// CTA, two CTA barriers per tile) showed a third of the warp time parked at those barriers behind the CTA's busiest warp
// and 18 % of the instructions computing cp.async addresses -- and the bytes moved per machine stay what they were,
// because a CTA-wide tile staged P + 1 rows for 256 machines and a warp stages 3 for 32.
// One work item: the 32 machines of warp-slot `wslot` (thread slots wslot * 32 ...) on symbol `sym`, chunk `c`.
constexpr long long LS_WAIT_CYCLES = 40ll * 1000 * 1000;     // ~20 ms at 1.9 GHz; a tile normally lands within microseconds

// the 32 machines of (warp-slot, symbol, chunk) are not scanned: their chunks are marked lost
__device__ __forceinline__ void lane_scan_give_up(const LaneScanArgs& A, const int wslot, const int sym, const int c) {
    const int k = wslot * 32 + (int)(threadIdx.x & 31);
    const int slot = k < A.n_slots ? (A.slots ? A.slots[k] : (k < A.pop ? k : -1)) : -1;
    if (slot >= 0) mark_lost(A, sym * (A.pop * A.K) + slot * A.K + c);
}

// -> false: a tile of this item did not arrive (see the wait below); the warp must not take another item
template <bool ZONES, int UNROLL>
__device__ __forceinline__ bool lane_scan_item(const LaneScanArgs& A, const bool vec16, const int wslot, const int sym, const int c,
                                               float* const wtile, float2* const wzone, unsigned long long* const full,
                                               float (*ls_mul)[LS_THREADS], double (*ls_tpsl)[LS_THREADS], const void* (*ls_src_w)[3],
                                               int& ring_stage, unsigned& ring_parity) {
    constexpr int ZB = LS_T / LS_ZONE;                  // zone blocks per tile
    constexpr int FG = LS_T / 4;                        // 4-bar groups per tile
    constexpr int ZR = ZB + FG;                         // float2 per staged row: coarse ranges, then fine ranges
    const int lane = threadIdx.x & 31;
    const int k = wslot * 32 + lane;
    const int slot = k < A.n_slots ? (A.slots ? A.slots[k] : (k < A.pop ? k : -1)) : -1;
    const bool active = slot >= 0;
    const int ind = active ? slot : 0;
    const b200bt_individual iv = A.indiv[ind];
    // the screening multipliers are needed on events only: shared memory, [multiplier][thread] (conflict-free),
    // side-major so that the side selects an address instead of a value: long hi_c lo_c hi_d lo_d, short ...
    const float os_f = iv.rsi_lo, ob_f = iv.rsi_hi;
    {
        ScanConst sc;
        init_scan_const(sc, iv);
        float* m = &ls_mul[0][threadIdx.x];
        m[0 * LS_THREADS] = sc.hiL_c; m[1 * LS_THREADS] = sc.loL_c; m[2 * LS_THREADS] = sc.hiL_d; m[3 * LS_THREADS] = sc.loL_d;
        m[4 * LS_THREADS] = sc.hiS_c; m[5 * LS_THREADS] = sc.loS_c; m[6 * LS_THREADS] = sc.hiS_d; m[7 * LS_THREADS] = sc.loS_d;
        // take-profit / stop-loss of the float64 exit decision inside the screening band, beside them: read back from
        // here, the step no longer re-reads A.indiv[ind] (whose address the scan loop otherwise keeps in registers)
        ls_tpsl[0][threadIdx.x] = iv.take_profit;
        ls_tpsl[1][threadIdx.x] = iv.stop_loss;
    }
    __syncwarp();
    // The ring's barriers are initialised ONCE per warp (lane_scan_kernel) and their phases roll on from item to item: every
    // copy of the previous item has landed and been waited for, so the ring continues at (ring_stage, ring_parity).  (The
    // first persistent form invalidated and re-initialised the barriers at every item; about once in 10^4 launches a tile
    // then never completed -- a re-initialisation racing with the copy engine's last update of the barrier it had just
    // completed is the suspected cause -- which is also why the wait below is bounded.)

    const int n = (int)A.N;
    const int T0 = (int)chunk_begin(A.N, c, A.K);       // first recorded bar (multiple of SW_GROUP, hence of LS_T)
    const int T1 = (int)chunk_begin(A.N, c + 1, A.K);   // end (exclusive)
    int s0 = (c == 0) ? 0 : T0 - A.warm;
    if (s0 < 0) s0 = 0;
    s0 &= ~(LS_T - 1);
    const int tl_begin = s0 / LS_T, n_tiles = (T1 + LS_T - 1) / LS_T - tl_begin;
    const int seg = sym * (A.pop * A.K) + ind * A.K + c;

    // the warp's distinct RSI rows: staged row 1 + j holds the j-th of them (in lane order of first use)
    const unsigned amask = __ballot_sync(FULL, active);
    if (amask == 0u) return true;                       // an empty warp (padding of the last CTA)
    const unsigned peers = __match_any_sync(FULL, active ? iv.rsi_row : -1 - lane);
    const int leader = __ffs(peers) - 1;
    const unsigned heads = __ballot_sync(FULL, active && lane == leader);
    const int n_rsi = __popc(heads);
    const int my_row = 1 + __popc(heads & ((1u << leader) - 1u));       // staged row this machine reads
    if (n_rsi > LS_RSI_ROWS) {
        // not packed for this schedule: the lanes are flagged and re-run by the caller's exact fallback (fused kernel)
        if (active) mark_lost(A, seg);
        return true;
    }
    // lane L <= n_rsi issues the copies of staged row L (0 = price)
    const unsigned src_lane = __fns(heads, 0, lane);                    // lane of the (lane)-th head (1-based), or ~0u
    const int row_of_lane = __shfl_sync(FULL, iv.rsi_row, src_lane < 32u ? (int)src_lane : 0);
    const bool issuer = lane <= n_rsi;
    const int zrow = (lane == 0 || !issuer) ? 0 : 1 + row_of_lane;      // row of the zone map (0 = price)
    // source rows of the warp's staged rows: a small table in shared memory (read by the issuing lanes only: three
    // 64-bit pointers per thread would not fit the register budget of the scan loop)
    if (issuer) {
        ls_src_w[lane][0] = (lane == 0) ? A.price + (int64_t)sym * A.ld_price : A.rsi + ((int64_t)sym * A.P + row_of_lane) * A.ld_rsi;
        ls_src_w[lane][1] = ZONES ? A.zones + ((int64_t)sym * (A.P + 1) + zrow) * A.n_zone_blocks : nullptr;   // (n_zone_blocks = row stride)
        ls_src_w[lane][2] = ZONES ? A.fine + ((int64_t)sym * (A.P + 1) + zrow) * A.n_fine : nullptr;
    }
    __syncwarp();
    const unsigned stage_bytes = (unsigned)(1 + n_rsi) * (LS_T * 4 + (ZONES ? ZR * 8 : 0));

    // fill stage `stage` of this warp's ring with tile `tl`
    auto issue = [&](int tl, int stage) {
        float* dst0 = wtile + (size_t)stage * LS_ROWS * LS_STRIDE;
        float2* zdst = wzone + (size_t)stage * LS_ROWS * ZR;
        const int t0 = tl * LS_T;
        if (vec16 && t0 + LS_T <= n) {
            if (lane == 0) mbar_arrive_expect_tx(&full[stage], stage_bytes);
            __syncwarp();
            if (issuer) {
                fence_proxy_async();      // the warp's reads of the stage (generic proxy) are ordered before the async writes
                bulk_g2s(dst0 + lane * LS_STRIDE, static_cast<const float*>(ls_src_w[lane][0]) + t0, LS_T * 4, &full[stage]);
                if (ZONES) {
                    bulk_g2s(zdst + lane * ZR, static_cast<const float2*>(ls_src_w[lane][1]) + (int64_t)tl * ZB, ZB * 8, &full[stage]);
                    bulk_g2s(zdst + lane * ZR + ZB, static_cast<const float2*>(ls_src_w[lane][2]) + (int64_t)tl * FG, FG * 8, &full[stage]);
                }
            }
        } else {
            const float qnan = __int_as_float(0x7fc00000);   // unaligned input or the ragged last tile: plain copies
            for (int r = 0; r <= n_rsi; ++r) {
                const float* src = static_cast<const float*>(ls_src_w[r][0]);
                for (int col = lane; col < LS_T; col += 32) dst0[r * LS_STRIDE + col] = (t0 + col < n) ? __ldg(src + t0 + col) : qnan;
                if (ZONES) {
                    const float2* zs = static_cast<const float2*>(ls_src_w[r][1]);
                    const float2* fs = static_cast<const float2*>(ls_src_w[r][2]);
                    if (lane < ZB) {
                        const int64_t zblk = (int64_t)tl * ZB + lane;
                        zdst[r * ZR + lane] = (zblk * LS_ZONE < n) ? zs[zblk] : make_float2(qnan, qnan);
                    }
                    zdst[r * ZR + ZB + lane] = fs[(int64_t)tl * FG + lane];        // (FG == 32; rows are padded to whole tiles)
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&full[stage]);     // (release: the stores above are visible after the wait)
        }
    };
    for (int it = 0; it < LS_STAGES && it < n_tiles; ++it) issue(tl_begin + it, (ring_stage + it) % LS_STAGES);

    // machine state (per thread)
    int pos = 0, entry_bar = 0;
    float e_px = 0.f, rlo = iv.rsi_lo, rhi = iv.rsi_hi, plo = -INFINITY, phi = INFINITY;
    // event sink: this thread's chunk owns a chain of pool blocks
    int cur_block = -1, fill = CK_BLOCK;
    unsigned count = 0;
    bool rec = false, dead = false;
    uint2* wptr = A.pool;
    auto record = [&](unsigned word, float p) {
        if (fill == CK_BLOCK && !dead) {
            if (!pool_take_block(A, seg, cur_block)) dead = true;
            else { fill = 0; wptr = A.pool + (int64_t)cur_block * CK_BLOCK; }
        }
        if (!dead) { *wptr++ = make_uint2(word, __float_as_uint(p)); ++fill; }
        ++count;
    };

    // one bar of the state machine; same decisions as scan_window (sweep_dev.cuh).  Written as straight-line
    // selects: the threads of a warp that fire on the same bar (entries and exits alike) share one pass.
    auto step = [&](float p, float r, int t) {
        const bool rsi_hit = (r < rlo) | (r > rhi);
        if (!(rsi_hit | (p <= plo) | (p >= phi))) return;
        const bool flat = pos == 0, lng_open = pos > 0;
        bool ev = true;
        if (!flat && !rsi_hit) {
            // price trigger: definite outside the fp32 screening band, else the reference's float64 expression
            const float* m = &ls_mul[lng_open ? 2 : 6][threadIdx.x];
            const float hd = e_px * m[0], ld = e_px * m[LS_THREADS];
            if (!((p >= hd) || (p <= ld))) {
                const double ed = (double)e_px, pd = (double)p;
                const double q = lng_open ? __ddiv_rn(__dsub_rn(pd, ed), ed) : __ddiv_rn(__dsub_rn(ed, pd), ed);
                ev = (q >= ls_tpsl[0][threadIdx.x]) || (q <= -ls_tpsl[1][threadIdx.x]);
            }
        }
        if (!ev) return;
        const bool lng = r < os_f;                        // entry side: long has priority (:784, :799)
        const unsigned word = flat ? ((unsigned)t | (lng ? 0u : B200BT_EVENT_SELL))
                                   : ((unsigned)t | B200BT_EVENT_EXIT | (lng_open ? B200BT_EVENT_SELL : 0u));
        pos = flat ? (lng ? 1 : -1) : 0;
        rlo = (flat && lng) ? -INFINITY : os_f;
        rhi = (flat && !lng) ? INFINITY : ob_f;
        const float* mc = &ls_mul[lng ? 0 : 4][threadIdx.x];
        phi = flat ? p * mc[0] : INFINITY;
        plo = flat ? p * mc[LS_THREADS] : -INFINITY;
        e_px = flat ? p : e_px;
        entry_bar = flat ? t : entry_bar;
        if (rec) record(word, p);
    };

    int stage = ring_stage;
    unsigned parity = ring_parity;
    for (int it = 0; it < n_tiles; ++it) {
        // A copy that never completes must not hang the GPU: the wait is bounded.  On a timeout the item is given up -- its
        // chunks are marked as having lost their events, so the repair pass re-scans them (or the lane takes the exact
        // fallback) -- and the warp never touches its ring again (copies may still be in flight into it): it goes on taking
        // items only to give them up as well (lane_scan_kernel), while the other warps scan theirs.
        // (wait_cycles < 0 is the test hook: the warp gives up at its (-wait_cycles)-th tile as if the tile had not arrived)
        const bool lost = A.wait_cycles < 0 ? (it + 1 == (int)-A.wait_cycles || !mbar_wait_bounded(&full[stage], parity, LS_WAIT_CYCLES))
                                            : !mbar_wait_bounded(&full[stage], parity, A.wait_cycles);
        if (__any_sync(FULL, lost)) {
            lane_scan_give_up(A, wslot, sym, c);
            if (lane == 0 && atomicAdd(&A.ctr->stalls, 1) == 0) {
                int* const d = A.ctr->stall;
                d[0] = (int)blockIdx.x; d[1] = (int)(threadIdx.x >> 5); d[2] = wslot * 65536 + sym * 256 + c;
                d[3] = it; d[4] = n_tiles; d[5] = stage * 2 + (int)parity; d[6] = tl_begin; d[7] = n_rsi;
            }
            return false;
        }
        const int t0 = (tl_begin + it) * LS_T;
        if (active) {
            if (t0 == T0) { A.seg_in[seg] = make_int2(pos, pos != 0 ? entry_bar : -1); rec = true; }
            const float4* __restrict__ pp = reinterpret_cast<const float4*>(wtile + (size_t)stage * LS_ROWS * LS_STRIDE);
            const float4* __restrict__ rr = reinterpret_cast<const float4*>(wtile + ((size_t)stage * LS_ROWS + my_row) * LS_STRIDE);
            const float2* __restrict__ zp = wzone + (size_t)stage * LS_ROWS * ZR;
            const float2* __restrict__ zr = zp + my_row * ZR;
#pragma unroll 1
            for (int zb = 0; zb < ZB; ++zb) {
                if (ZONES) {
                    // nothing can fire in a block whose (min, max) stay inside the machine's thresholds; the skip is
                    // taken when NO machine of the warp can fire (a warp-uniform branch: a machine that could skip alone
                    // would wait for its neighbours anyway, and the divergent form costs the re-convergence on top)
                    const float2 rz = zr[zb], pz = zp[zb];
                    if (!__any_sync(amask, (rz.x < rlo) | (rz.y > rhi) | (pz.x <= plo) | (pz.y >= phi))) continue;
                }
#pragma unroll UNROLL
                for (int g = zb * (LS_ZONE / 4); g < (zb + 1) * (LS_ZONE / 4); ++g) {
                    bool hit;
                    if (ZONES) {
                        // the group's precomputed range decides whether any of its four bars can fire (tested against the
                        // machine's CURRENT thresholds: they move whenever it fires)
                        const float2 rm = zr[ZB + g], pm = zp[ZB + g];
                        hit = (rm.x < rlo) | (rm.y > rhi) | (pm.x <= plo) | (pm.y >= phi);
                        if (!hit) continue;
                    }
                    const float4 p = pp[g], r = rr[g];
                    if (!ZONES) {
                        // any bar of the four beyond a threshold?  (fminf / fmaxf drop NaNs, as the per-bar compares do)
                        const float r_min = fminf(fminf(r.x, r.y), fminf(r.z, r.w)), r_max = fmaxf(fmaxf(r.x, r.y), fmaxf(r.z, r.w));
                        const float p_min = fminf(fminf(p.x, p.y), fminf(p.z, p.w)), p_max = fmaxf(fmaxf(p.x, p.y), fmaxf(p.z, p.w));
                        hit = (r_min < rlo) | (r_max > rhi) | (p_min <= plo) | (p_max >= phi);
                    }
                    if (hit) {
                        const int t = t0 + g * 4;
                        step(p.x, r.x, t);
                        step(p.y, r.y, t + 1);
                        step(p.z, r.z, t + 2);
                        step(p.w, r.w, t + 3);
                    }
                }
            }
        }
        __syncwarp();      // every machine of the warp is done with the stage: refill it with the tile LS_STAGES ahead
        if (it + LS_STAGES < n_tiles) issue(tl_begin + it + LS_STAGES, stage);
        if (++stage == LS_STAGES) { stage = 0; parity ^= 1u; }
    }
    ring_stage = stage;
    ring_parity = parity;
    if (!active) return true;
    A.seg_out[seg] = make_int2(pos, pos != 0 ? entry_bar : -1);
    if (c == A.K - 1 && pos != 0)   // force-close at the last bar (:849-876; the last chunk always records: T0 < N)
        record((unsigned)(n - 1) | B200BT_EVENT_EXIT | (pos > 0 ? B200BT_EVENT_SELL : 0u), __ldg(A.price + (int64_t)sym * A.ld_price + (n - 1)));
    A.seg_count[seg] = dead ? SEG_LOST : count;
    return true;
}

// Persistent form: the grid is one resident set of CTAs; every WARP takes work items -- (warp-slot, chunk, symbol), the
// most expensive warp-slots first -- from a global counter until none is left, so all warp slots of the GPU stay busy until
// the queue is empty and the last items to run are the cheapest ones (a static grid left the busiest CTAs running alone
// at the end while the rest of their SM sat idle).
template <bool ZONES, int UNROLL>
__global__ void __launch_bounds__(LS_THREADS, B200BT_LS_MIN_BLOCKS)
lane_scan_kernel(const LaneScanArgs A, const bool vec16) {   // by value, not __grid_constant__ (see sweep.cu)
    // [LS_WARPS][LS_STAGES][LS_ROWS][LS_STRIDE] floats, then (ZONES) per warp and stage [LS_ROWS][LS_T / 32 + LS_T / 4] float2
    extern __shared__ __align__(16) float ls_tile[];
    __shared__ __align__(8) unsigned long long ls_full[LS_WARPS][LS_STAGES];   // "tile landed" (1 arrival + the copies' bytes)
    __shared__ float ls_mul[8][LS_THREADS];
    __shared__ double ls_tpsl[2][LS_THREADS];
    __shared__ const void* ls_src[LS_WARPS][LS_ROWS][3];
    constexpr int ZR = LS_T / LS_ZONE + LS_T / 4;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* const wtile = ls_tile + (size_t)warp * LS_STAGES * LS_ROWS * LS_STRIDE;
    float2* const wzone = reinterpret_cast<float2*>(ls_tile + (size_t)LS_WARPS * LS_STAGES * LS_ROWS * LS_STRIDE) + (size_t)warp * LS_STAGES * LS_ROWS * ZR;
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < LS_STAGES; ++s) mbar_init(&ls_full[warp][s], 1);
        mbar_fence_init();
        fence_proxy_async();
    }
    __syncwarp();
    int ring_stage = 0;            // the warp's position in its tile ring, carried from item to item
    unsigned ring_parity = 0;
    bool retired = false;          // a tile of this warp's ring did not arrive: the ring is not used again
    const int per_slot = A.K * A.S;
    const int n_items = (A.n_slots / 32) * per_slot;
    for (;;) {
        int item = 0;
        if (lane == 0) item = (int)atomicAdd(A.work, 1u);
        item = __shfl_sync(FULL, item, 0);
        if (item >= n_items) break;
        const int wslot = item / per_slot, rest = item - wslot * per_slot;
        const int c = rest / A.S, sym = rest - c * A.S;
        if (retired) { lane_scan_give_up(A, wslot, sym, c); continue; }     // (every item is either scanned or marked)
        retired = !lane_scan_item<ZONES, UNROLL>(A, vec16, wslot, sym, c, wtile, wzone, ls_full[warp], ls_mul, ls_tpsl, ls_src[warp],
                                            ring_stage, ring_parity);
        __syncwarp();
    }
}

// ---- metrics, chunk-parallel -------------------------------------------------------------------------
// The trade-record metrics are a fold over the lane's events in time order, but every piece of it is
// either a sum / max / xor (associative) or depends on the past only through the index of the chunk's
// first record -- except the max drawdown, which needs the equity and the running equity peak at the
// chunk's start (E0, P0).  A chunk whose equity never rises above the peak it inherits has drawdown
// (P0 - (E0 + smallest prefix)) / P0, so only the chunks that set a new peak need their records again:
//   chunk_partial_kernel warp per (chunk, symbol): exclusive sum of the record counts of the lane's earlier
//                        chunks -> record index, then the batch arithmetic (batch_core) over the chunk's own
//                        events into a ChunkPartial, plus the chunk's PnL sum and largest / smallest prefix sum.
//   chunk_prefix_kernel  thread per (individual, symbol): E0 / P0 of every chunk in time order; the drawdown of
//                        a chunk below its inherited peak in closed form, the others listed.
//   chunk_peak_kernel    warp per listed chunk: equity, running peak and drawdown record by record from E0 / P0.
//   lane_combine_kernel  thread per (individual, symbol): verifies the boundaries, merges the partials
//                        (calendar days that straddle a chunk boundary are re-joined) and finalises.
struct ChunkPartial {
    double tot_profit, tot_loss, largest_p, largest_l, maxdd, first_sum, pivot, s1, s2, day_sum;
    long long sum_dur;
    unsigned long long hash;
    unsigned n_win, n_loss, n_days, count;
    int first_done, first_day, day_cur;
    unsigned n_neg;
    double npivot, ns1, ns2;          // the chunk's finished negative days (DayAcc)
    double min_prefix;                // smallest equity of the chunk relative to its start (+inf: no records)
};
static_assert(sizeof(ChunkPartial) == 160, "ChunkPartial layout");

// One step of walk_records, per lane: records 4 lane + j (j = 0..3) of the step, priced.  A record that does not exist
// (a[j] false: the step's last lane may be partial) has PnL 0 and the equity of the record in front of it.
constexpr int WR_PER_LANE = 4;
constexpr int WR_STEP = 32 * WR_PER_LANE;     // records per step; CK_BLOCK is a whole number of steps
static_assert(CK_BLOCK % WR_STEP == 0, "a step never straddles two pool blocks");
struct RecordQuad {
    int cnt;                                  // records in the step (<= WR_STEP)
    bool a[WR_PER_LANE];
    unsigned w[WR_PER_LANE];                  // event words
    double pnl[WR_PER_LANE];                  // PnL of each record (0 for an entry)
    double eq[WR_PER_LANE];                   // equity after each record
    double sum;                               // the lane's PnL sum
    int dur[WR_PER_LANE];
};

// The records of chunk `seg` in time order, WR_STEP per step, four per lane (two 16-byte loads): every record is priced
// against the one before it (the lane's first by shuffle from the lane in front; lane 0's against the last record of the
// previous step, or the entry the chunk's verified start state holds), the equity runs on from `equity` by an in-lane
// prefix over the four PnLs and one inclusive warp scan, and body(quad, step's PnL sum) consumes the step.  -> the
// chunk's record count (0: lost).
template <class Body>
__device__ __forceinline__ unsigned walk_records(const uint2* __restrict__ pool, const int* __restrict__ next, const int pool_blocks,
                                                 const int* __restrict__ seg_first, const unsigned* __restrict__ seg_count,
                                                 const int2* __restrict__ seg_in, const float* __restrict__ pr, const int seg,
                                                 const double size, double& equity, Body&& body) {
    const int lane = threadIdx.x & 31;
    const double fee1 = __dmul_rn(size, 0.001), fee2 = __dmul_rn(size, 0.002);
    const unsigned count = seg_records(seg_count[seg]);
    unsigned left = count;
    const int2 in = seg_in[seg];
    unsigned w_carry = 0u;
    float p_carry = 0.f;
    if (in.x != 0) {
        w_carry = (unsigned)in.y | (in.x < 0 ? B200BT_EVENT_SELL : 0u);
        p_carry = __ldg(pr + in.y);
    }
    int b = left ? seg_first[seg] : -1, off = 0;
    if ((unsigned)b >= (unsigned)pool_blocks) left = 0;
    while (left) {
        RecordQuad r;
        r.cnt = (int)min((unsigned)WR_STEP, left);
        const int first = WR_PER_LANE * lane;
#pragma unroll
        for (int j = 0; j < WR_PER_LANE; ++j) r.a[j] = first + j < r.cnt;
        const uint4* src = reinterpret_cast<const uint4*>(pool + (int64_t)b * CK_BLOCK + off + first);
        const uint4 e01 = r.a[0] ? src[0] : make_uint4(0u, 0u, 0u, 0u);
        const uint4 e23 = r.a[2] ? src[1] : make_uint4(0u, 0u, 0u, 0u);
        r.w[0] = e01.x; r.w[1] = e01.z; r.w[2] = e23.x; r.w[3] = e23.z;
        const float pf[WR_PER_LANE] = {__uint_as_float(e01.y), __uint_as_float(e01.w), __uint_as_float(e23.y), __uint_as_float(e23.w)};
        float p_prev = __shfl_up_sync(FULL, pf[3], 1);
        unsigned w_prev = __shfl_up_sync(FULL, r.w[3], 1);
        if (lane == 0) { p_prev = p_carry; w_prev = w_carry; }
        double run = 0.0;                         // in-lane prefix of the PnLs
#pragma unroll
        for (int j = 0; j < WR_PER_LANE; ++j) {
            r.pnl[j] = record_pnl(r.a[j], r.w[j], pf[j], j ? r.w[j - 1] : w_prev, j ? pf[j - 1] : p_prev, size, fee1, fee2, r.dur[j]);
            run = j ? run + r.pnl[j] : r.pnl[j];
            r.eq[j] = run;
        }
        r.sum = run;
        double cs = run;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const double up = shfl_up_d(cs, d);
            if (lane >= d) cs += up;
        }
        const double base = equity + (cs - run);  // equity in front of the lane's first record
#pragma unroll
        for (int j = 0; j < WR_PER_LANE; ++j) r.eq[j] = base + r.eq[j];
        const double step_sum = shfl_d(cs, 31);
        equity += step_sum;
        body(r, step_sum);
        // (only a full step is followed by another one: its last record is lane 31's last)
        w_carry = __shfl_sync(FULL, r.w[3], 31);
        p_carry = __shfl_sync(FULL, pf[3], 31);
        left -= r.cnt;
        off += WR_STEP;
        if (off == CK_BLOCK && left) { b = next[b]; off = 0; if ((unsigned)b >= (unsigned)pool_blocks) break; }
    }
    return count;
}

#ifndef B200BT_M2_MIN_BLOCKS
#define B200BT_M2_MIN_BLOCKS 5      // 96 registers, 20 B spilled (nvcc 12.9, sm_90a); at 4 CTAs/SM (108, no spill) ~6 % slower
#endif
__global__ void __launch_bounds__(128, B200BT_M2_MIN_BLOCKS)
chunk_partial_kernel(const float* __restrict__ price, int64_t ld_price, const b200bt_individual* __restrict__ indiv,
                     const b200bt_chunk_item* __restrict__ items, int n_items, int S, int n_seg,
                     const uint2* __restrict__ pool, const int* __restrict__ next, const int* __restrict__ seg_first,
                     const unsigned* __restrict__ seg_count, const int2* __restrict__ seg_in,
                     double* __restrict__ seg_sum, double* __restrict__ seg_max,
                     const b200bt_sweep_config cfg, uint32_t* __restrict__ events, int64_t ev_cap,
                     ChunkPartial* __restrict__ partial, const int* __restrict__ n_items_dev, int pool_blocks) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int sym = (int)(blockIdx.x % (unsigned)S);
    const int it = (int)(blockIdx.x / (unsigned)S) * 4 + wid;
    if (it >= (n_items_dev ? *n_items_dev : n_items)) return;
    const b200bt_chunk_item item = items[it];
    const int seg = sym * n_seg + item.segment;
    const int base = seg - item.chunk;
    const b200bt_individual iv = indiv[item.individual];

    // index of the chunk's first record: exclusive sum over the lane's earlier chunks
    unsigned first_index = 0;
    for (int c0 = 0; c0 < item.chunk; c0 += 32) {
        const int c = c0 + lane;
        first_index += __reduce_add_sync(FULL, c < item.chunk ? seg_records(seg_count[base + c]) : 0u);
    }

    // Order-dependent state (equity relative to the chunk's start, calendar day) is warp-uniform and lives in registers;
    // what is a plain sum / max / min / xor over the records is accumulated PER LANE and reduced once at the end of the chunk.
    double equity = 0.0, l_top = -INFINITY, l_bottom = INFINITY;
    DayAcc da{0.0, 0.0, 0.0, 0u, 0};   // this lane's share of the chunk's finished days (merged in lane order at the end)
    int day_valid = 0, day_cur = 0, first_done = 0, first_id = 0;
    double day_sum = 0.0, first_sum = 0.0;
    unsigned index = first_index;
    double l_gain = 0.0, l_loss = 0.0, l_maxp = 0.0, l_minl = 0.0;
    unsigned l_win = 0, l_los = 0, l_dur = 0;   // (l_dur: a lane's trades do not overlap, so the chunk's sum is < N < 2^30)
    unsigned l_hlo = 0u, l_hhi = 0u;
    uint32_t* const ev_out = events ? events + ((int64_t)item.individual * S + sym) * ev_cap : nullptr;
    const unsigned minute0 = (unsigned)cfg.minute0, bar_minutes = (unsigned)cfg.bar_minutes;
    const unsigned gap_bar = cfg.gap_bar > 0 ? (unsigned)cfg.gap_bar : 0xffffffffu, gap_minutes = (unsigned)cfg.gap_minutes;
    auto day_of = [&](unsigned w) {   // calendar day of a record (a glued series jumps gap_minutes at gap_bar)
        const unsigned bar = w & B200BT_EVENT_BAR_MASK;
        return (int)((minute0 + bar * bar_minutes + (bar >= gap_bar ? gap_minutes : 0u)) / 1440u);
    };
    constexpr int R = WR_PER_LANE;

    // equity relative to the chunk's start
    const unsigned count = walk_records(pool, next, pool_blocks, seg_first, seg_count, seg_in, price + (int64_t)sym * ld_price, seg,
                                        iv.position_size, equity, [&](const RecordQuad& r, const double batch_sum) {
        const int cnt = r.cnt;
        const unsigned i0 = index + R * lane;
        int d[R];                     // calendar day of each record (a missing record: its predecessor's)
#pragma unroll
        for (int j = 0; j < R; ++j) {
            const double pnl = r.pnl[j];
            if (pnl > 0.0) { l_gain += pnl; ++l_win; l_maxp = fmax(l_maxp, pnl); }
            else if (pnl < 0.0) { l_loss += pnl; ++l_los; l_minl = fmin(l_minl, pnl); }
            l_dur += (unsigned)r.dur[j];
            if (r.a[j]) {
                const unsigned long long h = event_hash(i0 + j, r.w[j]);
                l_hlo ^= (unsigned)h; l_hhi ^= (unsigned)(h >> 32);
                if (ev_out && (int64_t)i0 + j < ev_cap) ev_out[i0 + j] = r.w[j];
                l_top = fmax(l_top, r.eq[j]); l_bottom = fmin(l_bottom, r.eq[j]);
            }
            d[j] = r.a[j] ? day_of(r.w[j]) : (j ? d[j - 1] : 0);
        }

        // calendar-day buckets
        const int last_lane = (cnt - 1) / R;
        const int first_day = __shfl_sync(FULL, d[0], 0);
        const int last_day = __shfl_sync(FULL, d[R - 1], last_lane);
        if (first_day == last_day && (!day_valid || first_day == day_cur)) {
            day_sum = (day_valid ? day_sum : 0.0) + batch_sum;      // the whole step falls into the open day
        } else {
            // a record is a HEAD if it opens a day within the step; running day sum = segmented scan by heads, in-lane
            // over the four records, then across the warp.  As a function of the running sum it receives, a lane is
            // either additive (no head) or constant.
            const bool merge_carry = day_valid && (first_day == day_cur);
            const int d_before = __shfl_up_sync(FULL, d[R - 1], 1);
            bool head[R];
            double part[R];           // running day sum of the lane's own records (from its last head)
            bool flag = false;
#pragma unroll
            for (int j = 0; j < R; ++j) {
                head[j] = r.a[j] && (j ? d[j] != d[j - 1] : (lane == 0 ? !merge_carry : d[0] != d_before));
                part[j] = (j == 0 || head[j]) ? r.pnl[j] : part[j - 1] + r.pnl[j];
                flag = flag || head[j];
            }
            double sg = part[R - 1];
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const double up = shfl_up_d(sg, s);
                const int fup = __shfl_up_sync(FULL, (int)flag, s);
                if (lane >= s && !flag) { sg += up; flag = fup; }
            }
            // (the open day carried in is part of lane 0's chain when it continues)
            if (merge_carry && !flag) sg += day_sum;          // lanes whose chain reaches back to the step's start
            double carry_in = shfl_up_d(sg, 1);
            if (lane == 0) carry_in = merge_carry ? day_sum : 0.0;
            // running day sum after each record: records behind a head of their own lane have it in part[]
            double run[R];
            bool seen = false;
#pragma unroll
            for (int j = 0; j < R; ++j) {
                seen = seen || head[j];
                run[j] = seen ? part[j] : carry_in + part[j];
            }
            // TAIL = last record of its day within the step, except the step's last record (its day stays open)
            const int d_after = __shfl_down_sync(FULL, d[0], 1);
            unsigned tails = 0u;      // bit j: record j is a tail
#pragma unroll
            for (int j = 0; j < R - 1; ++j) tails |= (r.a[j] && head[j + 1]) ? 1u << j : 0u;
            tails |= (r.a[R - 1] && lane < last_lane && d_after != d[R - 1]) ? 1u << (R - 1) : 0u;
            // Finished days go to the lane that closes them; the chunk's first finished day, which may continue the
            // previous chunk's last one, is kept aside (first_sum).  A day carried in that ends at the step's start
            // comes before every tail of the step.
            if (day_valid && !merge_carry) {
                if (!first_done) { first_done = 1; first_id = day_cur; first_sum = day_sum; }
                else if (lane == 0) day_complete(da, day_sum);
            }
            if (!first_done) {
                const unsigned lanes_with = __ballot_sync(FULL, tails != 0u);
                if (lanes_with) {
                    const int src = __ffs(lanes_with) - 1;
                    const int j = __ffs(tails) - 1;   // (this lane's first tail)
                    const double x = j == 0 ? run[0] : j == 1 ? run[1] : j == 2 ? run[2] : run[3];
                    const int id = j == 0 ? d[0] : j == 1 ? d[1] : j == 2 ? d[2] : d[3];
                    first_sum = shfl_d(x, src);
                    first_id = __shfl_sync(FULL, id, src);
                    first_done = 1;
                    if (lane == src) tails &= tails - 1u;
                }
            }
#pragma unroll
            for (int j = 0; j < R; ++j)
                if (tails & (1u << j)) day_complete(da, run[j]);
            day_sum = shfl_d(run[R - 1], last_lane);          // (a missing record repeats its predecessor's run)
        }
        day_cur = last_day;
        day_valid = 1;
        index += cnt;
    });
    // per-lane accumulators -> chunk totals
    const double tot_profit = warp_sum_d(l_gain), tot_loss = warp_sum_d(l_loss);
    const double largest_p = warp_max_d(l_maxp), largest_l = warp_min_d(l_minl);
    unsigned n_win, n_loss;
    if (count < 0x10000u) {           // both counts fit a 16-bit half: one reduction
        const unsigned both = __reduce_add_sync(FULL, l_win | (l_los << 16));
        n_win = both & 0xffffu; n_loss = both >> 16;
    } else {
        n_win = __reduce_add_sync(FULL, l_win); n_loss = __reduce_add_sync(FULL, l_los);
    }
    const long long sum_dur = (long long)__reduce_add_sync(FULL, l_dur);
    const unsigned hlo = __reduce_xor_sync(FULL, l_hlo), hhi = __reduce_xor_sync(FULL, l_hhi);
    double top = l_top, bottom = l_bottom;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
        top = fmax(top, shfl_xor_d(top, m));
        bottom = fmin(bottom, shfl_xor_d(bottom, m));
    }
    // the lanes' finished days, merged in lane order (lane l takes lane l + s's, which come after its own)
    if (__any_sync(FULL, da.n_days != 0u)) {
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            DayAcc o;
            o.pivot = __shfl_down_sync(FULL, da.pivot, s); o.s1 = __shfl_down_sync(FULL, da.s1, s);
            o.s2 = __shfl_down_sync(FULL, da.s2, s); o.n_days = __shfl_down_sync(FULL, da.n_days, s); o.pivot_set = 1;
            o.npivot = __shfl_down_sync(FULL, da.npivot, s); o.ns1 = __shfl_down_sync(FULL, da.ns1, s);
            o.ns2 = __shfl_down_sync(FULL, da.ns2, s); o.n_neg = __shfl_down_sync(FULL, da.n_neg, s);
            if (lane + s < 32) day_merge(da, o);
        }
    }
    if (lane == 0) {
        ChunkPartial q;
        q.tot_profit = tot_profit; q.tot_loss = tot_loss; q.largest_p = largest_p; q.largest_l = largest_l;
        q.maxdd = 0.0; q.first_sum = first_sum; q.pivot = da.pivot; q.s1 = da.s1; q.s2 = da.s2; q.day_sum = day_sum;
        q.sum_dur = sum_dur; q.hash = ((unsigned long long)hhi << 32) | hlo;
        q.n_win = n_win; q.n_loss = n_loss; q.n_days = da.n_days; q.count = count;
        q.first_done = first_done; q.first_day = first_id; q.day_cur = day_cur;
        q.n_neg = da.n_neg; q.npivot = da.npivot; q.ns1 = da.ns1; q.ns2 = da.ns2; q.min_prefix = bottom;
        partial[seg] = q;
        seg_sum[seg] = equity;
        seg_max[seg] = top;
    }
}

// Drawdown, thread per (individual, symbol): the chunks' PnL sums and largest prefixes give every chunk's starting equity E0
// and inherited peak P0, in time order.  A chunk that does not rise above P0 (E0 + largest prefix <= P0: the strict > of the
// running peak's update) has drawdown (P0 - (E0 + smallest prefix)) / P0 when positive -- division by a fixed P0 is monotone,
// so that is the largest of its records' values.  A chunk that sets a new peak is listed for chunk_peak_kernel, its seg_sum /
// seg_max overwritten with E0 / P0.
__global__ void __launch_bounds__(128)
chunk_prefix_kernel(int pop, int S, const int32_t* __restrict__ seg_base, const int32_t* __restrict__ n_chunks, int n_seg,
                    double* __restrict__ seg_sum, double* __restrict__ seg_max, ChunkPartial* __restrict__ partial,
                    double initial_capital, int4* __restrict__ peaks, unsigned* __restrict__ n_peaks) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)pop * S) return;
    const int ind = (int)(t / S), sym = (int)(t % S);
    const int K = n_chunks[ind];
    const int base = sym * n_seg + seg_base[ind];
    double e0 = initial_capital, p0 = initial_capital;
    for (int c = 0; c < K; ++c) {
        const int seg = base + c;
        const double sum = seg_sum[seg], top = __dadd_rn(e0, seg_max[seg]);   // (a chunk without records: 0, -inf)
        if (top > p0) {
            seg_sum[seg] = e0;
            seg_max[seg] = p0;
            peaks[atomicAdd(n_peaks, 1u)] = make_int4(seg, ind, sym, 0);
        } else {
            const double gap = __dsub_rn(p0, __dadd_rn(e0, partial[seg].min_prefix));
            partial[seg].maxdd = gap > 0.0 ? __ddiv_rn(gap, p0) : 0.0;
        }
        p0 = fmax(p0, top);
        e0 = __dadd_rn(e0, sum);
    }
}

// Drawdown of the listed chunks (chunk_prefix_kernel), one warp per chunk over a device-side count: equity from E0, running
// peak from P0 and the drawdown candidates record by record (the arithmetic of batch_core, four records per lane).
__global__ void __launch_bounds__(128)
chunk_peak_kernel(const float* __restrict__ price, int64_t ld_price, const b200bt_individual* __restrict__ indiv,
                  const uint2* __restrict__ pool, const int* __restrict__ next, const int* __restrict__ seg_first,
                  const unsigned* __restrict__ seg_count, const int2* __restrict__ seg_in, const double* __restrict__ seg_e0,
                  const double* __restrict__ seg_p0, const int4* __restrict__ peaks, const unsigned* __restrict__ n_peaks,
                  ChunkPartial* __restrict__ partial, int pool_blocks) {
    const int lane = threadIdx.x & 31;
    const unsigned n = *n_peaks, warps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const int4 pk = peaks[i];
        const int seg = pk.x;
        double equity = seg_e0[seg], peak = seg_p0[seg], maxdd = 0.0;
        walk_records(pool, next, pool_blocks, seg_first, seg_count, seg_in, price + (int64_t)pk.z * ld_price, seg,
                     indiv[pk.y].position_size, equity, [&](const RecordQuad& r, double) {
            constexpr int R = WR_PER_LANE;
            double m = -INFINITY;                          // the lane's largest equity
#pragma unroll
            for (int j = 0; j < R; ++j) m = fmax(m, r.a[j] ? r.eq[j] : -INFINITY);
            double pkj[R];
#pragma unroll
            for (int j = 0; j < R; ++j) pkj[j] = peak;
            if (__any_sync(FULL, m > peak)) {
                double p = m;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const double up = shfl_up_d(p, d);
                    if (lane >= d) p = fmax(p, up);
                }
                double before = shfl_up_d(p, 1);           // peak over the records of the lanes in front
                before = fmax(lane == 0 ? peak : before, peak);
#pragma unroll
                for (int j = 0; j < R; ++j) pkj[j] = fmax(j ? pkj[j - 1] : before, r.eq[j]);
                peak = fmax(peak, shfl_d(p, 31));
            }
            const double lim = maxdd * (1.0 - 1e-12);
            double cand = 0.0;
            bool any = false;
#pragma unroll
            for (int j = 0; j < R; ++j) {
                const double gap = __dsub_rn(pkj[j], r.eq[j]);
                const bool c = r.a[j] && gap > 0.0 && gap >= lim * pkj[j];
                if (c) cand = fmax(cand, __ddiv_rn(gap, pkj[j]));
                any = any || c;
            }
            if (__any_sync(FULL, any)) maxdd = fmax(maxdd, warp_max_d(cand));
        });
        if (lane == 0) partial[seg].maxdd = maxdd;
    }
}

// Work items (all chunks) of the individuals flagged in `redo`, for the recomputation after the overlapped repairs.
__global__ void fix_items_kernel(const b200bt_chunk_item* __restrict__ items, int n_items, const unsigned char* __restrict__ redo,
                                 b200bt_chunk_item* __restrict__ out, int* __restrict__ n_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const b200bt_chunk_item it = items[i];
    if (redo[it.individual]) out[atomicAdd(n_out, 1)] = it;
}

// Individuals with a lane the chunked evaluation could not settle (a boundary still inconsistent after the repair passes, a
// full event pool, a warp not packed for the thread-per-lane scan): listed on the device for the exact fallback.
__global__ void redo_list_kernel(int pop, int S, const unsigned char* __restrict__ invalid, int32_t* __restrict__ list,
                                 int* __restrict__ n_list, int* __restrict__ n_invalid_lanes) {
    const int ind = blockIdx.x * blockDim.x + threadIdx.x;
    if (ind >= pop) return;
    int bad = 0;
    for (int s = 0; s < S; ++s) bad += invalid[(int64_t)ind * S + s] ? 1 : 0;
    if (bad) {
        list[atomicAdd(n_list, 1)] = ind;
        atomicAdd(n_invalid_lanes, bad);
    }
}

__global__ void lane_combine_kernel(const b200bt_individual* __restrict__ indiv, int pop, int S,
                                    const int32_t* __restrict__ seg_base, const int32_t* __restrict__ n_chunks, int n_seg,
                                    const unsigned* __restrict__ seg_count, const int2* __restrict__ seg_in,
                                    const int2* __restrict__ seg_out, const ChunkPartial* __restrict__ partial,
                                    const b200bt_sweep_config cfg, b200bt_lane_stats* __restrict__ stats,
                                    unsigned char* __restrict__ invalid) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)pop * S) return;
    const int ind = (int)(t / S), sym = (int)(t % S);
    const int K = n_chunks[ind];
    const int base = sym * n_seg + seg_base[ind];
    bool ok = true;
    for (int c = 0; c < K; ++c) {
        const int2 a = seg_in[base + c];
        if (c == 0) ok = ok && (a.x == 0);
        else {
            const int2 z = seg_out[base + c - 1];
            ok = ok && (a.x == z.x) && (a.y == z.y);
        }
        ok = ok && (seg_count[base + c] != SEG_LOST);
    }
    invalid[t] = ok ? 0 : 1;
    if (!ok) return;
    WarpAcc a;
    init_acc(a, indiv[ind], cfg, nullptr);
    DayAcc da{0.0, 0.0, 0.0, 0u, 0};
    bool open = false;      // the lane's open (last, not yet finished) calendar day
    int open_day = 0;
    double open_sum = 0.0;
    for (int c = 0; c < K; ++c) {
        const ChunkPartial q = partial[base + c];
        if (q.count == 0) continue;
        a.n_events += q.count;
        a.n_win += q.n_win; a.n_loss += q.n_loss;
        a.tot_profit += q.tot_profit; a.tot_loss += q.tot_loss;
        a.largest_p = fmax(a.largest_p, q.largest_p); a.largest_l = fmin(a.largest_l, q.largest_l);
        a.maxdd = fmax(a.maxdd, q.maxdd);
        a.sum_dur += q.sum_dur;
        a.hash ^= q.hash;
        if (!q.first_done) {
            // the whole chunk lies in one calendar day, which stays open
            if (open && open_day == q.day_cur) open_sum += q.day_sum;
            else {
                if (open) day_complete(da, open_sum);
                open = true; open_day = q.day_cur; open_sum = q.day_sum;
            }
            continue;
        }
        double x = q.first_sum;
        if (open) {
            if (open_day == q.first_day) x += open_sum; else day_complete(da, open_sum);
        }
        day_complete(da, x);
        // the chunk's own finished days, accumulated about its pivots: shifted to the lane's
        day_merge(da, DayAcc{q.pivot, q.s1, q.s2, q.n_days, 1, q.npivot, q.ns1, q.ns2, q.n_neg});
        open = true; open_day = q.day_cur; open_sum = q.day_sum;
    }
    a.pivot = da.pivot; a.s1 = da.s1; a.s2 = da.s2; a.n_days = da.n_days; a.pivot_set = da.pivot_set;
    a.npivot = da.npivot; a.ns1 = da.ns1; a.ns2 = da.ns2; a.n_neg = da.n_neg;
    a.day_valid = open ? 1 : 0; a.day_sum = open_sum; a.day_cur = open_day;
    b200bt_lane_stats o;
    finalize_lane(a, cfg, o);
    stats[t] = o;
}

}  // namespace b200bt

using namespace b200bt;

namespace {

// The sweep workspace: byte offsets of its sections, each 16-byte aligned (so must the base be), and its size.  segs =
// S x n_seg chunks; `tables`: b200bt_sweep_tiled's work items, seg_base and n_chunks of its uniform chunks.  The sections
// in front of `cleared` are zeroed at the start of every sweep.
struct ChunkLayout {
    int64_t seg_in, seg_out, seg_first, seg_count, counters, redo, cleared;
    int64_t pool, next, peaks, partial, seg_sum, seg_max, fix_items, items, seg_base, n_chunks, bytes;
};

ChunkLayout chunk_layout(int pool_blocks, int64_t segs, int n_seg, int pop, bool tables) {
    ChunkLayout L;
    int64_t at = 0;
    auto section = [&](int64_t bytes) { const int64_t o = at; at += (bytes + 15) & ~(int64_t)15; return o; };
    L.seg_in = section(segs * sizeof(int2));
    L.seg_out = section(segs * sizeof(int2));
    L.seg_first = section(segs * sizeof(int));
    L.seg_count = section(segs * sizeof(unsigned));
    L.counters = section(sizeof(SweepCounters));
    L.redo = section(pop);                                            // individuals the overlapped repair touched
    L.cleared = at;
    L.pool = section((int64_t)pool_blocks * CK_BLOCK * sizeof(uint2));
    L.next = section((int64_t)pool_blocks * sizeof(int));
    L.peaks = section(segs * sizeof(int4));                           // chunks that set a new equity peak
    L.partial = section(segs * sizeof(ChunkPartial));
    L.seg_sum = section(segs * sizeof(double));
    L.seg_max = section(segs * sizeof(double));
    L.fix_items = section((int64_t)n_seg * sizeof(b200bt_chunk_item));   // fix-up items, then the exact fallback's list
    L.items = section(tables ? (int64_t)n_seg * sizeof(b200bt_chunk_item) : 0);
    L.seg_base = section(tables ? (int64_t)pop * sizeof(int32_t) : 0);
    L.n_chunks = section(tables ? (int64_t)pop * sizeof(int32_t) : 0);
    L.bytes = at;
    return L;
}

struct ChunkWorkspace : ChunkTables {
    SweepCounters* ctr; int4* peaks; ChunkPartial* partial; double* seg_sum; double* seg_max;
    b200bt_chunk_item* fix_items; unsigned char* redo;
    b200bt_chunk_item* items; int32_t* seg_base; int32_t* n_chunks;
};

ChunkWorkspace carve(void* workspace, const ChunkLayout& L, int pool_blocks) {
    unsigned char* const at = (unsigned char*)workspace;
    ChunkWorkspace w;
    w.pool = (uint2*)(at + L.pool); w.pool_blocks = pool_blocks; w.next = (int*)(at + L.next);
    w.seg_first = (int*)(at + L.seg_first); w.seg_count = (unsigned*)(at + L.seg_count);
    w.seg_in = (int2*)(at + L.seg_in); w.seg_out = (int2*)(at + L.seg_out);
    w.ctr = (SweepCounters*)(at + L.counters);
    w.alloc = &w.ctr->alloc; w.overflow = &w.ctr->overflow;
    w.peaks = (int4*)(at + L.peaks); w.partial = (ChunkPartial*)(at + L.partial);
    w.seg_sum = (double*)(at + L.seg_sum); w.seg_max = (double*)(at + L.seg_max);
    w.fix_items = (b200bt_chunk_item*)(at + L.fix_items); w.redo = at + L.redo;
    w.items = (b200bt_chunk_item*)(at + L.items); w.seg_base = (int32_t*)(at + L.seg_base); w.n_chunks = (int32_t*)(at + L.n_chunks);
    return w;
}

// arguments of the warp-per-chunk scan and of the repair and metrics kernels both schedules share
ChunkScanArgs scan_args(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                        const b200bt_individual* indiv, const b200bt_chunk_item* items, int n_items, int n_seg,
                        const int32_t* n_chunks, int warm, const ChunkWorkspace& w) {
    ChunkScanArgs A;
    static_cast<ChunkTables&>(A) = w;
    A.price = price; A.ld_price = ld_price; A.rsi = rsi; A.ld_rsi = ld_rsi; A.P = P; A.S = S; A.N = N;
    A.indiv = indiv; A.items = items; A.n_items = n_items; A.n_seg = n_seg; A.warm = warm;
    A.n_chunks = n_chunks; A.redo = nullptr;
    return A;
}

// second stream + events for the overlapped repair tail, one set per device
struct SideStream { cudaStream_t stream = nullptr; cudaEvent_t fork = nullptr, join = nullptr; };
int side_stream(SideStream** out) {
    static SideStream table[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return cuda_status(e, "cudaGetDevice");
    B200BT_REQUIRE(dev >= 0 && dev < 64, B200BT_ELIMIT, "device ordinal %d out of range", dev);
    SideStream& s = table[dev];
    if (!s.stream) {
        int lo_p = 0, hi_p = 0;
        cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p);   // highest priority: its few small kernels go first
        e = cudaStreamCreateWithPriority(&s.stream, cudaStreamNonBlocking, hi_p);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming);
        if (e != cudaSuccess) { s.stream = nullptr; return cuda_status(e, "side stream"); }
    }
    *out = &s;
    return B200BT_OK;
}

// Everything after the speculative scan: verify + repair (lane_repair_kernel) -> chunk-parallel metrics.
//
// chunk_repair_kernel on the critical path makes almost every lane consistent; what it leaves is a handful of lanes whose
// trajectories do not meet the recorded ones inside a chunk (always in the market) and which have to be re-scanned chunk
// after chunk by a single warp each.  That is lane_repair_kernel, on another stream BESIDE the metrics kernels of all
// lanes; the individuals it touches are flagged and only their metrics are recomputed afterwards.
// max_repair_rounds: 0 = no repair (every inconsistent lane takes the exact fallback), 1 = chunk_repair_kernel only, >= 2 = both.
int finish_chunks(const ChunkScanArgs& A, const ChunkWorkspace& w, const bool vec16, const int32_t* seg_base, int pop,
                  int max_repair_rounds, const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats, uint32_t* events,
                  int64_t event_cap, unsigned char* lane_invalid, int* overflow_host_or_null, cudaStream_t st) {
    const int S = A.S, n_seg = A.n_seg, n_items = A.n_items;
    const b200bt_chunk_item* const items = A.items;
    auto kern_fix = vec16 ? chunk_repair_kernel<true> : chunk_repair_kernel<false>;
    auto kern_walk = vec16 ? lane_repair_kernel<true> : lane_repair_kernel<false>;
    int rc = allow_sw_smem(kern_fix, "sweep_chunked: cudaFuncSetAttribute");
    if (!rc) rc = allow_sw_smem(kern_walk, "sweep_chunked: cudaFuncSetAttribute");
    if (rc) return rc;
    const int64_t lanes = (int64_t)pop * S;
    const int64_t mblocks = (int64_t)((n_items + 3) / 4) * S;
    B200BT_REQUIRE(mblocks < (1ll << 31), B200BT_ELIMIT, "sweep_chunked: too many work items");
    B200BT_REQUIRE(lanes < (1ll << 30), B200BT_ELIMIT, "sweep_chunked: too many lanes");

    // Both repair kernels run a persistent grid (3 CTAs per SM) whose warps take work from a counter.
    const unsigned repair_grid = 3u * (unsigned)device_sm_count();
    auto repair_pass = [&](cudaStream_t rs, int pass, unsigned char* redo) -> int {
        ChunkScanArgs R = A;
        R.redo = redo;
        if (pass == 0) kern_fix<<<repair_grid, SW_WARPS * 32, SW_SMEM, rs>>>(R, &w.ctr->chunk_repair_work);
        else kern_walk<<<repair_grid, SW_WARPS * 32, SW_SMEM, rs>>>(R, pop, seg_base, &w.ctr->lane_repair_work);
        B200BT_LAUNCH_CHECK("repair launch");
        return B200BT_OK;
    };
    // (the fix-up pass reuses the full-size grid with a device-side item count: CTAs beyond it leave at once)
    auto metrics = [&](const b200bt_chunk_item* its, const int* n_dev) -> int {
        chunk_partial_kernel<<<(unsigned)mblocks, 128, 0, st>>>(A.price, A.ld_price, A.indiv, its, n_items, S, n_seg, w.pool, w.next,
                                                                 w.seg_first, w.seg_count, w.seg_in, w.seg_sum, w.seg_max,
                                                                 *cfg_host, events, event_cap, w.partial, n_dev, A.pool_blocks);
        B200BT_LAUNCH_CHECK("chunk_partial launch");
        return B200BT_OK;
    };

    cudaError_t e;
    const bool tail = max_repair_rounds >= 2;
    if (max_repair_rounds >= 1 && (rc = repair_pass(st, 0, nullptr))) return rc;
    SideStream* side = nullptr;
    if (tail) {
        if ((rc = side_stream(&side))) return rc;
        e = cudaEventRecord(side->fork, st);
        if (e != cudaSuccess) return cuda_status(e, "sweep_chunked: fork");
    }
    if ((rc = metrics(items, nullptr))) return rc;
    if (tail) {
        e = cudaStreamWaitEvent(side->stream, side->fork, 0);
        if (e != cudaSuccess) return cuda_status(e, "sweep_chunked: side wait");
        if ((rc = repair_pass(side->stream, 1, w.redo))) return rc;
        e = cudaEventRecord(side->join, side->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(st, side->join, 0);
        if (e != cudaSuccess) return cuda_status(e, "sweep_chunked: join");
        fix_items_kernel<<<(n_items + 255) / 256, 256, 0, st>>>(items, n_items, w.redo, w.fix_items, &w.ctr->n_fix_items);
        B200BT_LAUNCH_CHECK("fix_items launch");
        if ((rc = metrics(w.fix_items, &w.ctr->n_fix_items))) return rc;
    }
    // drawdown: chunks below their inherited peak in closed form, the chunks that set a new peak record by record
    // (a persistent grid walks their list)
    chunk_prefix_kernel<<<(unsigned)((lanes + 127) / 128), 128, 0, st>>>(pop, S, seg_base, A.n_chunks, n_seg, w.seg_sum, w.seg_max,
                                                                        w.partial, cfg_host->initial_capital, w.peaks,
                                                                        &w.ctr->peak_chunks);
    B200BT_LAUNCH_CHECK("chunk_prefix launch");
    chunk_peak_kernel<<<8u * (unsigned)device_sm_count(), 128, 0, st>>>(A.price, A.ld_price, A.indiv, w.pool, w.next, w.seg_first,
                                                                       w.seg_count, w.seg_in, w.seg_sum, w.seg_max, w.peaks,
                                                                       &w.ctr->peak_chunks, w.partial, A.pool_blocks);
    B200BT_LAUNCH_CHECK("chunk_peak launch");
    lane_combine_kernel<<<(unsigned)((lanes + 127) / 128), 128, 0, st>>>(A.indiv, pop, S, seg_base, A.n_chunks, n_seg, w.seg_count,
                                                                        w.seg_in, w.seg_out, w.partial, *cfg_host, stats,
                                                                        lane_invalid);
    B200BT_LAUNCH_CHECK("lane_combine launch");
    // exact fallback, driven from the device: the flagged individuals are listed and re-evaluated by the fused (serial)
    // kernel; with nothing flagged its warps leave at once.
    int32_t* redo_list = reinterpret_cast<int32_t*>(w.fix_items);      // (the fix-up item list is no longer needed)
    redo_list_kernel<<<(pop + 127) / 128, 128, 0, st>>>(pop, S, lane_invalid, redo_list, &w.ctr->n_redo, &w.ctr->fallback_lanes);
    B200BT_LAUNCH_CHECK("redo_list launch");
    if ((rc = launch_sweep(A.price, A.ld_price, A.rsi, A.ld_rsi, A.P, S, A.N, A.indiv, redo_list, pop, &w.ctr->n_redo, cfg_host,
                           stats, events, event_cap, st)))
        return rc;
    if (overflow_host_or_null) {   // (read by the host after its next sync)
        e = cudaMemcpyAsync(overflow_host_or_null, w.ctr, SWEEP_FLAGS * sizeof(int), cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) return cuda_status(e, "sweep_chunked: overflow readback");
    }
    if (trace_launches()) {
        SweepCounters c;
        const int* d = c.stall;
        if (cudaMemcpy(&c, w.ctr, sizeof(c), cudaMemcpyDeviceToHost) == cudaSuccess && c.stalls)
            fprintf(stderr, "[b200bt] lane_scan: %d tile(s) timed out; first: block %d warp %d item(wslot,sym,c) %d,%d,%d tile %d of %d stage %d parity %d tl_begin %d rows %d\n",
                    c.stalls, d[0], d[1], d[2] >> 16, (d[2] >> 8) & 255, d[2] & 255, d[3], d[4], d[5] >> 1, d[5] & 1, d[6], d[7]);
    }
    return B200BT_OK;
}

}  // namespace

extern "C" int64_t b200bt_sweep_chunked_workspace_bytes(int pool_blocks, int S, int n_seg) {
    return chunk_layout(pool_blocks, (int64_t)S * n_seg, n_seg, n_seg, false).bytes;   // pop <= n_seg
}

extern "C" int b200bt_sweep_chunked(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S,
                                    int64_t N, const b200bt_individual* indiv, const int32_t* order, int pop,
                                    const b200bt_chunk_item* items, int n_items, const int32_t* seg_base,
                                    const int32_t* n_chunks, int n_seg, int warm, int max_repair_rounds, int pool_blocks,
                                    void* workspace, int64_t workspace_bytes, const b200bt_sweep_config* cfg_host,
                                    b200bt_lane_stats* stats, uint32_t* events, int64_t event_cap,
                                    unsigned char* lane_invalid, int* overflow_host_or_null, b200bt_stream_t stream) {
    (void)order;
    B200BT_REQUIRE(indiv && items && seg_base && n_chunks && workspace && stats && lane_invalid, B200BT_EINVAL,
                   "sweep_chunked: null pointer");
    B200BT_REQUIRE(pop > 0 && n_items > 0 && n_seg > 0 && pool_blocks > 0 && warm >= 0, B200BT_EINVAL, "sweep_chunked: bad sizes");
    int rc = check_sweep_args("sweep_chunked", price, ld_price, rsi, ld_rsi, P, S, N, cfg_host, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE(workspace_bytes >= b200bt_sweep_chunked_workspace_bytes(pool_blocks, S, n_seg), B200BT_EINVAL,
                   "sweep_chunked: workspace too small");
    B200BT_REQUIRE(((uintptr_t)workspace & 15) == 0, B200BT_EINVAL, "sweep_chunked: workspace must be 16-byte aligned");
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    B200BT_REQUIRE(pop <= n_seg, B200BT_EINVAL, "sweep_chunked: fewer segments than individuals");
    const ChunkLayout L = chunk_layout(pool_blocks, (int64_t)S * n_seg, n_seg, pop, false);
    const ChunkWorkspace w = carve(workspace, L, pool_blocks);
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)L.cleared, st);
    if (e != cudaSuccess) return cuda_status(e, "sweep_chunked: memset");

    const ChunkScanArgs A = scan_args(price, ld_price, rsi, ld_rsi, P, S, N, indiv, items, n_items, n_seg, n_chunks, warm, w);
    const bool vec16 = vec16_rows(price, ld_price, rsi, ld_rsi);
    auto kern = vec16 ? chunk_scan_kernel<true> : chunk_scan_kernel<false>;
    if ((rc = allow_sw_smem(kern, "sweep_chunked: cudaFuncSetAttribute"))) return rc;
    const int64_t blocks = (int64_t)((n_items + SW_WARPS - 1) / SW_WARPS) * S;
    B200BT_REQUIRE(blocks < (1ll << 31), B200BT_ELIMIT, "sweep_chunked: too many work items");
    kern<<<(unsigned)blocks, SW_WARPS * 32, SW_SMEM, st>>>(A);
    B200BT_LAUNCH_CHECK("chunk_scan launch");
    return finish_chunks(A, w, vec16, seg_base, pop, max_repair_rounds, cfg_host, stats, events, event_cap, lane_invalid,
                         overflow_host_or_null, st);
}

extern "C" int64_t b200bt_zone_map_floats(int P, int S, int64_t N) {
    if (P <= 0 || S <= 0 || N <= 0) return 0;
    return (int64_t)S * (P + 1) * (zone_row_stride(N) + zone_fine_stride(N)) * 2;
}

extern "C" int b200bt_zone_map(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                               float* zones, b200bt_stream_t stream) {
    B200BT_REQUIRE(price && rsi && zones, B200BT_EINVAL, "zone_map: null pointer");
    B200BT_REQUIRE(P > 0 && S > 0 && N > 0 && ld_price >= N && ld_rsi >= N, B200BT_EINVAL, "zone_map: bad sizes");
    B200BT_REQUIRE(((uintptr_t)zones & 15) == 0, B200BT_EINVAL, "zone_map: output must be 16-byte aligned");
    int rc = check_device();
    if (rc) return rc;
    const int64_t stride = zone_row_stride(N), fstride = zone_fine_stride(N);
    const int64_t blocks = max(stride, fstride / (LS_ZONE / 4));
    const unsigned gx = (unsigned)min((int64_t)1024, (blocks + 7) / 8);
    float2* coarse = (float2*)zones;
    float2* fine = coarse + (int64_t)S * (P + 1) * stride;          // (16-byte aligned: stride is even)
    zone_map_kernel<<<dim3(gx, (unsigned)(S * (P + 1))), 256, 0, (cudaStream_t)stream>>>(price, ld_price, rsi, ld_rsi, P, N, stride, fstride,
                                                                                       coarse, fine);
    B200BT_LAUNCH_CHECK("zone_map launch");
    return B200BT_OK;
}

extern "C" int64_t b200bt_sweep_tiled_workspace_bytes(int pool_blocks, int S, int pop, int K) {
    const int64_t n_seg = (int64_t)pop * K;
    return chunk_layout(pool_blocks, S * n_seg, (int)n_seg, pop, true).bytes;
}

// measurement hook: a pair of caller-owned CUDA events recorded around the scan kernel of the next b200bt_sweep_tiled calls
static cudaEvent_t g_scan_ev[2] = {nullptr, nullptr};
static long long g_wait_cycles = 0;
extern "C" int b200bt_sweep_scan_wait_cycles(int64_t cycles) {
    g_wait_cycles = cycles;
    return B200BT_OK;
}
extern "C" int b200bt_sweep_scan_timing(void* start_event, void* stop_event) {
    g_scan_ev[0] = (cudaEvent_t)start_event;
    g_scan_ev[1] = (cudaEvent_t)stop_event;
    return B200BT_OK;
}

extern "C" int b200bt_sweep_tiled(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S,
                                  int64_t N, const float* zones_or_null, const b200bt_individual* indiv, const int32_t* slots,
                                  int n_slots, const int32_t* order, int pop, int K, int warm, int max_repair_rounds, int pool_blocks, void* workspace,
                                  int64_t workspace_bytes, const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats,
                                  uint32_t* events, int64_t event_cap, unsigned char* lane_invalid, int* overflow_host_or_null,
                                  b200bt_stream_t stream) {
    B200BT_REQUIRE(indiv && workspace && stats && lane_invalid, B200BT_EINVAL, "sweep_tiled: null pointer");
    B200BT_REQUIRE(pop > 0 && K > 0 && K <= 120 && pool_blocks > 0 && warm >= 0, B200BT_EINVAL, "sweep_tiled: bad sizes (1 <= K <= 120)");
    B200BT_REQUIRE(slots ? (n_slots > 0 && n_slots % 32 == 0) : true, B200BT_EINVAL, "sweep_tiled: n_slots must be a positive multiple of 32");
    if (!slots) n_slots = (pop + 31) & ~31;
    int rc = check_sweep_args("sweep_tiled", price, ld_price, rsi, ld_rsi, P, S, N, cfg_host, events, event_cap);
    if (rc) return rc;
    B200BT_REQUIRE((int64_t)pop * K * S < (1ll << 31), B200BT_ELIMIT, "sweep_tiled: too many chunks");
    B200BT_REQUIRE(K == 1 || N / K >= SW_GROUP, B200BT_EINVAL, "sweep_tiled: chunks shorter than %d bars", SW_GROUP);
    // shared-memory rings: one per warp, LS_STAGES tiles of LS_ROWS rows (+ their zone ranges): independent of P
    const size_t smem = (size_t)LS_WARPS * LS_STAGES * LS_ROWS * (LS_STRIDE * sizeof(float) + (zones_or_null ? (LS_T / LS_ZONE + LS_T / 4) * sizeof(float2) : 0));
    B200BT_REQUIRE(zones_or_null == nullptr || ((uintptr_t)zones_or_null & 15) == 0, B200BT_EINVAL, "sweep_tiled: zone map must be 16-byte aligned");
    B200BT_REQUIRE(workspace_bytes >= b200bt_sweep_tiled_workspace_bytes(pool_blocks, S, pop, K), B200BT_EINVAL,
                   "sweep_tiled: workspace too small");
    B200BT_REQUIRE(((uintptr_t)workspace & 15) == 0, B200BT_EINVAL, "sweep_tiled: workspace must be 16-byte aligned");
    rc = check_device();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int n_seg = pop * K;
    const ChunkLayout lay = chunk_layout(pool_blocks, (int64_t)S * n_seg, n_seg, pop, true);
    const ChunkWorkspace w = carve(workspace, lay, pool_blocks);
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)lay.cleared, st);
    if (e != cudaSuccess) return cuda_status(e, "sweep_tiled: memset");
    lane_tables_kernel<<<(n_seg + 255) / 256, 256, 0, st>>>(pop, K, order, w.items, w.seg_base, w.n_chunks);
    B200BT_LAUNCH_CHECK("lane_tables launch");

    LaneScanArgs L;
    static_cast<ChunkTables&>(L) = w;
    L.price = price; L.ld_price = ld_price; L.rsi = rsi; L.ld_rsi = ld_rsi; L.P = P; L.S = S; L.N = N;
    L.zones = (const float2*)zones_or_null; L.n_zone_blocks = zone_row_stride(N);    // (row stride of the zone map)
    L.fine = zones_or_null ? L.zones + (int64_t)S * (P + 1) * zone_row_stride(N) : nullptr; L.n_fine = zone_fine_stride(N);
    L.indiv = indiv; L.slots = slots; L.n_slots = n_slots; L.pop = pop; L.K = K; L.warm = warm;
    L.work = &w.ctr->scan_work; L.ctr = w.ctr;
    const bool vec16 = vec16_rows(price, ld_price, rsi, ld_rsi);
    const bool dense = (double)pool_blocks * CK_BLOCK >= LS_DENSE_EVENTS * (double)pop * S * (double)N;
    auto kern = zones_or_null ? (dense ? lane_scan_kernel<true, LS_UNROLL_DENSE> : lane_scan_kernel<true, LS_UNROLL_SPARSE>)
                              : (dense ? lane_scan_kernel<false, LS_UNROLL_DENSE> : lane_scan_kernel<false, LS_UNROLL_SPARSE>);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return cuda_status(e, "sweep_tiled: cudaFuncSetAttribute");
    const int64_t n_items = (int64_t)(n_slots / 32) * K * S;
    B200BT_REQUIRE(n_items < (1ll << 30), B200BT_ELIMIT, "sweep_tiled: too many work items");
    L.wait_cycles = g_wait_cycles != 0 ? g_wait_cycles : LS_WAIT_CYCLES;
    // persistent grid: one resident set of CTAs (warps take work items from the counter), no more CTAs than items need
    int dev = 0, sms = 0, per_sm = 0;
    e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, LS_THREADS, smem);
    if (e != cudaSuccess) return cuda_status(e, "sweep_tiled: occupancy");
    int64_t blocks = (int64_t)sms * (per_sm > 0 ? per_sm : 1);
    if (blocks > (n_items + LS_WARPS - 1) / LS_WARPS) blocks = (n_items + LS_WARPS - 1) / LS_WARPS;
    if (g_scan_ev[0]) cudaEventRecord(g_scan_ev[0], st);
    kern<<<(unsigned)blocks, LS_THREADS, smem, st>>>(L, vec16);
    if (g_scan_ev[1]) cudaEventRecord(g_scan_ev[1], st);
    B200BT_LAUNCH_CHECK("lane_scan launch");

    const ChunkScanArgs A = scan_args(price, ld_price, rsi, ld_rsi, P, S, N, indiv, w.items, n_seg, n_seg, w.n_chunks, warm, w);
    return finish_chunks(A, w, vec16, w.seg_base, pop, max_repair_rounds, cfg_host, stats, events, event_cap, lane_invalid,
                         overflow_host_or_null, st);
}
