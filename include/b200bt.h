/*
 * b200bt.h -- C-ABI of the H100-native backtest / evolution / Monte-Carlo engine.
 *
 * This is the drop-in boundary below the reference's Python call surface
 * (zd87pl/ai-crypto-trader; SURVEY.md section 8b).  The reference has no FFI
 * of its own -- every function on the path is plain Python -- so each entry
 * point below cites the reference function (file:line, relative to the
 * reference tree) whose arithmetic it replaces.  All pointers are DEVICE
 * pointers unless a name ends in `_host`.  No torch types cross this
 * boundary: sizes are plain integers, `stream` is a `cudaStream_t` passed as
 * `void*`.  Every function returns 0 on success and a non-zero status on
 * failure (a `cudaError_t` value, or one of the B200BT_E* codes); nothing
 * throws across the boundary.  `b200bt_last_error()` returns a thread-local,
 * human-readable description of the last failure.
 *
 * There is NO CPU fallback behind this ABI.  If no sm_90 device is present
 * the compute entry points return B200BT_ENODEVICE.
 */
#ifndef B200BT_H_
#define B200BT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200BT_ABI_VERSION 1

#define B200BT_OK 0
#define B200BT_EINVAL 10001   /* bad argument (null pointer, size <= 0, ...)   */
#define B200BT_ENODEVICE 10002 /* no CUDA device / wrong architecture          */
#define B200BT_ELIMIT 10003   /* argument exceeds a documented limit           */

typedef void* b200bt_stream_t; /* cudaStream_t */

int b200bt_abi_version(void);
const char* b200bt_last_error(void);
/* Number of kernels launched by this library in this process (all threads);
 * bench.py reports the delta over the timed region as `gpu_launches`. */
int64_t b200bt_launch_count(void);

/* ------------------------------------------------------------------------
 * Family 1: rolling indicators over fp32 OHLCV.
 * Series layout: row-major [S][N] fp32, one row per symbol ("SoA per field").
 * Bank layout:   row-major [S][P][N] fp32, one row per (symbol, period).
 * Arithmetic is fp64 internally (so that a float64 CPU evaluation of the same
 * recurrence rounds to the same fp32 value), outputs are fp32.
 * NaN policy follows TechnicalAnalyzer._handle_nan_values
 * (binance_ml_strategy.py:28-38): leading undefined values are back-filled
 * with the first defined value (`fill=1`) or written as NaN (`fill=0`).
 * Limits (B200BT_ELIMIT outside): windows in [1, 1024] and 1..64 windows per bank call,
 * MACD spans in [1, 512]; the RSI and ATR banks state their own below.
 * ------------------------------------------------------------------------ */

/* RSI bank.  Replaces ta.momentum.RSIIndicator(close, window=w).rsi() as called
 * at binance_ml_strategy.py:112 (and services/market_monitor_service.py:228),
 * for every window in periods_host[0..P).  Wilder smoothing
 * ewm(alpha=1/w, adjust=False) of up/down moves; rsi = 100 where the smoothed
 * down move is 0.  1 <= P <= 128 (P = 0: B200BT_EINVAL, above: B200BT_ELIMIT), every window in
 * [1, 4096] (B200BT_ELIMIT outside). */
int b200bt_rsi_bank(const float* close, int S, int64_t N, int64_t ld,
                    const int* periods_host, int P, int fill,
                    float* out, b200bt_stream_t stream);

/* TechnicalAnalyzer._calculate_all_indicators + _handle_nan_values (binance_ml_strategy.py:28-182) for S symbols in three
 * fused launches (close -> EMA / MACD / RSI; close -> SMA / Bollinger; high, low, close, volume -> stochastic / Williams %R /
 * Ichimoku / ATR / VWAP) plus one batched NaN-policy call, with the reference's windows (20/50/200, 12/26/9, 9/26/52, 14, 14/3,
 * 14, 20 x 2.0, 14, 14).  cols: [B200BT_ANALYZER_COLUMNS][S][N] fp32 (device, out), column c at cols + c * S * N in the order
 * below; workspace: b200bt_analyzer_workspace_floats(S, N) floats (device). */
enum b200bt_analyzer_column {
    B200BT_COL_SMA_20 = 0, B200BT_COL_SMA_50, B200BT_COL_SMA_200, B200BT_COL_EMA_12, B200BT_COL_EMA_26, B200BT_COL_MACD,
    B200BT_COL_MACD_SIGNAL, B200BT_COL_MACD_DIFF, B200BT_COL_ICHIMOKU_A, B200BT_COL_ICHIMOKU_B, B200BT_COL_RSI, B200BT_COL_BB_HIGH,
    B200BT_COL_BB_MID, B200BT_COL_BB_LOW, B200BT_COL_BB_WIDTH, B200BT_COL_ATR,
    /* columns that can be undefined in mid-series (zero volume / zero range): general ffill-bfill pass */
    B200BT_COL_VWAP, B200BT_COL_STOCH_K, B200BT_COL_STOCH_D, B200BT_COL_WILLIAMS_R, B200BT_COL_BB_POSITION,
    B200BT_ANALYZER_COLUMNS
};
int64_t b200bt_analyzer_workspace_floats(int S, int64_t N);
int b200bt_analyzer(const float* high, const float* low, const float* close, const float* volume, int S, int64_t N, int64_t ld,
                    float* cols, float* workspace, b200bt_stream_t stream);

/* b200bt_rsi_bank (NaN policy applied) that also writes the bank's rows of a sweep zone map (see b200bt_zone_map: row 0 =
 * the close prices, rows 1..P = the RSI rows) while the values are in registers, so that the first sweep of a fresh bank can
 * already skip quiet blocks.  `zones` is the WHOLE zone map of S_total symbols (b200bt_zone_map_floats(P, S_total, N) floats);
 * this call fills the rows of symbols [sym0, sym0 + S), whose closes / bank rows `close` / `out` point at. */
int b200bt_rsi_bank_zones(const float* close, int S, int64_t N, int64_t ld, const int* periods_host, int P,
                          float* out, float* zones, int S_total, int sym0, b200bt_stream_t stream);

/* EMA bank: ta.trend.EMAIndicator(close, window=w) = ewm(span=w, min_periods=w, adjust=False)
 * (binance_ml_strategy.py:79-83).  out [S][P][N]; undefined leading values are NaN. */
int b200bt_ema_bank(const float* x, int S, int64_t N, int64_t ld, const int* spans_host, int P,
                    float* out, b200bt_stream_t stream);

/* SMA bank: ta.trend.SMAIndicator = rolling(w, min_periods=w).mean() (:67-76). out [S][P][N]. */
int b200bt_sma_bank(const float* x, int S, int64_t N, int64_t ld, const int* windows_host, int P,
                    float* out, b200bt_stream_t stream);

/* MACD: ta.trend.MACD(close, slow, fast, sign) (:91-94).  line/signal/diff each [S][N]. */
int b200bt_macd(const float* x, int S, int64_t N, int64_t ld, int fast, int slow, int sign,
                float* line, float* signal, float* diff, b200bt_stream_t stream);

/* Bollinger bands: ta.volatility.BollingerBands(close, window, k) plus the analyzer's
 * bb_width and bb_position (zero range -> NaN) (:148-156).  Five outputs, each [S][N]. */
int b200bt_bollinger(const float* x, int S, int64_t N, int64_t ld, int window, double k,
                     float* high, float* mid, float* low, float* width, float* position,
                     b200bt_stream_t stream);

/* Stochastic oscillator %K / %D: ta.momentum.StochasticOscillator(high, low, close, window,
 * smooth_window) (:121-127). */
int b200bt_stochastic(const float* high, const float* low, const float* close, int S, int64_t N,
                      int64_t ld, int window, int smooth, float* k, float* d, b200bt_stream_t stream);

/* Williams %R: ta.momentum.WilliamsRIndicator(high, low, close, lbp) (:135-140). */
int b200bt_williams_r(const float* high, const float* low, const float* close, int S, int64_t N,
                      int64_t ld, int lbp, float* out, b200bt_stream_t stream);

/* Ichimoku a / b: ta.trend.IchimokuIndicator(high, low, w1, w2, w3, visual=False) (:102-104). */
int b200bt_ichimoku(const float* high, const float* low, int S, int64_t N, int64_t ld, int w1, int w2,
                    int w3, float* a, float* b, b200bt_stream_t stream);

/* ATR bank: ta.volatility.AverageTrueRange(high, low, close, window=w) (:164); zeros before
 * bar w-1 (ta writes 0, not NaN).  out [S][P][N].  1 <= P <= 64 and every window in [1, 541]
 * (B200BT_ELIMIT otherwise: the warm-up halo of the longest window is staged in shared memory). */
int b200bt_atr_bank(const float* high, const float* low, const float* close, int S, int64_t N,
                    int64_t ld, const int* windows_host, int P, float* out, b200bt_stream_t stream);

/* VWAP: ta.volume.VolumeWeightedAveragePrice(high, low, close, volume, window) (:173-179). */
int b200bt_vwap(const float* high, const float* low, const float* close, const float* volume, int S,
                int64_t N, int64_t ld, int window, float* out, b200bt_stream_t stream);

/* Multi-timeframe (BASELINE configs[3]; recipe: services/market_monitor_service.py:219-301, where
 * each timeframe is its own kline series, :168-171).  b200bt_resample derives clock-aligned k-minute
 * OHLCV [5][S][M] from 1-minute (or bar_minutes) OHLCV [5][S][N]; M = b200bt_resample_bars(...).
 * b200bt_align maps a higher-timeframe series [S][M] back onto the base clock [S][N] using the last
 * COMPLETED higher-timeframe bar (NaN before the first one).  Buckets are aligned to the Unix epoch (pandas'
 * origin="epoch").  minute0 < 0 is refused: EINVAL from both, and b200bt_resample_bars returns 0. */
int64_t b200bt_resample_bars(int64_t N, int64_t minute0, int bar_minutes, int k);
int b200bt_resample(const float* ohlcv, int S, int64_t N, int64_t minute0, int bar_minutes, int k,
                    float* out, int64_t M, b200bt_stream_t stream);
int b200bt_align(const float* src, int S, int64_t M, int64_t N, int64_t minute0, int bar_minutes, int k,
                 float* out, b200bt_stream_t stream);

/* TechnicalAnalyzer._handle_nan_values (:28-38) on `rows` contiguous rows of length N, in place:
 * forward-fill, then back-fill, then 0.  workspace: b200bt_nanfill_workspace_floats(rows, N) floats. */
int64_t b200bt_nanfill_workspace_floats(int64_t rows, int64_t N);
int b200bt_nanfill(float* x, int64_t rows, int64_t N, float* workspace, b200bt_stream_t stream);

/* ------------------------------------------------------------------------
 * Family 2: the per-bar entry/exit/stop/PnL state machine over
 * (GA-individual x symbol) lanes.
 * Replaces, for a whole population at once:
 *   StrategyEvaluationSystem._simulate_trades   services/strategy_evaluation.py:746-878
 *   StrategyPerformanceMetrics.calculate_metrics services/strategy_evaluation.py:32-228
 *   StrategyEvaluationSystem._calculate_strategy_score              :579-633
 * which GeneticAlgorithm.evaluate_population (services/genetic_algorithm.py:119-133)
 * calls once per individual.
 * ------------------------------------------------------------------------ */

/* One GA individual, already decoded by the host:
 *  rsi_row       row of the RSI bank holding this individual's rsi_period
 *  rsi_lo        `rsi < rsi_oversold`  is evaluated as  r < rsi_lo  (fp32)
 *  rsi_hi        `rsi > rsi_overbought` is evaluated as r > rsi_hi  (fp32)
 *                (host rounds the float64 thresholds up/down to fp32 so the
 *                 fp32 compare decides exactly like the float64 one)
 *  take_profit   take_profit/100  (float64, strategy_evaluation.py:773)
 *  stop_loss     stop_loss/100    (float64, :774)
 *  position_size dollars, 10000*min(max_position_size,20)/100 (:762-764)
 */
typedef struct b200bt_individual {
    int32_t rsi_row;
    float rsi_lo;
    float rsi_hi;
    int32_t reserved;
    double take_profit;
    double stop_loss;
    double position_size;
} b200bt_individual; /* 40 bytes */

/* Per-lane result, 20 x 8 bytes.  Field meaning follows calculate_metrics
 * (strategy_evaluation.py:187-225) on the lane's trade RECORDS (an entry and
 * an exit record per round trip, as the reference emits them). */
typedef struct b200bt_lane_stats {
    double n_records;      /* total_trades                                   */
    double n_wins;         /* #records with pnl > 0                          */
    double n_losses;       /* #records with pnl < 0                          */
    double total_profit;   /* sum of positive pnl                            */
    double total_loss;     /* sum of negative pnl (<= 0)                     */
    double net_profit;     /* total_profit + total_loss                      */
    double max_drawdown;   /* fraction of peak equity                        */
    double sharpe_ratio;   /* daily-bucket Sharpe, sqrt(252) annualised      */
    double n_days;         /* distinct calendar days holding a record        */
    double largest_profit;
    double largest_loss;
    double sum_duration_bars; /* sum over round trips of exit_bar-entry_bar  */
    double score;          /* _calculate_strategy_score                      */
    double win_rate;
    double profit_factor;  /* +inf when total_loss == 0 (reference :113)     */
    /* ingredients of calculate_advanced_metrics (strategy_evaluation.py:231-319) that need the daily buckets */
    double sortino_ratio;  /* mean(daily) / std(negative dailies, ddof 0) * sqrt(252); +inf without a negative
                              spread, 0 without daily buckets (:250-263)      */
    double n_negative_days;
    double downside_deviation; /* np.std of the negative daily sums           */
    double mean_daily_pnl; /* profit_per_day (:307-312)                       */
    uint64_t trade_hash;   /* xor of event_hash(event_index, event word) over all events */
} b200bt_lane_stats; /* 160 bytes */

/* Scoring rule (config.json evolution.optimization_goals; SURVEY 8-a15). */
#define B200BT_PRIMARY_SHARPE 0
#define B200BT_PRIMARY_RETURN_PCT 1
#define B200BT_PRIMARY_PROFIT_FACTOR 2
#define B200BT_PRIMARY_WIN_RATE 3
#define B200BT_PRIMARY_NET_PROFIT 4
/* any other scalar key of the metrics dict may be the primary metric (`metrics.get(primary, 0)`, :589-590) */
#define B200BT_PRIMARY_TOTAL_TRADES 5
#define B200BT_PRIMARY_MAX_DRAWDOWN 6
#define B200BT_PRIMARY_TOTAL_PROFIT 7
#define B200BT_PRIMARY_TOTAL_LOSS 8
#define B200BT_PRIMARY_LARGEST_PROFIT 9
#define B200BT_PRIMARY_LARGEST_LOSS 10
#define B200BT_PRIMARY_AVERAGE_PROFIT 11
#define B200BT_PRIMARY_AVERAGE_LOSS 12
/* keys only calculate_advanced_metrics adds (:231-319): present when the score is taken on the advanced dict
 * (evaluate_strategy :545-557); on the plain dict (cross_validate_strategy :683-691) the host passes ZERO for them */
#define B200BT_PRIMARY_SORTINO 13
#define B200BT_PRIMARY_EXPECTANCY 14
#define B200BT_PRIMARY_CALMAR 15
#define B200BT_PRIMARY_PROFIT_PER_DAY 16
#define B200BT_PRIMARY_RECOVERY_FACTOR 17
#define B200BT_PRIMARY_ZERO 99           /* a key the metrics dict does not hold: metrics.get(key, 0) */
#define B200BT_SEC_MAX_DRAWDOWN 1
#define B200BT_SEC_WIN_RATE 2
#define B200BT_SEC_PROFIT_FACTOR 4
#define B200BT_SEC_EXPECTANCY 8          /* score *= 1 + min(expectancy / 100, 1) (:615-620); set by the host only when
                                            the score is taken on the advanced dict (else the key is absent: factor 1) */

typedef struct b200bt_sweep_config {
    double initial_capital;  /* 10000.0 (strategy_evaluation.py:33,761)       */
    int64_t minute0;         /* minutes since 1970-01-01T00:00Z of bar 0      */
    int32_t bar_minutes;     /* bar spacing; day = (minute0+t*bar_minutes)/1440 */
    int32_t primary;         /* B200BT_PRIMARY_*                              */
    int32_t secondary_mask;  /* B200BT_SEC_* bits                             */
    int32_t variant;         /* kernel variant selector, 0 = default          */
    int32_t gap_bar;         /* > 0: the series is two pieces glued at this bar (training folds of            */
    int32_t gap_minutes;     /*      cross_validate_strategy :674-682): bars >= gap_bar lie gap_minutes later  */
} b200bt_sweep_config;   /* 40 bytes */

/* Event word written to the optional trade buffer: bits 0..29 bar index,
 * bit 30 = 1 for an exit record, bit 31 = 1 for side "sell"
 * (short entry / long exit).  */
#define B200BT_EVENT_EXIT 0x40000000u
#define B200BT_EVENT_SELL 0x80000000u
#define B200BT_EVENT_BAR_MASK 0x3fffffffu

/* Run the population sweep.
 *  price   [S][N] fp32 (row stride ld_price)       close prices
 *  rsi     [S][P][N] fp32 (row stride ld_rsi)      RSI bank
 *  indiv   [pop] individuals (device)
 *  order   [pop] int32 (device) evaluation order of individuals (a permutation;
 *          the host sorts by rsi_row so neighbouring warps share a stream);
 *          may be NULL for identity
 *  stats   [pop][S] lane stats (device, out)
 *  events  optional [pop][S][event_cap] uint32 (device, out), first event_cap
 *          event words per lane; NULL to skip
 * Limits: N < 2^30 (else B200BT_ELIMIT); bar_minutes > 0, minute0 >= 0 and gap_minutes >= 0 (else B200BT_EINVAL);
 * minute0 + N*bar_minutes + gap_minutes < 2^32 - 1440 (else B200BT_ELIMIT).  The time-chunked forms below check the same.
 */
int b200bt_sweep(const float* price, int64_t ld_price,
                 const float* rsi, int64_t ld_rsi, int P,
                 int S, int64_t N,
                 const b200bt_individual* indiv, const int32_t* order, int pop,
                 const b200bt_sweep_config* cfg_host,
                 b200bt_lane_stats* stats,
                 uint32_t* events, int64_t event_cap,
                 b200bt_stream_t stream);

/* Time-chunked form of b200bt_sweep (same results; csrc/sweep_chunked.cu).  Expensive lanes are split
 * into n_chunks time chunks scanned concurrently, each started `warm` bars early from the flat state;
 * the chunk-boundary states are verified lane by lane and a chunk whose assumed state was wrong is re-scanned from the
 * true state until its trajectory meets the recorded one again (the rest of the recorded events is then kept).
 * max_repair_rounds: 0 = no repair, 1 = one chunk-parallel pass (every wrong chunk re-scanned once, trusting its
 * predecessor's recorded end state), >= 2 = that pass plus a lane-sequential one beside the metrics kernels that finishes
 * the lanes whose re-scans run through chunk after chunk; nothing is read back.
 * A lane that still has a mismatch (or lost events to a full pool) is flagged in lane_invalid[pop][S] and re-evaluated
 * exactly inside this call (see below).  One work item per (individual, chunk); `segment` = seg_base[individual] + chunk.
 *  order      unused (kept for the ABI), may be NULL
 *  items      [n_items] device      seg_base, n_chunks  [pop] device int32      n_seg = sum of n_chunks
 *  pool_blocks  event pool size in blocks of 256 events; a chunk that cannot get a block flags its lane
 *  workspace  b200bt_sweep_chunked_workspace_bytes(pool_blocks, S, n_seg) device bytes
 *  overflow_host_or_null  optional PINNED host int[5], written asynchronously on `stream` (read after synchronising it):
 *                         [0] = 1 if the event pool ran out (grow it next time), [1] = number of (individual, symbol)
 *                         lanes that were flagged and re-evaluated by the exact fallback, [2] = pool blocks handed out
 *                         (what the next sweep of a similar population needs), [3] = tiles of the thread-per-lane scan
 *                         whose bulk copy did not complete in time (b200bt_sweep_tiled; their work was redone, see there),
 *                         [4] = time chunks that set a new equity peak (their drawdown took the record-by-record pass).
 * Flagged lanes are re-evaluated by the fused kernel (b200bt_sweep's) inside this call, from a device-side list: the call
 * reads nothing back and never synchronises; lane_invalid reports which lanes took that path. */
typedef struct b200bt_chunk_item {
    int32_t individual;
    int32_t chunk;
    int32_t n_chunks;
    int32_t segment;
} b200bt_chunk_item;

int64_t b200bt_sweep_chunked_workspace_bytes(int pool_blocks, int S, int n_seg);
int b200bt_sweep_chunked(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P,
                         int S, int64_t N, const b200bt_individual* indiv, const int32_t* order, int pop,
                         const b200bt_chunk_item* items, int n_items, const int32_t* seg_base,
                         const int32_t* n_chunks, int n_seg, int warm, int max_repair_rounds, int pool_blocks,
                         void* workspace, int64_t workspace_bytes, const b200bt_sweep_config* cfg_host,
                         b200bt_lane_stats* stats, uint32_t* events, int64_t event_cap,
                         unsigned char* lane_invalid, int* overflow_host_or_null, b200bt_stream_t stream);

/* Same contract as b200bt_sweep_chunked, thread-per-lane form: EVERY individual is cut into the same K time
 * chunks (chunk c of K covers [floor(N c / K) & ~511, ...)) and each THREAD steps the state machine of one (individual,
 * symbol, chunk) through shared-memory tiles.  Every warp stages its own tiles -- the price row and the RSI rows its 32
 * machines read -- through a private ring of bulk async copies (cp.async.bulk + mbarrier), so warps never wait for each other.
 * Verification, in-place repair, metrics and the lane_invalid / overflow outputs are those of b200bt_sweep_chunked.
 * slots: device int32[n_slots] (n_slots a multiple of 32): individual run by each thread slot, -1 = empty; 32 consecutive
 *        slots form a warp, which may read at most TWO distinct RSI rows (rsi_row) -- the host packs individuals by row and
 *        similar cost; a warp that breaks the rule is not scanned: its lanes are flagged in lane_invalid and re-evaluated
 *        by the fused kernel inside this call (exact).  NULL = identity (thread k runs individual k).
 * order: device int32[pop], the individuals in dispatch order (by predicted cost), NULL = identity: the order in which the
 *        per-chunk metrics kernels list their work (one thread per chunk: neighbours should hold similar record counts).
 * zones: optional zone map of the same price / RSI arrays (b200bt_zone_map), NULL = none: (min, max) per 32-bar
 *        block of every row, which lets a warp skip blocks in which none of its machines' thresholds can be crossed.
 * Shared memory does not depend on P (any number of RSI rows). */
int64_t b200bt_zone_map_floats(int P, int S, int64_t N);     /* floats in the zone map: coarse (32-bar) ranges [S][P+1][ceil(N/32) rounded up to even][2], then fine (4-bar) ranges [S][P+1][ceil(N/128)*32][2]; 16-byte aligned */
int b200bt_zone_map(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                    float* zones, b200bt_stream_t stream);
int64_t b200bt_sweep_tiled_workspace_bytes(int pool_blocks, int S, int pop, int K);
int b200bt_sweep_tiled(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S,
                       int64_t N, const float* zones, const b200bt_individual* indiv, const int32_t* slots, int n_slots,
                       const int32_t* order, int pop, int K, int warm, int max_repair_rounds, int pool_blocks, void* workspace, int64_t workspace_bytes,
                       const b200bt_sweep_config* cfg, b200bt_lane_stats* stats, uint32_t* events,
                       int64_t event_cap, unsigned char* lane_invalid, int* overflow_host_or_null,
                       b200bt_stream_t stream);

/* Measurement hook (bench.py's roofline): a pair of caller-owned cudaEvent_t that the following b200bt_sweep_tiled calls of
 * this process record on their stream immediately before and after the scan kernel (lane_scan_kernel); NULL, NULL switches
 * it off.  The caller reads cudaEventElapsedTime after synchronising.  Not thread-safe (one measuring thread). */
int b200bt_sweep_scan_timing(void* start_event, void* stop_event);
/* Bound of one tile wait of the scan kernel in SM clocks (0 = the default, ~20 ms).  A tile whose bulk copy does not complete
 * within the bound is not waited for any longer: the work item is marked as lost (its chunks are re-scanned by the repair pass
 * or its lanes re-run by the exact fallback), the warp stops using its tile ring, and overflow_host[3] counts the event.  Results
 * do not depend on it.  A negative value -k is the test hook: every warp gives up at the k-th tile of an item as if it had
 * not arrived. */
int b200bt_sweep_scan_wait_cycles(int64_t cycles);

/* fitness[i] = mean over symbols of stats[i][s].score  (float64, device). */
int b200bt_fitness_reduce(const b200bt_lane_stats* stats, int pop, int S,
                          double* fitness, b200bt_stream_t stream);

/* Book metrics: the score of ONE account trading every symbol.  StrategyEvaluationSystem.evaluate_strategy
 * (services/strategy_evaluation.py:528-577) passes one trade list to calculate_metrics (:32-228), which sorts it by timestamp
 * (:67) and walks one equity curve, one drawdown and one set of daily buckets over all of it (:118-188).  The book of
 * individual i is the concatenation, in symbol order 0..S-1, of its records on every symbol (_simulate_trades :746-878),
 * sorted stably by timestamp: the order (bar, symbol, record index within the lane).  book_stats[i] holds calculate_metrics'
 * scalars on that list, with the lane rules of b200bt_lane_stats: Sharpe / Sortino over the calendar days of the whole
 * book, n_records < 2 gives the short dict of :43-92; and _calculate_strategy_score (:579-633) under cfg's score rule, with
 * two book-specific fields:
 *   sum_duration_bars  sum over the merged pairs (2k, 2k+1) of bar(2k+1) - bar(2k): avg_trade_duration pairs neighbouring
 *                      records of the merged list (:166-178) even when they belong to different symbols (a quirk of the
 *                      reference, kept for parity)
 *   trade_hash         xor over merged records r (index r in the book) of event_hash(r, word_r ^ (symbol_r * 0x9E3779B1));
 *                      with S = 1 it is the lane's trade_hash
 * Records are priced as b200bt_trade_pnl prices them.  Inputs are a sweep's: lane_stats [pop][S] (n_records), events
 * [pop][S][event_cap] and price [S][ld_price] (device), indiv [pop] (device), cfg (host; its clock is checked like the
 * sweeps').  A book with a lane of n_records > event_cap lost records: it gets n_records = -1, score and fitness NaN, and
 * must be computed again from a sweep with a larger event_cap.  fitness_or_null: optional device float64 [pop] = score.
 * Limits: S <= 64 (B200BT_ELIMIT above: one 64-bit symbol mask per bar), N < 2^30, S * (N + 1) < 2^32.  No synchronisation. */
int b200bt_book_metrics(const float* price, int64_t ld_price, int S, int64_t N,
                        const b200bt_individual* indiv, int pop, const b200bt_sweep_config* cfg,
                        const b200bt_lane_stats* lane_stats, const uint32_t* events, int64_t event_cap,
                        b200bt_lane_stats* book_stats, double* fitness_or_null, b200bt_stream_t stream);

/* ------------------------------------------------------------------------
 * The reference's own single-symbol bar loop (BASELINE configs[0]):
 *   StrategyTester.backtest_strategy   backtesting/strategy_tester.py:156-312
 *   open_position / close_position     :314-369
 *   PositionSizer.calculate_position_size  binance_ml_strategy.py:251-291
 * One warp per symbol; the entry gate (technical signal x AI decision, constant per
 * symbol in the reference, SURVEY 8-a6) is decided on the host and passed as can_enter.
 * ------------------------------------------------------------------------ */
typedef struct b200bt_bt_params {
    double initial_balance;
    double position_pct;       /* 0.25 / 0.20 / 0.15 by volatility class (:256-264)      */
    double stop_loss_pct;      /* 0.02 / 0.015 / 0.01 -- a FRACTION compared with a PERCENT
                                  pnl (strategy_tester.py:206-215), quirk kept            */
    double take_profit_pct;    /* 2 x stop_loss_pct (:287)                                */
    double volume_factor;      /* min(avg_volume/50000, 1) (:267)                         */
    double max_risk_per_trade; /* 0.15                                                    */
    int32_t can_enter;         /* technical BUY x strength>=70 x AI gate (:371-401)       */
    int32_t skip;              /* 10 (:192)                                               */
} b200bt_bt_params; /* 56 bytes */

/* stats  [S][16] float64: final_balance, total_trades, winning, losing, total_profit,
 *                         total_loss(positive), max_drawdown, max_drawdown_pct, n_equity_points, open_at_end
 * trades [S][trade_cap][8] float64: entry_bar, exit_bar, reason(1 SL,2 TP,3 end), entry_price,
 *                         quantity, position_size, pnl, pnl_pct
 * equity [S][equity_cap][2] float64: bar, cash balance at that (flat or entry) bar */
int b200bt_backtest_ref(const float* price, int64_t ld, int S, int64_t N,
                        const b200bt_bt_params* params, double* stats, double* trades,
                        int64_t trade_cap, double* equity, int64_t equity_cap,
                        b200bt_stream_t stream);

/* ------------------------------------------------------------------------
 * Family 3: Monte-Carlo risk projection.
 * Replaces the path generation and per-path loops of
 *   MonteCarloService.run_monte_carlo_simulation  services/monte_carlo_service.py:197-394
 * Randomness: Philox4x32-10, counter = (path index lo, hi, step/4, mode),
 * key = seed; normals by Box-Muller on 24-bit uniforms.  A path's values depend
 * only on (seed, path_offset + local index, step), never on sharding.
 * Outputs: finals[n] = S_T, maxdd[n] = max_t (runmax_t - S_t)/runmax_t (:327-336),
 * optional paths[(steps+1)][n] fp32 (the reference's `paths` array, shape (days, n)).
 * ------------------------------------------------------------------------ */

/* Geometric Brownian motion (:266-273): `steps` = days-1 multiplicative steps of
 * exp((mu - sigma^2/2) dt + sigma sqrt(dt) Z). */
int b200bt_mc_gbm(double s0, double mu, double sigma, double dt, int64_t n_paths, int steps,
                  uint64_t seed, uint64_t path_offset, float* finals, float* maxdd,
                  float* paths_or_null, b200bt_stream_t stream);

/* 'historical' simulation (:277-298): bootstrap of the return sample with
 * replacement.  block_len = 1 reproduces the reference (iid); block_len > 1 is a
 * circular block bootstrap.  log_returns != 0: P_t = P_{t-1} exp(r); else
 * P_t = P_{t-1} (1 + r).  `returns` is a device array of R <= 12288 fp32 values (B200BT_ELIMIT above). */
int b200bt_mc_bootstrap(const float* returns, int R, int block_len, int log_returns, double s0,
                        int64_t n_paths, int steps, uint64_t seed, uint64_t path_offset,
                        float* finals, float* maxdd, float* paths_or_null, b200bt_stream_t stream);

/* Exact order statistics: out[r] = ranks[r]-th smallest (0-based) of x[0..n).
 * ranks_dev: device int64[n_ranks] in any order, repeats allowed, 1 <= n_ranks <= 64.  Two-level radix
 * select; workspace of b200bt_select_workspace_bytes(n_ranks) device bytes.
 * Feeds np.percentile's linear interpolation (:308-317) on the host side. */
int64_t b200bt_select_workspace_bytes(int n_ranks);
int b200bt_select(const float* x, int64_t n, const int64_t* ranks_dev, int n_ranks, float* out,
                  void* workspace, int64_t workspace_bytes, b200bt_stream_t stream);

/* Moments of the final prices (:305-336).  out7 (device, float64):
 *  [0] sum S_T  [1] sum pct  [2] #(S_T > s0)  [3] sum maxdd  [4] max maxdd
 *  [5] sum pct[pct <= var_threshold]  [6] #(pct <= var_threshold)
 * with pct = (S_T/s0 - 1)*100 in float64; maxdd may be NULL. */
int b200bt_mc_moments(const float* finals, const float* maxdd, int64_t n, double s0,
                      double var_threshold, double* out7, b200bt_stream_t stream);

/* Joint paths of a portfolio of 1 <= S <= 32 assets (B200BT_ELIMIT above), simulated together instead of one
 * asset at a time.  Replaces the per-asset loop of MonteCarloService.run_portfolio_monte_carlo
 * (services/monte_carlo_service.py:492-575) and the correlation-free sums of _calculate_portfolio_stats (:577-659,
 * "Simplified approach - ignores correlations", :630-631).  Portfolio value V_t = sum_i qty_i s0_i exp(logS_i,t)
 * (qty_i >= 0, V_0 > 0).  Outputs: finals[n] = V_T, maxdd[n] = max_t (runmax_t - V_t)/runmax_t (the :327-336 rule
 * on V_t), optional asset_finals[S][n] = s0_i exp(logS_i,T); finals / maxdd feed b200bt_select and b200bt_mc_moments
 * with s0 = V_0.  Randomness: counter = (path index lo, hi, step/4, (factor << 8) | mode), key = seed.
 *
 * GBM (:266-273 per asset): every step draws S standard normals z; asset i moves by drift_i + vol_i (L z)_i with the
 * per-step drift_i = (mu_i - sigma_i^2/2) dt and vol_i = sigma_i sqrt(dt).  chol_host: [S][S] row-major, the
 * lower-triangular Cholesky factor L of the correlation matrix (the upper triangle is not read).  Factor 0 draws
 * b200bt_mc_gbm's stream: with L_00 = 1, asset 0 equals b200bt_mc_gbm's path for the same (seed, path, s0, drift, vol). */
int b200bt_mc_portfolio_gbm(int S, const double* s0_host, const double* qty_host, const double* drift_host,
                            const double* vol_host, const float* chol_host, int64_t n_paths, int steps, uint64_t seed,
                            uint64_t path_offset, float* finals, float* maxdd, float* asset_finals_or_null,
                            b200bt_stream_t stream);

/* Historical bootstrap (:277-298) of whole days: `returns` is a device table [R][S] fp32 (one row per day that has a
 * return for every asset, R x S <= 12288), each step draws ONE row and applies it to every asset, which keeps the
 * cross-asset dependence.  block_len and log_returns as in b200bt_mc_bootstrap, whose index stream this one is:
 * asset i equals b200bt_mc_bootstrap on column i. */
int b200bt_mc_portfolio_bootstrap(int S, const float* returns, int R, int block_len, int log_returns,
                                  const double* s0_host, const double* qty_host, int64_t n_paths, int steps,
                                  uint64_t seed, uint64_t path_offset, float* finals, float* maxdd,
                                  float* asset_finals_or_null, b200bt_stream_t stream);

/* ---- trade-sequence Monte-Carlo of backtested strategies --------------------------------------------
 * The reference's open backtesting item "BACK-04: Add Monte Carlo simulations" (BACKLOG.md:194): resample the round
 * trips of a strategy's own trade records many times and report the spread of final equity and maximum drawdown.
 * Records as _simulate_trades emits them (services/strategy_evaluation.py:746-878): an entry record with pnl -fee and an
 * exit record with the trip's pnl; equity walk and drawdown rule of calculate_metrics (:119-139), resampling rule of
 * MonteCarloService (services/monte_carlo_service.py:277-298), statistics block as :339-374 with equity for price. */

/* Round-trip PnL from a sweep's event words.  For every lane = i * S + s of a sweep with an event buffer:
 *  n_trips[lane] (device int32) = n_records / 2, or -1 when n_records > event_cap (records were lost)
 *  fee[lane]     (device float64) = position_size * 0.001, the pnl of every entry record is -fee (:796-797, :810-811)
 *  trip_pnl[lane][j] (device float64, row stride ld_trip >= event_cap / 2) = pnl of the j-th exit record,
 *                qty * (price - entry) - position_size * 0.002 for a long trip, qty * (entry - price) - ... for a short
 *                one (entry word's B200BT_EVENT_SELL bit), qty = position_size / entry, prices = the fp32 closes widened
 *                to float64 (:819-820, :836-837, :852-853, :866-867); bit-identical to those float64 expressions.
 * price [S][ld] fp32, indiv [pop], stats [pop][S] and events [pop][S][event_cap] are the sweep's (device). */
int b200bt_trade_pnl(const float* price, int64_t ld, int S, int64_t N, const b200bt_individual* indiv, int pop,
                     const b200bt_lane_stats* stats, const uint32_t* events, int64_t event_cap, double* trip_pnl,
                     int64_t ld_trip, int32_t* n_trips, double* fee, b200bt_stream_t stream);

/* Monte-Carlo over the round trips of L lanes.  Unit of resampling: the round trip (entry and exit records stay
 * paired, so every path is again a valid record sequence).  Per path, T = n_trips_host[r] trip indices are drawn and the
 * equity walks in float64: E = initial_capital, peak = initial_capital; per drawn trip j, E += -fee, then
 * E += trip_pnl[r][j]; after each record a new peak needs E > peak, otherwise the record's drawdown is
 * (peak - E) / peak.  finals[r][p] = fp32(E_T), maxdd[r][p] = fp32(largest drawdown, 0 if none), each rounded once from
 * float64 (rows of n_paths; they feed b200bt_select / b200bt_mc_moments with s0 = initial_capital).  T = 0 gives
 * initial_capital and 0.
 * method B200BT_TRADE_MC_BOOTSTRAP: T draws with replacement, index __umulhi(u, T) (b200bt_mc_bootstrap's draw); with
 *        block_len > 1 circular blocks of consecutive trips by b200bt_mc_bootstrap's block rule.
 * method B200BT_TRADE_MC_SHUFFLE: every trip exactly once; position j holds pi(j), pi a balanced four-round Feistel
 *        bijection over the smallest even bit width 2h >= 8 with 2^2h >= T, six rounds, cycle-walked into [0, T); round
 *        keys = the first six words of the path's Philox blocks 0xFFFFFFFE and 0xFFFFFFFF (on fewer than 8 bits
 *        the position marginals were visibly skewed even with eight rounds).  This order is NOT uniform over
 *        all T! permutations (a keyed family of them, O(1) state per index); its position marginals pass chi-square
 *        tests and positions 0 and 1 are uncorrelated beyond the -1/(T-1) of a uniform permutation.
 * Randomness: Philox4x32-10, key = seed, counter = (gid lo, gid hi, block, lane id) with block = trip / 4 (bootstrap)
 * or 0xFFFFFFFE / 0xFFFFFFFF (shuffle),
 * gid = path_offset + p and lane id = lane_ids_host[r] (NULL = r).  A path is a pure function of (seed, lane id, gid, the
 * lane's trips): it does not depend on path sharding or on the other lanes of the call; lane id 1's bootstrap index
 * stream is b200bt_mc_bootstrap's for a table of T entries.
 * n_trips_host, fee_host, lane_ids_host: HOST arrays of L entries; trip_pnl: device [L][ld_trip] float64; finals, maxdd:
 * device [L][n_paths] fp32.  Limits: 0 <= T < 2^30 (ELIMIT above), T <= ld_trip, n_paths >= 1 (<= 2^38), block_len
 * >= 1, initial_capital > 0.  Lanes with T <= 6144 are staged in shared memory, larger ones read through L2. */
#define B200BT_TRADE_MC_BOOTSTRAP 0
#define B200BT_TRADE_MC_SHUFFLE 1
int b200bt_trade_mc(const double* trip_pnl, int64_t ld_trip, const int32_t* n_trips_host, const double* fee_host,
                    const uint32_t* lane_ids_host, int L, int method, int block_len, double initial_capital,
                    int64_t n_paths, uint64_t seed, uint64_t path_offset, float* finals, float* maxdd,
                    b200bt_stream_t stream);

/* ---- backtest overfitting of a population (csrc/overfitting.cu) -------------------------------------
 * The best of many backtests is biased upward by the search that found it.  These entry points give the inputs and
 * the core of the two standard measures: the Probability of Backtest Overfitting by combinatorially symmetric
 * cross-validation (CSCV; Bailey, Borwein, Lopez de Prado, Zhu 2015) and the Deflated Sharpe Ratio (Bailey, Lopez de
 * Prado 2014). */

/* Per-day PnL rows from a sweep's records: the daily buckets of calculate_metrics (services/strategy_evaluation.py
 * :141-159) kept as an array instead of folded into Sharpe / Sortino moments.  Inputs as b200bt_book_metrics: price
 * [S][ld_price], indiv [pop], lane_stats [pop][S], events [pop][S][event_cap] (device), cfg (host; clock checked like the
 * sweeps').  Records are priced with the expression of b200bt_trade_pnl (an entry record is -position_size * 0.001).
 * The calendar day of a record on bar b is (minute0 + b * bar_minutes + (b >= gap_bar ? gap_minutes : 0)) / 1440 in
 * unsigned 32 bits (gap_bar <= 0: no gap); first_day = minute0 / 1440 is the day of bar 0.
 *   lane_pnl [pop][S][D] float64 (device): [i][s][d] = sum of the pnl of lane (i, s)'s records on day first_day + d, in
 *            record order within each warp batch of 32 records; a day without records holds exactly 0.0 (the skipped
 *            days of a glued series are zero columns).  A lane with n_records > event_cap lost records: its row is NaN.
 *   book_pnl_or_null [pop][D] float64 (device, optional): sum over symbols 0..S-1, in that order, of lane_pnl[i][s][d]
 *            (NaN when any lane of the individual lost records).
 * D must cover the series: D >= day(N - 1) - first_day + 1 (B200BT_EINVAL otherwise).  Limits: N < 2^30, pop * S * D
 * fits int64.  Deterministic: every cell is written by one warp in a fixed order, no atomics. */
int b200bt_daily_pnl(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv, int pop,
                     const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats, const uint32_t* events,
                     int64_t event_cap, double* lane_pnl, int64_t D, double* book_pnl_or_null, b200bt_stream_t stream);

/* CSCV of N trials.  pnl: device float64 [N][ld >= T], one row of T per-period returns per trial (the periods must be
 * the same for every trial: rows of b200bt_daily_pnl's book_pnl hold every calendar day, zeros included); B even,
 * 2 <= B <= 20 (ELIMIT above 20), L = T / B >= 2, N >= 2.  The earliest r = T - B*L days are dropped; block b holds the
 * days [r + b*L, r + (b+1)*L).  Arithmetic (correctly rounded float64, no FMA contraction, sums in ascending order from
 * +0.0), per trial n over the kept days x_t:
 *   mu = (sum x_t) / (B*L);  d_t = x_t - mu;  a_b = sum over block b of d_t;  q_b = sum over block b of d_t*d_t
 *   m2 = (sum d_t*d_t) / (B*L), m3 = (sum (d_t*d_t)*d_t) / (B*L), m4 = (sum (d_t*d_t)*(d_t*d_t)) / (B*L)   (day order)
 *   sr = mu / sqrt(m2) * sqrt(252) if m2 > 0, else 0
 * Set J of k = B/2 blocks (ascending): A = sum a_b, Q = sum q_b, n = k*L, m = A/n, v = Q/n - m*m,
 *   SR_J = (mu + m) / sqrt(v) * sqrt(252) if v > 0, else 0
 * -- calculate_metrics' daily Sharpe rule, mean / std(ddof 0) * sqrt(252), 0 for std 0 (:180-188), but over every
 * calendar day of J including days without records, so that all trials share the same rows.
 * Combination c = 0 .. C(B, B/2) - 1 in itertools.combinations(range(B), B // 2) order: J_c in sample, its complement
 * out of sample.  Outputs (device): sel[c] = argmax over n of SR_IS (ties to the lowest n), is_sr[c] = SR_IS[sel],
 * oos_sr[c] = SR_OOS[sel], n_below[c] = #{n : SR_OOS_n < oos_sr[c]}, n_tied[c] = #{n != sel : SR_OOS_n == oos_sr[c]}
 * (int32 [C]); mu, m2, m3, m4, sr float64 [N].  Rows must be finite.  Deterministic.  Workspace: device, 16-byte aligned,
 * of b200bt_cscv_workspace_bytes(N, T, B) bytes (0 for arguments outside the limits). */
int64_t b200bt_cscv_workspace_bytes(int N, int64_t T, int B);
int b200bt_cscv(const double* pnl, int64_t ld, int N, int64_t T, int B, void* workspace, int64_t workspace_bytes,
                int32_t* sel, double* is_sr, double* oos_sr, int32_t* n_below, int32_t* n_tied, double* mu, double* m2,
                double* m3, double* m4, double* sr, b200bt_stream_t stream);

/* Data-snooping tests of N trials against one benchmark: White's Reality Check (2000), Hansen's Superior Predictive
 * Ability test (2005) and Romano and Wolf's StepM (2005), on the stationary bootstrap of Politis and Romano (1994).
 * d: device float64 [N][ld >= T] of differentials d[k][t] = x[k][t] - bench[t] (the host forms them); rows finite.
 * Arithmetic as b200bt_cscv: correctly rounded float64, no FMA contraction, sums in ascending order from +0.0.
 * Limits: 2 <= T <= 8192 (ELIMIT above, EINVAL below), 1 <= N < 2^31, ld >= T (EINVAL).
 *
 * b200bt_spa_moments, per trial k, with 0 < q <= 1 (EINVAL otherwise):
 *   mean[k] = (sum_t d_t) / T;  c_t = d_t - mean;  gamma_i = (sum_{t=0}^{T-1-i} c_t * c_{t+i}) / T
 *   p_0 = 1, p_i = p_{i-1} * (1 - q)  (running products, i = 1..T)
 *   kappa_i = ((T - i) / T) * p_i + (i / T) * p_{T-i}
 *   omega2[k] = gamma_0 + 2 * sum_{i=1}^{T-1} kappa_i * gamma_i   (Hansen's stationary-bootstrap variance)
 * mean and omega2 are exact restatements of these expressions.  Against kappa_i formed with pow((1-q), i) instead, the
 * running product p_i differs by at most i half-ulps (relative i * 2^-53), so omega2 agrees with such a restatement
 * within T * 2^-52 * (|gamma_0| + 2 sum |kappa_i gamma_i|) plus the rounding of the sums.  O(N T^2): one CTA per trial,
 * (3T + 1) * 8 bytes of shared memory.
 *
 * b200bt_spa_bootstrap: resample b = 0 .. n_boot - 1 draws the index sequence theta_b(0..T-1), forms
 *   m*[k][b] = (sum_t d[k][theta_b(t)]) / T   (t ascending; the N x n_boot matrix is never stored)
 * and writes out[j][b] = max over k of (m*[k][b] - shift[j][k]) * scale[j][k] for j < n_stats, 1 <= n_stats <= 8
 * (ELIMIT above, EINVAL at 0).  shift[j][k] = +inf excludes trial k from statistic j; NaN values are ignored; a
 * statistic with every trial excluded is -inf.  shift, scale: device float64 [n_stats][N]; out: device float64
 * [n_stats][n_boot].  The max does not depend on the order, so the output is deterministic.
 * Index stream: Philox4x32-10, key = seed, counter = (gid lo, gid hi, t >> 1, 0) with gid = boot_offset + b; day t uses
 * words x[2(t & 1)] (restart) and x[2(t & 1) + 1] (start).  Day 0 starts a block; day t >= 1 starts one iff
 * (uint64)x_restart < q32.  A block start is __umulhi(x_start, T); otherwise theta(t) = theta(t-1) + 1, wrapping at T.
 * q32 in [1, 2^32] (EINVAL outside): round(q * 2^32) for a mean block length 1 / q; 2^32 gives the iid bootstrap.  A
 * resample is a pure function of (seed, gid, T, q32): it does not depend on N, on the other trials, on how the
 * resamples are split over calls (boot_offset) or on the launch geometry.  n_boot >= 1.
 * Schedule: one CTA per (32-trial tile, resample range), one warp per resample, one lane per trial; a warp draws 64 days
 * at a time (one Philox block per lane, a max-scan for the latest block start).  Rows of T <= 768 days are staged in
 * shared memory as [t][32] (32 * T * 8 bytes); longer rows are read through L1 / L2.  The tiles' maxima meet in an
 * ordered-integer atomicMax over out (three launches: fill, bootstrap, decode). */
int b200bt_spa_moments(const double* d, int64_t ld, int N, int T, double q, double* mean, double* omega2,
                       b200bt_stream_t stream);
int b200bt_spa_bootstrap(const double* d, int64_t ld, int N, int T, uint64_t q32, int64_t n_boot, uint64_t seed,
                         uint64_t boot_offset, int n_stats, const double* shift, const double* scale, double* out,
                         b200bt_stream_t stream);

/* Model Confidence Set (Hansen, Lunde and Nason 2011) of N models on the stationary bootstrap of b200bt_spa_bootstrap.
 * x: device float64 [N][ld >= T], one per-day PnL row per model, finite.  The loss is the negated PnL, so the best model
 * has the highest mean.  Arithmetic as b200bt_spa_*: correctly rounded float64, no FMA contraction, every sum in the
 * ascending order stated from +0.0; every max is order-free.  So a NumPy restatement with the same loops matches bit for
 * bit, whatever the launch geometry or the split of the resamples over calls.
 *   xbar_k = (sum_t x[k][t]) / T                        (t ascending; b200bt_spa_moments' mean)
 *   m*[b][k] = (sum_t x[k][theta_b(t)]) / T              (t ascending; theta_b the index stream of b200bt_spa_bootstrap
 *                                                         for the same seed, gid = boot_offset + b, T and q32)
 *   zeta[b][k] = m*[b][k] - xbar_k                       (stored resample-major, [B][ld_z >= N])
 * T_R: sigma2_ij = (sum_b (zeta_bj - zeta_bi)^2) / B    (b ascending over all B resamples, 0 .. B-1)
 *      sigma_ij = sqrt(sigma2_ij), rho_ij = 1.0 / sigma_ij (a correctly rounded division, not a reciprocal
 *      approximation), t_ij = (xbar_j - xbar_i) / sigma_ij
 *      T_R(M) = max over i, j in M of t_ij; e_R(M) = argmax over i in M of (max over j in M of t_ij), lowest index on ties
 *      T*_R,b(M) = max over i, j in M of |zeta_bj - zeta_bi| * rho_ij
 * T_max: zbar_b(M) = (sum over j in M, ascending j, of zeta_bj) / m     (m = |M|)
 *      v_i(M) = (sum_b (zbar_b - zeta_bi)^2) / B (b ascending); s_i = sqrt(v_i)
 *      xbar_M = (sum over j in M, ascending j, of xbar_j) / m; t_i = (xbar_M - xbar_i) / s_i
 *      T_max(M) = max over i in M of t_i; e_max(M) = the argmax, lowest index on ties
 *      T*_b(M) = max over i in M of (zbar_b - zeta_bi) / s_i
 * Zero variance (sigma_ij = 0 or s_i = 0, whether the squares underflowed or not): t = 0 when the means are equal (the
 * difference is +-0), +inf or -inf with the sign of the difference otherwise; the pair or model adds 0 to every
 * bootstrap maximum (rho_ij = 0; the T_max term is 0).
 * Copies: these entries take the models as given.  Under T_R exact copies tie (t = 0, rho = 0) but leave one step
 * apart.  Under T_max a set's mean can differ from the copies' common value by rounding, so a step over copies of a
 * non-zero row compares rounding residues and can remove some copies at p = 0 while others stay.  Pass distinct rows:
 * overfitting.mcs makes byte-identical rows one model before it calls these entries.
 * Elimination: M_0 = all N models; step k = 0 .. N-2 removes e_k from M_k.  count[k] = #{b : T*_b(M_k) >= T(M_k)}: the
 * count is >= (not the strict > of b200bt_spa_bootstrap's tests), so under T_R, and under T_max for all-zero rows, N
 * identical rows give count B at every step (with a strict count they would all leave at p = 0).  The host forms p_k = count[k] / B and the MCS p-values.
 * Limits: 2 <= N <= 16384 (ELIMIT above, EINVAL below), n_boot >= 1, ld_z >= N, T as b200bt_spa_* (EINVAL for null
 * pointers and bad strides, before the device check).  max_bytes: the [B][N] and [N][N] float64 buffers an entry reads
 * or writes, counted with their strides, must total at most max_bytes, else ELIMIT.
 *
 * b200bt_boot_means (1 <= N <= 16384): out[b][k] at out + b * ld_out + k (ld_out >= N) = m*[b][k] - center[k], or m*[b][k]
 * when center_or_null is NULL, for resamples b = 0 .. n_boot-1 (gid = boot_offset + b).  b200bt_spa_bootstrap's
 * schedule and gather function, so m* is the very value whose maximum that entry takes.  Budget: n_boot * ld_out * 8.
 * b200bt_autocov (1 <= N < 2^31): per row, c_t = x_t - xbar and out[k][i] = (sum_{t=0}^{T-1-i} c_t * c_{t+i}) / T for
 * i = 0 .. K, 0 <= K < T (EINVAL otherwise): b200bt_spa_moments' gamma_i bit for bit; out: [N][K+1]; mean_or_null gets
 * xbar.  One CTA per row, T * 8 bytes of shared memory.
 * b200bt_mcs_pairwise: s2[i][j] (i < j, at s2 + i * N + j) += sum over this call's rows b of zeta (ascending) of
 * (zeta_bj - zeta_bi)^2; other entries untouched.  Zero s2 before the first call; calls over consecutive resample ranges
 * continue the ascending sum, so any split gives the same bits.  One CTA per upper (64 x 64) tile pair, 16 resamples
 * staged per step, 4 x 4 accumulators per thread.  Budget: n_boot * ld_z * 8 + N * N * 8.
 * b200bt_mcs_range_stats: from s2 in w over n_boot_total resamples, w becomes rho (symmetric, 0 on the diagonal) and t
 * gets t_ij at t + i * N + j (0 on the diagonal).  Budget: 2 * N * N * 8.
 * b200bt_mcs_range_order: the T_R elimination: order[k] = e_k (int32 [N], the last survivor last), stat[k] = T_R(M_k)
 * (float64 [N-1]); then rho_rank[r][c] = rho[order[r]][order[c]] for c > r, 0 otherwise.  rho_rank may alias t (which it
 * then overwrites), not rho.  One CTA keeps each live row's max and its column in shared memory (13 N bytes) and rescans
 * only the rows whose column was just eliminated.  Budget: 2 or 3 (t not aliased) * N * N * 8.
 * b200bt_mcs_range_boot: for this call's rows b of zeta (original model order), R_b(r) = max over c > r of
 * |zeta_b,order[c] - zeta_b,order[r]| * rho_rank[r][c] into rmax [n_boot][N], then count[k] (uint64 [N-1]) += #{b :
 * max over r >= k of R_b(r) >= stat[k]}: T*_R,b(M_k) = max over r >= k of R_b(r).  Calls over a split of the resamples
 * add up to the counts of one call.  One CTA per (64-resample, 64-rank) tile; O(B N^2 / 2).  Budget: n_boot * ld_z * 8 +
 * n_boot * N * 8 + N * N * 8.
 * b200bt_mcs_max: the whole T_max elimination over zeta [n_boot][ld_z] (every resample in one call): order, stat (as
 * above) and count[k] (uint64 [N-1], added to) for k = 0 .. N-2.  Per step three launches: v_i and t_i (a thread per
 * live model, b ascending), the argmax (one CTA), and the maxima, count and next zbar (a thread per resample).
 * Workspace: device, 16-byte aligned, b200bt_mcs_max_workspace_bytes(N, n_boot) bytes (0 outside the limits).  Budget:
 * n_boot * ld_z * 8. */
int b200bt_boot_means(const double* d, int64_t ld, int N, int T, uint64_t q32, int64_t n_boot, uint64_t seed,
                      uint64_t boot_offset, const double* center_or_null, double* out, int64_t ld_out, int64_t max_bytes,
                      b200bt_stream_t stream);
int b200bt_autocov(const double* d, int64_t ld, int N, int T, int K, double* out, double* mean_or_null,
                   b200bt_stream_t stream);
int b200bt_mcs_pairwise(const double* zeta, int64_t ld_z, int N, int64_t n_boot, double* s2, int64_t max_bytes,
                        b200bt_stream_t stream);
int b200bt_mcs_range_stats(const double* mean, int N, int64_t n_boot_total, double* w, double* t, int64_t max_bytes,
                           b200bt_stream_t stream);
int b200bt_mcs_range_order(const double* t, const double* rho, int N, int32_t* order, double* stat, double* rho_rank,
                           int64_t max_bytes, b200bt_stream_t stream);
int b200bt_mcs_range_boot(const double* zeta, int64_t ld_z, int N, int64_t n_boot, const int32_t* order,
                          const double* rho_rank, const double* stat, double* rmax, uint64_t* count, int64_t max_bytes,
                          b200bt_stream_t stream);
int64_t b200bt_mcs_max_workspace_bytes(int N, int64_t n_boot);
int b200bt_mcs_max(const double* zeta, int64_t ld_z, int N, int64_t n_boot, const double* mean, void* workspace,
                   int64_t workspace_bytes, int32_t* order, double* stat, uint64_t* count, int64_t max_bytes,
                   b200bt_stream_t stream);

/* ---- portfolio risk (SURVEY 8-f4) -------------------------------------------------------------------
 * Replaces the numeric core of services/portfolio_risk_service.py. */

/* Simple returns, df['close'].pct_change() (portfolio_risk_service.py:208): out[s][0] = NaN,
 * out[s][t] = close[s][t]/close[s][t-1] - 1 in float64, stored fp32 (after a zero close +-inf, or NaN for 0/0, as
 * pandas gives).  close, out: device [S][ld]; S <= 65535 (B200BT_ELIMIT above). */
int b200bt_pct_change(const float* close, int64_t ld, int S, int64_t N, float* out, int64_t ld_out,
                      b200bt_stream_t stream);

/* Tail sums for historical CVaR (calculate_conditional_var :248-284), NaN entries skipped (dropna; +-inf are kept):
 * out4 (device, float64) = [ sum x[x <= threshold], #(x <= threshold), #(non-NaN), sum non-NaN ].
 * Deterministic (fixed-order fold of per-CTA partials). */
int64_t b200bt_tail_stats_workspace_bytes(int64_t n);
int b200bt_tail_stats(const float* x, int64_t n, double threshold, double* out4, void* workspace,
                      int64_t workspace_bytes, b200bt_stream_t stream);

/* Pearson correlation matrix of S return rows (calculate_asset_correlation :286-326, pandas
 * DataFrame.corr(): pairwise-complete observations).  An entry is observed when it is finite: NaN and +-inf are both
 * missing, as pandas' np.isfinite mask makes them.  NaN out for no joint observation or zero variance over the pair's
 * joint observations; a series that is constant over them (a stale feed) gives exactly zero variance, hence NaN.
 * Deterministic (fixed-order fold of per-split partials, no atomics).  x: device [S][ld] fp32, out: device float64
 * [S][S], S <= 512. */
int64_t b200bt_correlation_workspace_bytes(int S, int64_t N);
int b200bt_correlation(const float* x, int64_t ld, int S, int64_t N, double* out, void* workspace,
                       int64_t workspace_bytes, b200bt_stream_t stream);

/* ---- GA operators on the device (SURVEY 8-f2) -------------------------------------------------------
 * The operators of services/genetic_algorithm.py:83-252 over a device matrix params [pop][genes] float64 (integer
 * genes hold integral values).  Ranges: host arrays lo / hi / is_int of length genes (<= 64).  Randomness is
 * Philox4x32-10 keyed by (seed; generation, slot): parity with the reference's Mersenne-twister stream is
 * DISTRIBUTIONAL (same operators and probabilities), results are a pure function of (seed, generation, inputs),
 * restated draw for draw by tests/ga_ref.py. */

/* initialize_population (:83-117): rows >= n_seeded are drawn uniformly from the ranges (randint / uniform),
 * rows < n_seeded (already written by the caller) are clamped to the ranges. */
int b200bt_ga_init(double* params, int pop, int genes, int n_seeded, const double* lo, const double* hi,
                   const int* is_int, uint64_t seed, b200bt_stream_t stream);

/* selection + crossover + mutation (:135-252) -> params_out (must not alias params).
 * ranked: device int32[pop], indices by descending fitness (stable); selected_workspace: device int32[pop].
 * elites = max(1, int(elitism_pct * pop)) best, copied unchanged to the first rows; every other selected slot is the
 * winner of a tournament of `tournament` (<= 8) distinct contenders; offspring pairs come from two uniform draws
 * of the selected list, uniform crossover with probability crossover_rate, per-gene mutation with mutation_rate.
 * elitism_pct must be finite (EINVAL otherwise, checked before the device); the elite count is clamped in double
 * precision, so any elitism_pct * pop >= pop gives pop elites (a plain copy of the best individuals) and any value
 * below 1 gives one. */
int b200bt_ga_next_generation(const double* params, const double* fitness, const int32_t* ranked, int pop, int genes,
                              const double* lo, const double* hi, const int* is_int, double elitism_pct,
                              int tournament, double crossover_rate, double mutation_rate, uint64_t seed,
                              uint32_t generation, int32_t* selected_workspace, double* params_out,
                              b200bt_stream_t stream);

/* ---- multi-objective ranking (NSGA-II; Deb, Pratap, Agarwal, Meyarivan 2002) ---------------------------------------
 * csrc/pareto.cu; restated by tests/pareto_ref.py. */

/* Objective matrix of a population: out[i][j] = (sum over s = 0..S-1, ascending, from +0.0, of stats[i][s].<field j>) / S
 * -- b200bt_fitness_reduce's expression, so field 12 (score) gives its fitness bit for bit.  stats: device [pop][S] (a
 * book's [pop] stats with S = 1); fields_host: host int[M], indices 0..18 of the fields of b200bt_lane_stats, trade_hash
 * is not one (EINVAL); out: device float64 [pop][ld_out].  1 <= M <= 8 (ELIMIT above), M <= ld_out (EINVAL).  Values are copied as
 * they are (NaN and +-inf included, no sign change). */
int b200bt_objective_matrix(const b200bt_lane_stats* stats, int pop, int S, const int* fields_host, int M, double* out,
                            int64_t ld_out, b200bt_stream_t stream);

/* Non-dominated fronts, crowding distance and crowded order of n points with M objectives.
 *   obj: device float64 [n][ld]; maximize_host: host int[M] (non-zero: larger is better).
 *   v[p][j] = maximize_j ? obj[p][j] : -obj[p][j], a NaN becomes -inf; larger v is better.
 *   p dominates q iff v[p][j] >= v[q][j] for every j and v[p][j] > v[q][j] for some j (identical vectors do not dominate
 *   each other; -inf == -inf).
 *   front (device int32 [n]): 0 for the non-dominated points; front k + 1 = the non-dominated points once fronts 0..k are
 *   removed.
 *   crowding (device float64 [n]): per front F and objective j, F's members ordered by (v[.][j], index) ascending; the
 *   first and the last get +inf; with r = v_max - v_min over F, an interior member adds (v_next - v_prev) / r unless r is
 *   0 or not finite.  Summed over j ascending from +0.0, correctly rounded (__dsub_rn, __ddiv_rn, __dadd_rn).  A front of
 *   one or two members is all +inf; crowding is never NaN.
 *   order (device int32 [n]): the indices sorted by (front asc, crowding desc, index asc).
 *   key_or_null (device float64 [n], optional): key[p] = -(position of p in order), +0.0 for the first -- the fitness
 *   with which b200bt_ga_next_generation's "first maximum wins" tournament is NSGA-II's crowded-comparison tournament.
 * Limits: 1 <= n <= 65536 (ELIMIT above), 1 <= M <= 8 (ELIMIT above), ld >= M.  Workspace: device, 256-byte aligned, of
 * b200bt_pareto_workspace_bytes(n, M) bytes (n^2 / 8 bytes of dominance bits and O(n M) more; 0 outside the limits).
 * No host synchronisation; deterministic (integer atomics only, and no output depends on their order).  Cost: the
 * dominance pass is O(n^2 M); the fronts take one grid-wide barrier each, so a chain of n fronts (M = 1, or perfectly
 * correlated objectives) is the worst case; crowding and order are O(sum over fronts of |F|^2 M). */
int64_t b200bt_pareto_workspace_bytes(int n, int M);
int b200bt_pareto_rank(const double* obj, int64_t ld, int n, int M, const int* maximize_host, void* workspace,
                       int64_t workspace_bytes, int32_t* front, double* crowding, int32_t* order, double* key_or_null,
                       b200bt_stream_t stream);

/* ---- market regimes (csrc/regime.cu) -----------------------------------------------------------------------------
 * services/market_regime_service.py labels the market bull / bear / ranging / volatile (detect_regime_from_data
 * :503-603) in 24-hour windows (update_strategy_performance_by_regime :844-889) and scores strategies per regime.  These
 * entry points give the labels of a market's own bars and the trade metrics of a sweep's records per label. */
#define B200BT_REGIME_BULL 0
#define B200BT_REGIME_BEAR 1
#define B200BT_REGIME_RANGING 2
#define B200BT_REGIME_VOLATILE 3
#define B200BT_REGIME_UNKNOWN 4

typedef struct b200bt_regime_params {
    int32_t sample_minutes;          /* minutes per point; a positive multiple of 5 and of bar_minutes (60: hourly)     */
    int32_t reserved;
    double volatile_volatility;      /* 1.5   VOLATILE_THRESHOLD                                                       */
    double bull_price_change;        /* 5.0   BULL_PRICE_CHANGE (percent)                                              */
    double bull_trend_strength;      /* 0.6   BULL_TREND_STRENGTH (compared with the fraction of uptrend points)        */
    double bear_price_change;        /* -5.0  BEAR_PRICE_CHANGE                                                        */
    double bear_trend_strength;      /* 0.6   BEAR_TREND_STRENGTH (fraction of downtrend points)                        */
    double ranging_price_range;      /* 3.0   RANGING_PRICE_RANGE (|change| in percent)                                 */
    double ranging_trend_strength;   /* 0.3   RANGING_TREND_STRENGTH (mean trend_strength)                              */
} b200bt_regime_params; /* 64 bytes */

typedef struct b200bt_regime_window {
    int64_t start_minute;            /* t0 + 1440 k; -1 for rows past the symbol's last window                          */
    int32_t n_points;                /* 0: the window is skipped (the reference never forms it)                         */
    int32_t label;                   /* B200BT_REGIME_*                                                                 */
    double volatility;               /* std (ddof 1) of the returns * sqrt(24); NaN with fewer than 2 returns           */
    double change_pct;               /* (last - first) / first * 100                                                    */
    double mean_strength;            /* mean trend_strength                                                             */
    double up_frac, down_frac, sideways_frac;
} b200bt_regime_window; /* 64 bytes */

/* Regime labels of every bar.  close, sma20, sma50, sma20_5m_aligned: device float32 [S][ld], ld >= N (SMA20 / SMA50 of
 * the closes and SMA20 of the 5-minute closes brought to this clock by b200bt_align: the last COMPLETED 5-minute bar; NaN
 * where undefined).  Bar t starts at minute m_t = minute0 + t * bar_minutes (minute0 >= 0: the unbroken clock, no glued
 * series).
 *   Points: one per epoch-aligned sample_minutes bucket, at its last bar t (the next bar starts in a later bucket; a
 *   bucket cut by the end of the series has none), from the first such bar where all three averages are defined.  The
 *   point's price is close[t]; with s1 = (c - sma20) / sma20 * 100 and s5 = (c - sma20_5m) / sma20_5m * 100 its
 *   trend_strength is |s1 * 0.6 + s5 * 0.4| and its trend up if c > sma20 > sma50, down if c < sma20 < sma50, else
 *   sideways (market_monitor_service.py:263-280; float64, correctly rounded, no FMA contraction).
 *   Windows: k = 0, 1, ... cover the minutes [t0 + 1440 k, t0 + 1440 (k + 1)), t0 = the first point's minute, while their
 *   start < the last point's minute.  Per window over its points p_0..p_{n-1} in time order: returns p_i / p_{i-1} - 1,
 *   volatility = their sample std * sqrt(24) (NaN below 2 returns, and NaN is never volatile), change = (p_{n-1} - p_0) /
 *   p_0 * 100, the mean trend_strength and the up / down / sideways fractions.  Fewer than 2 points: UNKNOWN.  Otherwise,
 *   in order: VOLATILE if volatility > volatile_volatility; BULL if change > bull_price_change and up >
 *   bull_trend_strength; BEAR if change < bear_price_change and down > bear_trend_strength; RANGING if |change| <
 *   ranging_price_range and mean strength < ranging_trend_strength; else BULL if up > down and up > sideways, BEAR if
 *   down > up and down > sideways, else RANGING.
 *   labels: device uint8 [S][ld_labels] (ld_labels >= N unless S == 1): the label of the window holding m_t; UNKNOWN
 *   before t0, after the last window and in skipped or unknown windows.
 *   window_stats_or_null: device [S][max_windows] rows, row k = window k; max_windows >= b200bt_regime_max_windows(N,
 *   bar_minutes) (EINVAL otherwise).
 * Checked before the device: null pointers, sizes, minute0 < 0, sample_minutes not a positive multiple of 5 and of
 * bar_minutes (all EINVAL), N >= 2^30 (ELIMIT).  No atomics on outputs; deterministic. */
int64_t b200bt_regime_max_windows(int64_t N, int bar_minutes);
int b200bt_regime_labels(const float* close, const float* sma20, const float* sma50, const float* sma20_5m_aligned, int S,
                         int64_t N, int64_t ld, int64_t minute0, int bar_minutes, const b200bt_regime_params* params,
                         uint8_t* labels, int64_t ld_labels, b200bt_regime_window* window_stats_or_null,
                         int64_t max_windows, b200bt_stream_t stream);

/* Trade metrics per bar label.  Inputs as b200bt_daily_pnl, plus labels: device uint8 [S][ld_labels] (ld_labels >= N),
 * or ld_labels = 0 for one row shared by every symbol.  class_stats: device [R][pop][S], 1 <= R <= 8 (ELIMIT above):
 * block r holds, for lane (i, s), calculate_metrics and the cfg's score on the sub-list of the lane's records whose own
 * bar carries label r (an entry and its exit may fall into different classes; labels >= R belong to no class).  Inside a
 * class everything is as b200bt_book_metrics on a mixed list: equity from initial_capital, the calendar days of the
 * class's records (the cfg's gap applies), sum_duration_bars over the pairs (2k, 2k + 1) of the class list, trade_hash =
 * xor of event_hash(index in the class list, word).  With R = 1 and every label 0, counts and hash equal the lane's.  A
 * lane with n_records > event_cap gives n_records = -1, score NaN and zeros in every class.  Deterministic. */
int b200bt_class_stats(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv, int pop,
                       const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats, const uint32_t* events,
                       int64_t event_cap, const uint8_t* labels, int64_t ld_labels, int R,
                       b200bt_lane_stats* class_stats, b200bt_stream_t stream);

/* ---- grid trading (csrc/grid.cu) ----------------------------------------------------------------------------------
 * A backtest of services/grid_trading_strategy.py's GridTradingStrategy, whose only evaluation is "simulation mode": the
 * live loop of run() (:122-233) against the exchange ticker.  Here every (individual, symbol) lane is ONE symbol's service
 * instance run over a market's bars (the reference keeps num_grids and the pcts service-wide, so a multi-symbol service
 * couples its symbols at each adjustment; that coupled form is b200bt_grid_service_sweep below).
 *
 * Clock: tick k = 0 .. T - 1 is bar start_bar + k (T = N - start_bar); its price is the bar's close widened to float64.
 * __init__ / _initialize_grid (:245-345) run at tick 0: start_time, last_rebalance and last_adjustment are t0.  On every tick,
 * tick 0 included, the loop body runs, in order:
 *   _process_grid_simulation (:679-779) with last = the previous tick's price (tick 0: last == cur, nothing happens).
 *     Up move (cur > last): every level with last <= L_i <= cur is a trade with profit (L_i - L_{f-1}) * qty, f the first
 *     index holding L_i's value (levels.index, :712: every copy of a repeated level earns the step under the first copy;
 *     0 for f = 0), profitable when the profit is > 0.  Down move (cur < last): every level with cur <= L_i <= last is a
 *     trade with no profit.  Equal prices do nothing, and so does a NaN close: the tick with it and the tick after it are
 *     neither move (the rebalance check's compares are false too, and mark_to_market is NaN when the last close is NaN).
 *     A level equal to the last price is counted again.  qty = qty[s] (symbol_settings' quantity_per_grid, else the
 *     global one, :387-400).
 *   The rebalance check (:178-186): (now - last_rebalance) > rebalance_frequency with a strict >, and last_rebalance is reset
 *     whenever the check runs, so it runs on the ticks k = m * rebalance_ticks (m >= 1), rebalance_ticks =
 *     floor(frequency / bar_seconds) + 1 (61 at 1-minute bars and 3600 s).  _rebalance_grid (:781-838): when cur <
 *     lower * 1.05 or cur > upper * 0.95 the grid is regenerated around cur with the CURRENT pcts and num_grids:
 *     lower = cur * (1 - lower_pct / 100), upper = cur * (1 + upper_pct / 100).  Quirks kept: with 5 % boundaries the two
 *     thresholds overlap, so nearly every check regenerates; symbol_settings' boundary pcts are never read.
 *   The adjustment check (:189-196), same timing with adjust_ticks from auto_adjust_period (1441 at 1-minute bars and one
 *     day), _adjust_grid_parameters (:840-905):
 *     regime rule (:847-883), only with B200BT_GRID_ADAPT_REGIME and a regime source (labels and table; none = the
 *       reference without market_regime_history in Redis): the label of the adjust tick's bar selects table[label]; an
 *       entry with apply != 0 sets num_grids and both pcts (ranging_* / volatile_* of the config; b200bt_regime_labels
 *       emits no "trending" label, so the trending_* branch never fires).
 *     win-rate rule (:886-905): when total_trades > 10, profitable / total < 0.4 gives num_grids = max(5, n - 2), > 0.7
 *       gives min(20, n + 2).  grid_spread feeds no level and is not simulated.
 *     Both take effect at the next regeneration.
 * Levels (_generate_grid_levels :347-385), i = 0 .. n: arithmetic lower + i * step, step = (upper - lower) / n, exact IEEE
 * float64 (no FMA contraction); geometric lower * pow(ratio, i), ratio = pow(upper / lower, 1 / n) with CUDA's pow, which
 * may differ from the C library's by a few ulps.  near_ties counts the up or down moves on which a price compared with a geometric
 * level lies within |L| * 2^-50 (<= 4 ulps) of it: only those ticks can decide a compare differently from the reference.
 * Levels must be non-decreasing in i (true for finite lower <= upper); "volatility_based" draws random numbers and is not
 * a grid type here.
 *
 * init_bounds (device float64 [pop][S][2]): the initial (lower, upper) of each lane, computed by the caller from the
 * individual's boundary rule (fixed pcts or auto_boundaries' volatility of the daily closes, :266-289).  qty: device float64
 * [S].  labels_or_null: device uint8 [S][ld_labels] bar labels (ld_labels = 0: one row for every symbol; B200BT_REGIME_*),
 * regime_table_host_or_null: host [B200BT_GRID_REGIME_RULES] rules indexed by label (labels >= 5 change nothing).
 * stats: device [pop][S].  day_profit_or_null: device float64 [pop][D]: row i, column d = the realised profit of
 * individual i on calendar day first_day + d summed over its symbols 0..S-1 in that order (first_day = minute0 / 1440, the
 * day of bar 0; a day is (minute0 + bar * bar_minutes) / 1440), b200bt_cscv's row shape; D >= day(N - 1) - first_day + 1.
 * With day_profit the symbols of an individual run one after another in one warp; stats are the same either way.
 * An individual outside the limits (num_grids 1 .. B200BT_GRID_MAX_GRIDS, grid_type 0 / 1, periods >= 1) gets NaN stats.
 * Checked before the device: null pointers, sizes, start_bar in [0, N - 1], bar_minutes > 0, minute0 >= 0, ld_labels, D,
 * the table's num_grids (all EINVAL); N >= 2^30, S > 65535 (ELIMIT).  Deterministic: no atomics. */
#define B200BT_GRID_ARITHMETIC 0
#define B200BT_GRID_GEOMETRIC 1
#define B200BT_GRID_ADAPT_REGIME 1       /* adapt_to_market_regime                                          */
#define B200BT_GRID_AUTO_BOUNDARIES 2    /* auto_boundaries: read by the host that makes init_bounds only   */
#define B200BT_GRID_MAX_GRIDS 127
#define B200BT_GRID_REGIME_RULES 5

typedef struct b200bt_grid_individual {
    int32_t num_grids;        /* service-wide num_grids at t0                                                     */
    int32_t grid_type;        /* B200BT_GRID_ARITHMETIC / _GEOMETRIC                                              */
    int32_t rebalance_ticks;  /* floor(rebalance_frequency / bar_seconds) + 1                                     */
    int32_t adjust_ticks;     /* floor(auto_adjust_period / bar_seconds) + 1                                      */
    int32_t flags;            /* B200BT_GRID_ADAPT_REGIME | B200BT_GRID_AUTO_BOUNDARIES                           */
    int32_t reserved;
    double lower_pct;         /* lower_boundary_pct: regenerations (and the initial grid without auto_boundaries)  */
    double upper_pct;         /* upper_boundary_pct                                                               */
} b200bt_grid_individual;     /* 40 bytes */

typedef struct b200bt_grid_regime_rule {
    int32_t apply;            /* 0: the label changes nothing                                                     */
    int32_t num_grids;
    double lower_pct;
    double upper_pct;
} b200bt_grid_regime_rule;    /* 24 bytes */

/* Per-lane result: 20 float64 fields (160 bytes, the size of b200bt_lane_stats), so b200bt_objective_matrix averages any
 * field 0..18 over the symbols unchanged. */
typedef struct b200bt_grid_stats {
    double total_profit;       /* grid_profits[symbol]['total_profit'] (order of float64 additions may differ)          */
    double total_trades;       /* up_crossings + down_crossings                                                         */
    double profitable_trades;
    double win_rate;           /* profitable / total, 0 without trades (_update_performance_metrics :941-958)           */
    double profit_per_day;     /* total_profit / ((t_last - t0) in days), 0 when T = 1 (:951)                           */
    double up_crossings;
    double down_crossings;
    double n_regenerations;    /* rebalance checks that regenerated the grid                                            */
    double num_grids;          /* the service's num_grids at the end                                                    */
    double lower;              /* the active grid's boundaries at the end                                               */
    double upper;
    /* beyond the reference: the simulated fills marked to market.  A down-crossing buys qty at the level, an up-crossing
     * sells qty at the level; the reference's profit ignores the inventory this accumulates and never goes negative. */
    double cash;               /* sum of +-level * qty                                                                  */
    double position;           /* (down - up crossings) * qty                                                           */
    double mark_to_market;     /* cash + position * last close                                                          */
    double max_position;       /* largest and smallest position after any tick (0 at t0)                                */
    double min_position;
    double n_rebalance_checks;
    double n_adjustments;
    double n_ticks;            /* T                                                                                     */
    double near_ties;          /* see above; 0 on arithmetic grids                                                      */
} b200bt_grid_stats;           /* 160 bytes */

int b200bt_grid_sweep(const float* price, int64_t ld_price, int S, int64_t N, int64_t start_bar, int bar_minutes,
                      int64_t minute0, const b200bt_grid_individual* indiv, int pop, const double* qty,
                      const double* init_bounds, const uint8_t* labels_or_null, int64_t ld_labels,
                      const b200bt_grid_regime_rule* regime_table_host_or_null, b200bt_grid_stats* stats,
                      double* day_profit_or_null, int64_t D, b200bt_stream_t stream);

/* The coupled multi-symbol service: one individual is ONE service instance trading all S symbols of the market, as run()
 * (:160-206) runs one instance for every configured symbol (config.json's grid_trading.symbols).  num_grids,
 * lower_boundary_pct and upper_boundary_pct are fields of the instance (:72-78), so they are per individual, not per lane.
 * The rule is b200bt_grid_sweep's with these differences:
 *   Every symbol initialises at tick 0, so all lanes of an individual share the check ticks.  On an adjust tick the loop
 *   body runs (:166-198): the crossings of every symbol, then every symbol's rebalance check (a regeneration uses the
 *   service's values before this tick's adjustment, :809-816), then _adjust_grid_parameters(symbol) (:840-905) for
 *   symbols 0 .. S-1 in order, each MUTATING the shared fields: the regime rule of the tick's label (absolute values),
 *   then the win-rate rule on that symbol's own grid_profits counts (total_trades > 10; < 0.4 gives max(5, n - 2),
 *   > 0.7 gives min(20, n + 2)).  So when the regime rule fires, only the last symbol's win rate survives it; without
 *   it, the +-2 steps of all symbols add up.
 *   Labels: the reference reads ONE key (market_regime_history), so labels_or_null is one row shared by every symbol
 *   (ld_labels = 0); per-symbol rows are EINVAL.  Labels >= 5 change nothing, as before.
 * stats: device [pop][S] in b200bt_grid_stats' layout (b200bt_objective_matrix reads it unchanged); num_grids, lower and
 * upper are the lane's final grid, n_adjustments the service's.  service_or_null: device [pop].  day_profit_or_null as
 * b200bt_grid_sweep (symbols 0 .. S-1 added in that order).  Counts, regeneration ticks, final grids and the service's
 * num_grids are exact on lanes without geometric near ties; profit sums differ from the reference only by the order of
 * float64 additions (a lane's sums are reduced over its warp at every adjust tick).  With S = 1, or with adjust_ticks >= T,
 * the lanes are b200bt_grid_sweep's lanes (bit-equal when adjust_ticks >= T).
 * Schedule: one CTA per individual, min(S, 16) warps, warp w running symbols w, w + W, ... between two adjust ticks, where
 * the warps meet and thread 0 applies the S rule pairs in order; with day rows one warp runs every symbol in order.
 * An individual outside the limits gets NaN stats and a NaN service record.  Checked before the device: as
 * b200bt_grid_sweep but any S, plus labels_or_null with ld_labels != 0 (EINVAL).  Deterministic: no atomics. */
typedef struct b200bt_grid_service_stats {
    double total_profit;        /* grid_performance (:941-958): the lanes' total_profit summed in symbol order          */
    double total_trades;
    double profitable_trades;
    double win_rate;            /* profitable / total, 0 without trades                                                  */
    double profit_per_day;      /* total_profit / ((t_last - t0) in days), 0 when T = 1                                  */
    double num_grids;           /* the service's num_grids, lower_boundary_pct and upper_boundary_pct at the end          */
    double lower_pct;
    double upper_pct;
    double n_adjustments;       /* adjust ticks                                                                          */
    double n_num_grids_changes; /* adjust ticks after which num_grids differs from its value before them                 */
    double min_num_grids;       /* smallest and largest value num_grids took (t0 and after every rule, within a tick too)  */
    double max_num_grids;
} b200bt_grid_service_stats;    /* 96 bytes */

int b200bt_grid_service_sweep(const float* price, int64_t ld_price, int S, int64_t N, int64_t start_bar, int bar_minutes,
                              int64_t minute0, const b200bt_grid_individual* indiv, int pop, const double* qty,
                              const double* init_bounds, const uint8_t* labels_or_null, int64_t ld_labels,
                              const b200bt_grid_regime_rule* regime_table_host_or_null, b200bt_grid_stats* stats,
                              b200bt_grid_service_stats* service_or_null, double* day_profit_or_null, int64_t D,
                              b200bt_stream_t stream);

/* ---- dollar-cost averaging (csrc/dca.cu) --------------------------------------------------------------------------
 * A backtest of services/dca_strategy.py's DCAStrategy, whose only evaluation is "simulation mode": the live loop of run()
 * (:140-239) against the exchange ticker.  Here one individual is ONE service instance trading all S symbols of a market
 * (the rebalance couples them), run over the market's bars.  Every float64 operation of the reference happens in a fixed
 * order within an individual, and the kernel performs the same operations in the same order with explicit _rn
 * intrinsics (no FMA contraction): every output field is bit-exact.
 *
 * Clock: tick k = 0 .. T - 1 is bar start_bar + k (T = N - start_bar); its time is the bar's start minute m, its price the
 * bar's close widened to float64, its weekday that of its UTC day ((m / 1440 + 3) % 7, Monday = 0; the reference reads the
 * naive local clock).  One tick per bar stands in for update_interval.  __init__ and _initialize_dca_strategy (:241-320)
 * run at tick 0: last_rebalance = t0 - rebalance_interval_days (:124), and each symbol's first next_scheduled_buy is
 * _calculate_next_purchase_time at t0.  On every tick, tick 0 included, in this order:
 *   1. _process_dca (:452-501) for each symbol in order: a scheduled purchase when now >= next_scheduled_buy, then
 *      next_scheduled_buy = now + interval (_calculate_next_purchase_time :347-450).  _check_market_conditions always
 *      proceeds (nothing in the reference writes market_volatility or market_sentiment to Redis).  The interval:
 *        with adaptive_scheduling and a non-empty market_regime_based dict, the tick's label picks bull_ / bear_ /
 *        volatile_interval_hours (crab_ never fires: b200bt_regime_labels emits ranging, not crab; ranging, unknown,
 *        labels >= 5 and no label source leave it unchanged);
 *        with adaptive_scheduling and weighted_scheduling, it is multiplied by 1 + 0.2 * day_of_week_weight on Saturday
 *        and Sunday and clamped to [0.5, 1.5] x itself; the volatility and sentiment factors stay 1 (no data source);
 *        timedelta(hours=x) rounds it to microseconds; the purchase fires on the first later tick whose time is >= next.
 *   2. The rebalance check (:191-200): (now - last_rebalance).days >= R, with last_rebalance = now whenever it runs: tick 0,
 *      then every ceil(R * 1440 / bar_minutes) ticks (every tick for R <= 0).  _rebalance_portfolio, simulation branch
 *      (:864-1021): v_s = Q_s * p_s after step 1, total = (v_0 + ... + v_{S-1}) + usdc_balance, alloc_s = v_s / total
 *      (0 when total <= 0); symbol s buys total * target_s - v_s USDC when |(alloc_s - target_s) / target_s| * 100 >
 *      max_deviation_pct (0 when target_s <= 0) and v_s < total * target_s.  All decisions precede the buys, which go
 *      through _update_position_after_purchase with no clamp and no effect on last_purchases or the dip state.
 *   3. _check_for_dips (:817-862) for each symbol in order, with price_dip_detection: skipped while (now - last
 *      dip).days < max_dip_frequency_days; otherwise a dip purchase when dip_pct[s][bar] >= dip_threshold_pct (NaN never).
 * A purchase (_execute_dca_purchase :548-649, _calculate_adjusted_order_size :651-740, _update_position_after_purchase
 * :742-802): order = base, * (1 + additional_dip_allocation) for a dip, * bear_market_adjustment when
 * increase_in_bear_market and the tick's label is bear, clamped to [min_order, max_order] (the host's table);
 * q = floor(order / p * 10^prec) / 10^prec; invested += p * q; quantity += q; average = invested / quantity.  The service's
 * own total_invested adds the order, not p * q (the stats' order_usdc).
 * Mirrored quirks (the host's tables carry them): _get_symbol_specific_settings (:322-345) REPLACES symbols_config per
 * symbol, so after initialisation only the LAST symbol keeps its symbol_settings: each symbol's first interval uses its own
 * interval_hours, later intervals, base orders and rebalance targets use the global values (1 / S) for every symbol but
 * the last.  _get_quantity_precision (:1094-1100) counts the decimals of str(float(stepSize)): a step of 1e-05 prints in
 * scientific notation and gives precision 0.  The service never sells; take_profit_*, stop_loss_*, schedule_type,
 * weekly / monthly_dca_day, total_allocation, auto_adjust_order_size and value_averaging are read and never used.  The USDC
 * balance (get_account) is constant: simulation mode places no orders.
 *
 * b200bt_dca_dip_pct: dip_pct [S][ld_dip] float64, the market-only series of step 3: at bar b (minute m) the klines are
 * the UTC days whose start is >= m - 7 days and that hold a bar with start <= m, each day's high the max high of those bars
 * (the current day is partial); with fewer than 2 klines, or a recent high of 0 (ZeroDivisionError, caught), NaN; else
 * ((H - close) / H) * 100 with H the max of the day highs.  Per-day prefix maxima plus the previous whole days: O(N).
 * b200bt_dca_sweep: workspace >= b200bt_dca_workspace_bytes(S, N) bytes of device memory (block maxima of dip_pct over 32,
 * 1 024 and 32 768 bars, rebuilt on every call: a lane skips every block below its threshold).  indiv: device [pop];
 * first_us: device int64 [pop][S][5][2], each symbol's first interval indexed [label][weekend]; target, pow10: device
 * float64 [S], the rebalance targets and 10^precision.  labels_or_null as b200bt_grid_sweep.  rebalance_any: nonzero when
 * some individual has B200BT_DCA_REBALANCE (an individual with it gets NaN stats otherwise).  stats: device [pop][S];
 * service_or_null: device [pop]; day_or_null: device float64 [pop][D]: row d = the change of sum_s (Q_s * c_s - I_s)
 * between the last ticks of calendar days first_day + d - 1 and first_day + d, the symbols' changes added in order (the
 * value before tick 0 is 0; days before the start tick's day are 0), b200bt_cscv's row shape; D as b200bt_grid_sweep.
 * One CTA per individual and one warp per symbol; the warps meet at rebalance ticks (and day ends with day rows) only.
 * Checked before the device: null pointers, sizes, ld, start_bar in [0, N - 1], bar_minutes > 0, minute0 >= 0 and the
 * clock in microseconds < 2^62, ld_labels, D, the workspace size (EINVAL); N >= 2^30, and S > 32 with rebalance_any or
 * day rows (ELIMIT).  Deterministic: no atomics. */
#define B200BT_DCA_DIP 1                 /* price_dip_detection                                              */
#define B200BT_DCA_REBALANCE 2           /* periodic_rebalancing.enabled                                     */
#define B200BT_DCA_MAX_COUPLED 32        /* symbols of one individual that meet at a rebalance / day end     */

typedef struct b200bt_dca_individual {
    int64_t later_us[2][5][2];    /* interval after a scheduled purchase, us: [last symbol?][label][weekend]            */
    double order[2][2][2];        /* clamped order size, USDC: [last symbol?][dip?][bear?]                              */
    double dip_threshold_pct;
    double max_deviation_pct;     /* periodic_rebalancing.max_deviation_pct                                             */
    int64_t dip_cooldown_minutes; /* ceil(max_dip_frequency_days) * 1440, 0 = none                                      */
    int64_t rebalance_first;      /* tick of the first rebalance (0)                                                    */
    int64_t rebalance_period;     /* ticks between rebalances, >= 1                                                     */
    int32_t flags;                /* B200BT_DCA_DIP | B200BT_DCA_REBALANCE                                              */
    int32_t reserved;
} b200bt_dca_individual;          /* 272 bytes */

/* Per-lane result: 20 float64 fields (160 bytes), so b200bt_objective_matrix averages any field unchanged. */
typedef struct b200bt_dca_stats {
    double total_invested;        /* dca_positions[symbol] at the last tick (:253-264)                                  */
    double total_quantity;
    double average_price;
    double current_value;         /* Q * last close                                                                     */
    double profit_loss;
    double profit_loss_pct;
    double n_scheduled;           /* purchases by kind                                                                  */
    double n_dip;
    double n_rebalance;
    double order_usdc;            /* sum of the clamped orders of the scheduled and dip purchases, in time order        */
    double last_purchase_price;   /* 0 without a purchase                                                               */
    double last_purchase_tick;    /* of any kind; -1 without                                                            */
    double next_scheduled_us;     /* next_scheduled_buy - t0 in microseconds                                            */
    double last_dip_tick;         /* -1 without                                                                         */
    /* beyond the reference */
    double n_zero_quantity;       /* purchases whose quantity rounded to 0                                              */
    double n_rebalance_checks;
    double min_day_profit_loss;   /* lowest Q * c - I at the last tick of a day                                         */
    double purchase_hash;         /* xor over the purchases of fmix32(4 * tick + kind) (MurmurHash3's finaliser, 32-bit), kind
                                   * 0 scheduled, 1 dip, 2 rebalance                                                    */
    double n_ticks;               /* T                                                                                  */
    double reserved;
} b200bt_dca_stats;               /* 160 bytes */

/* _update_performance_metrics (:1023-1092) at the last tick, the symbols summed in order. */
typedef struct b200bt_dca_service {
    double total_purchases;       /* scheduled + dip purchases (rebalance buys do not count, :640-642)                  */
    double total_invested;
    double total_value;
    double total_profit;
    double total_profit_pct;
} b200bt_dca_service;             /* 40 bytes */

int b200bt_dca_dip_pct(const float* high, const float* close, int64_t ld, int S, int64_t N, int64_t minute0,
                       int bar_minutes, double* dip_pct, int64_t ld_dip, b200bt_stream_t stream);
int64_t b200bt_dca_workspace_bytes(int S, int64_t N);
int b200bt_dca_sweep(const float* close, int64_t ld_close, const double* dip_pct, int64_t ld_dip, int S, int64_t N,
                     int64_t start_bar, int bar_minutes, int64_t minute0, void* workspace, int64_t workspace_bytes,
                     const b200bt_dca_individual* indiv, const int64_t* first_us, int pop, int rebalance_any,
                     const double* target, const double* pow10, const uint8_t* labels_or_null, int64_t ld_labels,
                     double usdc_balance, b200bt_dca_stats* stats, b200bt_dca_service* service_or_null,
                     double* day_or_null, int64_t D, b200bt_stream_t stream);

/* ---- reinforcement-learning agents (csrc/rl.cu) -------------------------------------------------------------------
 * services/reinforcement_learning.py's TradingRLAgent on its NumPy path, trained the way the strategy-evolution service's
 * `rl` method trains it (optimize_with_reinforcement_learning, strategy_evolution_service.py:696-791), for a population of
 * agents at once.  The reference trains on `historical_market_data` that nothing writes; the points here are OUR wiring
 * (the reference never defines them, as with the GA fitness, SURVEY 0): point t of a symbol is bar t of the market on the
 * caller's clock with price = close, rsi = RSI(14), macd / macd_signal = MACD(12, 26, 9), bb_* = BB(20, 2), ema_short /
 * ema_long = EMA 12 / 26, atr = ATR(14) (b200bt_analyzer's columns, NaN policy applied), volume = the bar volume,
 * price_change_1h / _24h = 100 (c_t - c_{t-h}) / c_{t-h} over h = 60 and 1 440 minutes of the clock (0 where t < h, the
 * reference's .get(..., 0)), trend = TechnicalAnalyzer.get_trend's rule (binance_ml_strategy.py:184-203) per bar on close,
 * SMA20 and SMA50.
 *
 * b200bt_rl_states: states [S][N][B200BT_RL_FEATURES] float64, _convert_market_data_to_state (:793-847) per point, in the
 * feature order of _initialize_rl_agent (:203-207): rsi / 100, (macd + 1) / 2, (macd_signal + 1) / 2, then with price p > 0
 * bb_upper = (upper - p) / range, bb_lower = (p - lower) / range (0.5 each when range = upper - lower <= 0), bb_middle =
 * (p - middle) / p, ema_short / p, ema_long / p, atr / p (p <= 0: 0.5, 0.5, 0.5, 1, 1, 0); min(volume / 10^6, 1);
 * (pc_1h + 10) / 20; (pc_24h + 30) / 60; the social features at their defaults 50, 0, 0 (no social data): 0.5, 0, 0;
 * market_trend 0.8 uptrend, 0.2 downtrend, else 0.5.  cols: b200bt_analyzer's output for the same S and N; close, volume:
 * [S][ld] fp32.  bar_minutes must divide 60.  Every value is formed with explicitly rounded float64 operations.
 *
 * b200bt_rl_train: A agents, one warp each, over a schedule of n_calls calls shared by all agents.  Call c covers the points
 * [max(0, end_c - points_per_call + 1), end_c] of the agent's symbol; per point i (:718-754): state s_i, action = act(s_i),
 * next state s_{i+1} (the LAST point uses itself, :739-741), reward r = _calculate_reward(action, s_i, next) (:849-899), done
 * only on the last point (:747), remember, and replay when the memory holds >= batch_size transitions.  After the points:
 * the online Q-values of the last point and the call's avg_reward = (r_0 + ... + r_{n-1}) / n (:758-779).  The agent
 * persists across calls and launches: memory and epsilon carry over.
 *   network (:132-155)   W1 [16][24], b1 [24], W2 [24][24], b2 [24], W3 [24][3], b3 [3] (B200BT_RL_PARAMS doubles in that
 *                        order, row-major); forward (:157-184) ReLU, ReLU, linear; actions BUY, HOLD, SELL = 0, 1, 2
 *   act (:292-318)       u = uniform (ACT stream); u < epsilon: below(3); else the argmax of the online Q-values (first
 *                        maximum); the uniform is drawn for every point
 *   remember (:320-333)  a deque(maxlen=memory_size): a ring of one word per transition (point, action, done); the state,
 *                        next state and reward are re-derived from the state table
 *   replay (:335-419)    1. batch_size distinct positions of the deque, j = the j-th oldest transition, drawn as below(fill)
 *                        with repeats rejected (SAMPLE stream), used in draw order; 2. current_q with the online, next_q
 *                        with the target weights, before any update; 3. target = current_q with target[a] = r if done else
 *                        r + gamma * max(next_q); 4. _numpy_train (:186-241): one SGD step per sample in minibatch order,
 *                        all six gradients from that sample's pre-update weights, ReLU mask where hidden <= 0, w -= alpha *
 *                        d (original_outputs has no effect); 5. loss = mean squared error of the post-update outputs (only
 *                        computed with a history); 6. step += 1, target = online every update_target_every replays; 7.
 *                        epsilon *= epsilon_decay while epsilon > epsilon_end (per replay); 8. mean_q = mean of max(current_q)
 *   init (:142-155)      randn * 0.1 for W1, W2, W3 in that order (Box-Muller of the INIT stream: normal pair p from block p,
 *                        r = sqrt(-2 log(1 - u1)), r cos(2 pi u2), r sin(2 pi u2)), biases 0, target = online; or the
 *                        caller's init_weights_or_null (device [A][B200BT_RL_PARAMS])
 * RNG: Philox4x32-10 with counter (global agent index agent_offset + a as two words, stream, block) and key = seed; streams
 * INIT 0, ACT 1, SAMPLE 2; words handed out as the GA operators' (uniform: 53 bits from two words; below(n): (word * n) >>
 * 32).  Parity with the reference's Mersenne-twister draws is DISTRIBUTIONAL, as for the GA operators.  An agent's results
 * do not depend on the launch geometry, the other agents or how the calls are split over launches.
 * Arithmetic: every float64 operation is rounded on its own (no contraction, no DMMA); every sum runs in index order from
 * its first term (dot products over the input index, then + bias; the loss over samples, then outputs; mean_q over
 * samples), so tests/rl_ref.py restates the kernel bit for bit.  The reference's BLAS order differs in the last bits.
 * Quirks mirrored: bb_upper / bb_middle's forms above; volume capped at 1; the sentiment bonus of _calculate_reward never
 * fires (sentiment is 0.5); HOLD scores 0.05 when |pc| < 0.01, else 0.05 when rsi in [0.4, 0.6], else -0.05, with pc =
 * (next.price_change_1h - 0.5) * 2; no replay until the memory holds a batch, possibly several calls later.
 * agent_state: b200bt_rl_workspace_bytes(A, memory_max) bytes of device memory, zero-filled before the first launch; agent a
 * at a * (that / A): a b200bt_rl_agent_state, the online then the target weights (B200BT_RL_PARAMS doubles each, canonical
 * layout), then memory_max ring words.  agents_host: host [A]; call_end_host: host [n_calls].  Outputs (device):
 * avg_reward [A][n_calls], q_values [A][n_calls][3], history_or_null [A][history_rows][4] = (loss, mean_q, epsilon, step)
 * per replay of this launch, in order (rows past an agent's replays are not written; null skips the loss pass).
 * Checked before the device: null pointers, sizes, symbol in [0, S), batch_size in [1, B200BT_RL_MAX_BATCH], memory_size
 * in [batch_size, memory_max], memory_max <= B200BT_RL_MAX_MEMORY, update_target_every >= 1, every call end in [0, N),
 * points_per_call >= 1, history_rows >= the launch's points, and the agent-state size (EINVAL). */
#define B200BT_RL_FEATURES 16
#define B200BT_RL_PARAMS 1083
#define B200BT_RL_MAX_BATCH 128
#define B200BT_RL_MAX_MEMORY (1 << 20)

typedef struct b200bt_rl_agent {
    uint64_t seed;
    int32_t symbol;
    int32_t batch_size;
    int32_t memory_size;
    int32_t update_target_every;
    double learning_rate;
    double gamma;
    double epsilon_start;
    double epsilon_end;
    double epsilon_decay;
} b200bt_rl_agent;                /* 64 bytes */

typedef struct b200bt_rl_agent_state {
    int64_t initialized;          /* 0 before the first launch (weights drawn or copied then)                           */
    int64_t n_transitions;        /* transitions remembered so far (the deque holds the last min(this, memory_size))    */
    int64_t replays;              /* step_counter                                                                       */
    double epsilon;
    uint64_t act_words;           /* words taken from the ACT and SAMPLE streams                                        */
    uint64_t sample_words;
    double mean_q;                /* of the last replay; NaN before the first                                           */
    int64_t reserved;
} b200bt_rl_agent_state;          /* 64 bytes */

int b200bt_rl_states(const float* cols, const float* close, const float* volume, int64_t ld, int S, int64_t N,
                     int bar_minutes, double* states, b200bt_stream_t stream);
int64_t b200bt_rl_workspace_bytes(int A, int memory_max);
int b200bt_rl_train(const double* states, int S, int64_t N, const b200bt_rl_agent* agents_host, int A, int64_t agent_offset,
                    int memory_max, void* agent_state, int64_t agent_state_bytes, const int64_t* call_end_host, int n_calls,
                    int points_per_call, const double* init_weights_or_null, double* avg_reward, double* q_values,
                    double* history_or_null, int64_t history_rows, b200bt_stream_t stream);

/* ---- volume profile (csrc/volume_profile.cu) ---------------------------------------------------------------------
 * services/utils/volume_profile_analyzer.py, as services/market_monitor_service.py runs it on its df_5m frame (:328-359):
 * analyze_volume_profile (:43-84; _calculate_volume_profile :86-173, _generate_signals :232-316, the inputs of
 * _create_summary :318-394), analyze_volume_delta (:564-684) and detect_volume_anomalies (:487-562), for every frame of W
 * consecutive bars of a market.  The frame ending at bar t is bars t - W + 1 .. t; there is one for every t >= W - 1.
 * Codes index the name tuples of ai_crypto_trader_b200/_lib.py. */
#define B200BT_VP_MAX_BINS 64
#define B200BT_VP_NO_LABEL 255          /* label of a bar without a frame, or of a flat frame (no profile) */
#define B200BT_VP_RECENT 5              /* recent_anomalies: the last five */

typedef struct b200bt_vp_params {
    int32_t num_bins;                /* B, 1 <= B <= B200BT_VP_MAX_BINS (20 in the analyzer)                            */
    int32_t frame_bars;              /* W >= 1 (the monitor's 100 five-minute klines, :170)                               */
    int32_t anomaly_window;          /* rolling window of the anomaly pass, >= 2 (20)                                     */
    int32_t reserved;
    double value_area_pct;           /* 0.7                                                                               */
    double std_threshold;            /* 2.0                                                                               */
} b200bt_vp_params; /* 32 bytes */

typedef struct b200bt_vp_row {
    int32_t n_bars;                  /* W for a frame, 0 for a bar without one (t < W - 1)                                */
    int32_t valid;                   /* 1: price_max > price_min (else the reference fails on int(NaN) and the monitor
                                        publishes no profile; every profile field below is NaN / -1 / 0)                */
    int32_t signal;                  /* overall signal (SIGNALS), B200BT_VP_NO_LABEL without a profile                   */
    int32_t poc_code;                /* POC_CODES                                                                         */
    int32_t value_area_code;         /* VALUE_AREA_CODES                                                                  */
    int32_t at_low_volume_node;      /* a low-volume node within 0.3 % of the close                                       */
    int32_t at_high_volume_node;
    int32_t poc_bin;                 /* np.argmax: the first maximum                                                      */
    int32_t value_area_low_bin, value_area_high_bin;
    int32_t hvn_count, lvn_count;    /* bins >= 0.7 max / <= 0.3 max                                                      */
    int32_t closest_lvn_bin;         /* the low-volume node nearest the close (the first on ties), -1 without one         */
    int32_t pressure;                /* PRESSURES                                                                         */
    int32_t recent_pressure;         /* 0 recent_buying (recent_delta > 0), 1 recent_selling                              */
    int32_t divergence;              /* DIVERGENCES                                                                       */
    int32_t has_momentum;            /* W >= 40                                                                           */
    int32_t anomaly_status;          /* 1: computed; 0: W < anomaly_window (the reference's error dict)                   */
    int32_t total_anomalies;
    int32_t strongest_offset;        /* frame offset (0 .. W-1) of the strongest anomaly (the first on ties), -1: none    */
    int32_t n_recent;                /* min(5, total_anomalies)                                                           */
    int32_t recent_offset[B200BT_VP_RECENT];   /* frame offsets of the last n_recent anomalies, oldest first              */
    int32_t reserved[4];
    double price_min, price_max, close;
    double poc, value_area_low, value_area_high;   /* price levels of those bins                                          */
    double total_volume, max_volume;               /* np.sum of the bins (pairwise); the largest bin                       */
    double hvn_price[3];                           /* the first three high-volume nodes, NaN past hvn_count                */
    double closest_lvn;                            /* NaN without one                                                      */
    double cumulative_delta;                       /* sequential cumsum's last value                                       */
    double net_period_delta, buying_volume, selling_volume;   /* pairwise sums of all / the positive / the negative deltas */
    double buy_sell_ratio;                         /* +inf without selling                                                 */
    double recent_delta;                           /* sum of the last min(20, W) deltas                                    */
    double delta_momentum;                         /* last 20 - the 20 before; NaN when W < 40                             */
    double recent_anomaly_pct;                     /* anomalies among the last min(20, W) bars, in percent                 */
    double strongest_significance, strongest_volume, strongest_ma;
    double recent_ma[B200BT_VP_RECENT], recent_significance[B200BT_VP_RECENT];
} b200bt_vp_row; /* 384 bytes */

/* Volume profile of every frame.  ohlcv: device float32 [5][S][ld] (MarketData's layout), ld >= N; values are widened to
 * float64 and must be finite.  Per frame, in float64 with every operation rounded on its own (no FMA contraction):
 *   profile   min / max of low / high; bin_size = (max - min) / B; candle c covers bins max(0, int((low - min) /
 *             bin_size)) .. min(B - 1, int((high - min) / bin_size)), and volume / bins covered is added to each, in bar
 *             order; edges i * bin_size + min (np.linspace), the last exactly max; level = (edge_i + edge_i+1) / 2.  POC =
 *             the first maximum; value area: bins in descending volume, EQUAL VOLUMES IN DESCENDING BIN INDEX
 *             (np.argsort(v, kind="stable")[::-1]; the reference's unstable argsort leaves this order to the platform),
 *             summed until >= total * value_area_pct.
 *   signals   poc_distance = |c - poc| / c * 100 etc. in the reference's expressions and priority order (:248-314); a
 *             single-bin value area at the close gives 0 / 0 = NaN: inside_value_area_middle.
 *   delta     +volume if close >= open else -volume; sums in numpy's pairwise order (np.sum / Series.sum), the cumulative
 *             delta sequential; divergence from close[-1] - close[-min(20, W)].
 *   anomalies rolling mean (sequential sum / w) and std (two-pass, ddof 1) over w = anomaly_window bars, a bar with frame
 *             offset >= w - 1 is an anomaly if volume > ma + std_threshold * std, significance (volume - ma) / std.
 *             pandas' rolling algorithm differs from this fixed order in the last bits of ma and std.
 * rows_or_null [S][ld_rows] (row t: the frame ending at bar t), bins_or_null [S][ld_rows][B] (the bin volumes; 0 without a
 * profile), labels_or_null uint8 [S][ld_rows] (the overall signal, B200BT_VP_NO_LABEL without a profile); at least one.
 * Checked before the device: null ohlcv / params / all outputs, S < 1, N < 1, ld < N, ld_rows < N, frame_bars < 1,
 * num_bins < 1, anomaly_window < 2, a non-finite value_area_pct or std_threshold (EINVAL); num_bins > B200BT_VP_MAX_BINS,
 * N >= 2^30, S > 65535 (ELIMIT).  One warp per frame; no atomics; deterministic. */
int b200bt_volume_profile(const float* ohlcv, int64_t ld, int S, int64_t N, const b200bt_vp_params* params,
                          b200bt_vp_row* rows_or_null, double* bins_or_null, uint8_t* labels_or_null, int64_t ld_rows,
                          b200bt_stream_t stream);

/* ---- market monitor (csrc/market_monitor.cu) ---------------------------------------------------------------------
 * services/market_monitor_service.py's market_update (:445-465) for every 1-minute bar of a market's history: the
 * technical snapshot of calculate_technical_indicators (:219-301) on the frames of the 1-, 3-, 5- and 15-minute clocks
 * (the monitor's 100 klines each, :168-171), the ticker fields current_price / avg_volume (:432-433), the trading-
 * opportunity test (:561-562), and the fifteen combinations of services/utils/indicator_combinations.py (:96-679) that
 * the monitor adds as combined_indicators (:474-485).  Codes index the name tuples of ai_crypto_trader_b200/_lib.py. */
#define B200BT_MM_NO_LABEL 255          /* label of a row that is not valid, or whose combination is None */
#define B200BT_MM_COMBINATIONS 15
#define B200BT_MM_LABEL_FIELDS 9        /* trend, tma_state, osc_signal, drsi_signal, vpc_confirmation, tsi_direction,
                                           regime, breakout_status, divergence (label_field 0 .. 8)                   */
/* present bits: the keys a market_update dict may lack (volume, ema_12, ema_26 are never set by the monitor) */
#define B200BT_MM_HAS_VOLUME 1
#define B200BT_MM_HAS_EMA_12 2
#define B200BT_MM_HAS_EMA_26 4
#define B200BT_MM_HAS_RSI_3M 8
#define B200BT_MM_HAS_RSI_5M 16
#define B200BT_MM_HAS_PRICE_CHANGE_3M 32
#define B200BT_MM_HAS_AVG_VOLUME 64

typedef struct b200bt_monitor_params {
    int32_t frame_bars;              /* W >= 1: klines per frame on every clock (the monitor's 100)                       */
    int32_t label_field;             /* 0 .. B200BT_MM_LABEL_FIELDS - 1: the categorical field written as the label       */
    double min_price_change_pct;     /* trading_params.min_price_change_pct (0.5)                                         */
    double min_volume_usdc;          /* trading_params.min_volume_usdc                                                    */
} b200bt_monitor_params; /* 24 bytes */

typedef struct b200bt_monitor_row {
    /* snapshot half: market_update's fields */
    int32_t valid;                   /* 1: the 1-, 3- and 5-minute frames are full and a 15-minute kline exists          */
    int32_t trend;                   /* 0 uptrend, 1 downtrend, 2 sideways (any other string in a caller's dict)          */
    int32_t present;                 /* B200BT_MM_HAS_* bits; the history sets rsi_3m, rsi_5m, price_change_3m, avg_volume */
    int32_t opportunity;             /* |price_change_1m| >= min_price_change_pct and avg_volume >= min_volume_usdc      */
    double current_price, avg_volume, rsi, rsi_3m, rsi_5m, stoch_k, macd, macd_3m, macd_5m, williams_r, bb_position,
           trend_strength, price_change_1m, price_change_3m, price_change_5m, price_change_15m;
    double volume, ema_12, ema_26;   /* read only where present                                                           */
    /* combination half: combined_indicators */
    int32_t computed;                /* bit c: combination c (dict order) computed; clear: the reference's None entry    */
    int32_t tma_state;               /* triple_moving_average.state                                                      */
    int32_t osc_signal;              /* oscillator_consensus.signal                                                      */
    int32_t drsi_signal;             /* double_rsi.signal                                                                */
    int32_t vpc_confirmation;        /* volume_price_confirmation.confirmation (neutral: strength is the int 0)          */
    int32_t tsi_direction;           /* trend_strength_index.direction + 1                                               */
    int32_t regime;                  /* market_regime_indicator.regime                                                   */
    int32_t breakout_status;         /* breakout_confirmation.status                                                     */
    int32_t divergence;              /* divergence_detector.divergence                                                   */
    int32_t breakout_direction;      /* breakout_confirmation.direction: -1, 0, 1                                        */
    int32_t reversal_signals;        /* reversal_probability.signals: bit i = name i, appended in bit order              */
    int32_t reserved;
    double trend_confirmation, momentum_trend_alignment, tma_score, volatility_adjusted_momentum, volatility_trend_score,
           osc_strength, osc_agreement, stoch_rsi, drsi_divergence, vwpm, vpc_strength, tsi_strength, tsi_confidence,
           regime_confidence, reversal_probability, breakout_confirmation, divergence_strength;
} b200bt_monitor_row; /* 352 bytes */

/* Market updates of every 1-minute bar.  ohlcv: device float32 [5][S][N] on a 1-minute clock starting at minute0 (Unix
 * minutes, >= 0); ohlcv_3m / _5m / _15m: [5][S][M_k] made from it by b200bt_resample (M_k = b200bt_resample_bars).
 * Row t is the update published at the close of bar t.  Frames: on each clock k the W klines ending at j_k(t), the last
 * kline COMPLETED by the close of t (b200bt_align's rule; j_1(t) = t), so a partial last bucket never enters a frame.
 * In float64 from the widened inputs, every operation rounded on its own (no FMA contraction):
 *   EMAs       pandas' ewm(adjust=False) loop: w = x_0; w = ((1-a) w + a x) / ((1-a) + a) unless w == x; a = 1 / (1 + com)
 *              with com = (1-alpha)/alpha (RSI, alpha = 1/14) or (span-1)/2 (MACD spans 12, 26); outputs before the
 *              window's length are NaN.  RSI's first up / down moves are 0 (diff.where turns the leading NaN into 0).
 *   windows    stochastic %K and Williams %R over 14, Bollinger (20, ddof 0, 2 std), SMA 20 / 50 and the 5-minute SMA 20:
 *              min / max exact; means the sequential sum (oldest first) / w; the variance the two-pass sum of squared
 *              deviations (oldest first) / w.
 *   trend      :262-280; trend_strength = |((c - s20) / s20 * 100) * 0.6 + ((c - s20_5m) / s20_5m * 100) * 0.4|.
 *   ticker     current_price = close[t]; avg_volume = (sequential sum of the volumes of bars max(0, t - 1439) .. t) *
 *              close[t] (the 24-hour ticker's v * c, cut at the series start).
 * A row that is not valid has valid = 0, NaN numeric fields, codes B200BT_MM_NO_LABEL and label B200BT_MM_NO_LABEL.
 * rows_or_null [S][N], labels_or_null uint8 [S][N] (the code of params->label_field); at least one.
 * Checked before the device: null ohlcv / resampled inputs / params / both outputs, S < 1, N < 1, bar_minutes != 1,
 * minute0 < 0, M_k != b200bt_resample_bars(N, minute0, 1, k), frame_bars < 1, label_field outside 0 .. 8 (EINVAL);
 * N >= 2^30, S > 65535 (ELIMIT).  One thread per row; no atomics; deterministic. */
int b200bt_market_monitor(const float* ohlcv, int S, int64_t N, int64_t minute0, int bar_minutes,
                          const float* ohlcv_3m, int64_t M3, const float* ohlcv_5m, int64_t M5, const float* ohlcv_15m,
                          int64_t M15, const b200bt_monitor_params* params, b200bt_monitor_row* rows_or_null,
                          uint8_t* labels_or_null, b200bt_stream_t stream);

/* The combination half of n rows whose snapshot half (valid, trend, present and the numeric fields) the caller filled:
 * calculate_combined_indicators (:56-92) on each row read as a dict of Python floats, through the same device step as
 * b200bt_market_monitor.  round(x, 4) is numpy's rint(x * 1e4) / 1e4 where the reference's value is a numpy float64
 * (np.tanh / np.sign in the expression), else Python's correctly rounded decimal rounding; min / max / comparisons follow
 * Python's NaN behaviour; np.tanh is CUDA's tanh.  Rows with valid == 0 are left as they are.  rows: device; n >= 1
 * (EINVAL), n < 2^31 (ELIMIT). */
int b200bt_indicator_combinations(b200bt_monitor_row* rows, int64_t n, b200bt_stream_t stream);

/* ---- walk-forward evaluation (csrc/walk_forward.cu) -----------------------------------------------------------------
 * The strategy-evolution loop (services/strategy_evolution_service.py:1584-1711) re-fits the deployed parameters and trades
 * them on the bars that follow; a walk-forward analysis scores that loop on history.  A lane of b200bt_sweep_segments trades
 * a list of bar segments, each with its own individual. */

/* Schedules of segments.  A segment is one 24-byte record, bars [start, end) of the series traded by indiv[individual]:
 *     int64_t start;       first bar of the segment                 byte B200BT_SEGMENT_START
 *     int64_t end;         one past its last bar                    byte B200BT_SEGMENT_END
 *     int32_t individual;  row of indiv that trades the segment     byte B200BT_SEGMENT_INDIVIDUAL
 *     int32_t reserved;    0                                        byte B200BT_SEGMENT_RESERVED
 * segments: device array of n_segments such records (8-byte aligned, declared as their int64_t words; host mirror
 * _lib.SEGMENT_DTYPE); seg_begin: device int32 [J + 1]; schedule j (0 <= j < J) is records seg_begin[j] .. seg_begin[j + 1].
 * Lane (j, s) trades schedule j on symbol s.
 *  stats[j][s]  calculate_metrics + _calculate_strategy_score under cfg's score rule (strategy_evaluation.py:32-228,
 *               :579-633) over the concatenation, in segment order, of the records _simulate_trades (:746-878) emits for
 *               indiv[individual] on bars [start, end) of symbol s: the reference function called once per segment, every
 *               segment starting flat and force-closing at end - 1, all segments' records then scored as one list.
 *               Equity, peak, drawdown, calendar-day buckets and the trade hash run on across segments; the position does not.
 *  events       optional [J][S][event_cap] (as b200bt_sweep): the lane's first event_cap event words, with GLOBAL bar indices;
 *               the calendar is the series' own (bar t on day (minute0 + t * bar_minutes) / 1440) and trade_hash is taken
 *               over the lane's records in that order with their global words.
 * Checked on the host, before the device: null pointers, n_indiv < 1, J < 1 and b200bt_sweep's argument checks (EINVAL /
 * ELIMIT: sizes, strides, N < 2^30, the calendar clock, the event buffer); cfg->gap_bar != 0 (EINVAL: a glued series is not
 * combined with segments).
 * Checked on the device, nothing read back: a schedule with no segment, a segment with start < 0, end <= start, end > N
 * or reserved != 0, a segment starting before the previous one ends (gaps are allowed), an individual outside [0, n_indiv) or an individual
 * whose rsi_row lies outside [0, P) makes the schedule invalid: its lanes get n_records = -1 and score = NaN (the rest zero),
 * no events are written for them, and the other lanes are unaffected. */
#define B200BT_SEGMENT_BYTES 24
#define B200BT_SEGMENT_START 0
#define B200BT_SEGMENT_END 8
#define B200BT_SEGMENT_INDIVIDUAL 16
#define B200BT_SEGMENT_RESERVED 20
int b200bt_sweep_segments(const float* price, int64_t ld_price, const float* rsi, int64_t ld_rsi, int P, int S, int64_t N,
                          const b200bt_individual* indiv, int n_indiv, const int64_t* segments, const int32_t* seg_begin,
                          int J, const b200bt_sweep_config* cfg_host, b200bt_lane_stats* stats, uint32_t* events,
                          int64_t event_cap, b200bt_stream_t stream);

/* decode_population (ai_crypto_trader_b200/sweep.py) on the device, byte for byte but for NaN payloads: params is the GA's
 * device float64 matrix [n][ld]; gene_cols_host[6] the columns of rsi_period, rsi_oversold, rsi_overbought, take_profit,
 * stop_loss, max_position_size, -1 = absent (decode_population's defaults 14, 30, 70, 3, 2, 5); period_row_host[n_period_row] the bank
 * row of each period, -1 = not in the bank.  The period is truncated towards zero; one outside the table, or whose entry is
 * -1, decodes to rsi_row = -1 (b200bt_sweep_segments reports such a lane as lost; the host decode raises KeyError).
 * Thresholds are rounded to fp32 towards the side that keeps the compares exact, take_profit / 100, stop_loss / 100,
 * position_size = 10000 * (min(max_position_size, 20) / 100), reserved = 0.  out: device [n].
 * NaN genes: a field decode_population gives as NaN is a NaN here too, but its bits may differ (NumPy keeps the operand's
 * payload, the device's conversion and division need not); every other field, and every field of a row without NaN, is
 * byte for byte.  A NaN or infinite period decodes to rsi_row = -1.
 * Checked before the device: null pointers, n < 1, ld < 1, n_period_row < 1, a column outside [-1, ld) (EINVAL);
 * n_period_row > 256 (ELIMIT). */
int b200bt_decode_individuals(const double* params, int64_t ld, int n, const int* gene_cols_host,
                              const int32_t* period_row_host, int n_period_row, b200bt_individual* out,
                              b200bt_stream_t stream);

/* ---- strategy selection replay (csrc/selection.cu) ------------------------------------------------------------------
 * StrategySelectionService (services/strategy_selection_service.py) run over history: at every check each candidate's
 * metrics snapshot (get_strategy_metrics :159-264, cached per candidate), its six factor scores (:299-687, with
 * market_regime_service.py:734-827), the weighted sum (:821-828), the time adjustments (:689-770), the best candidate
 * (:846) and the switch rule (:884-934).
 *
 * Parameters: a host float64 array [B200BT_SEL_PARAMS] whose slots are named below.  Weights are normalised as :80-83
 * does.  Risk volatility preference: 0 low, 1 medium, 2 high.  The time windows are [start, end) UTC hours. */
#define B200BT_SEL_P_START_BAR 0                /* bar of check 0                                              */
#define B200BT_SEL_P_CHECK_BARS 1               /* bars between checks (STRATEGY_CHECK_INTERVAL / bar seconds) */
#define B200BT_SEL_P_CACHE_EXPIRY 2             /* seconds a snapshot is reused (:128, :174)                   */
#define B200BT_SEL_P_W_MARKET_REGIME 3          /* the normalised weights, in the order of :821-828            */
#define B200BT_SEL_P_W_HISTORICAL_PERFORMANCE 4
#define B200BT_SEL_P_W_RISK_PROFILE 5
#define B200BT_SEL_P_W_SOCIAL_SENTIMENT 6
#define B200BT_SEL_P_W_MARKET_VOLATILITY 7
#define B200BT_SEL_P_W_FEATURE_IMPORTANCE 8
#define B200BT_SEL_P_MIN_IMPROVEMENT 9
#define B200BT_SEL_P_MIN_CONFIDENCE 10
#define B200BT_SEL_P_RISK_MAX_DRAWDOWN 11       /* the risk profile (:96-112)                                  */
#define B200BT_SEL_P_RISK_MIN_SHARPE 12
#define B200BT_SEL_P_RISK_VOLATILITY 13
#define B200BT_SEL_P_HIGH_VOL_START 14          /* time windows (:90-93)                                       */
#define B200BT_SEL_P_HIGH_VOL_END 15
#define B200BT_SEL_P_LOW_ACTIVITY_START 16
#define B200BT_SEL_P_LOW_ACTIVITY_END 17
#define B200BT_SEL_PARAMS 18
/* Genes the scores read, one float64 row [B200BT_SEL_GENES] per candidate; NaN = the key is absent (its .get default). */
#define B200BT_SEL_G_EMA_LONG 0
#define B200BT_SEL_G_TAKE_PROFIT 1
#define B200BT_SEL_G_STOP_LOSS 2
#define B200BT_SEL_G_RSI_OVERSOLD 3
#define B200BT_SEL_G_BOLLINGER_STD 4
#define B200BT_SEL_G_RSI_PERIOD 5
#define B200BT_SEL_G_ATR_MULTIPLIER 6
#define B200BT_SEL_G_ATR_PERIOD 7
#define B200BT_SEL_GENES 8
/* A check row, float64 [B200BT_SEL_ROW_WORDS]: the check's bar and regime label (>= 4: unknown), the best candidate
 * (-1: none valid) and its final score and six factor scores (:862-867), and the active candidate (-1: none) and its
 * score after the switch rule. */
#define B200BT_SEL_R_BAR 0
#define B200BT_SEL_R_REGIME 1
#define B200BT_SEL_R_BEST 2
#define B200BT_SEL_R_SCORE 3
#define B200BT_SEL_R_MARKET_REGIME 4
#define B200BT_SEL_R_HISTORICAL_PERFORMANCE 5
#define B200BT_SEL_R_RISK_PROFILE 6
#define B200BT_SEL_R_SOCIAL_SENTIMENT 7
#define B200BT_SEL_R_MARKET_VOLATILITY 8
#define B200BT_SEL_R_FEATURE_IMPORTANCE 9
#define B200BT_SEL_R_ACTIVE 10
#define B200BT_SEL_R_ACTIVE_SCORE 11
#define B200BT_SEL_ROW_WORDS 12

/* Scores of n_cand candidates at checks c = 0 .. n_checks - 1 (bar t_c = start_bar + c * check_bars), merged into rows.
 * Candidate j is global index cand_index[j] in [0, K) and trades as indiv[cand_row[j]]: its records are the event words of
 * lanes (cand_row[j], s) of a population sweep (lane_stats [n_indiv][S], events [n_indiv][S][event_cap]), merged over the
 * symbols in book order and priced as b200bt_book_metrics prices them.
 *  snapshot    at the candidate's refresh checks: a check with no cached snapshot whose prefix (records with bar <= t_c) is
 *              non-empty, or one at least cache-expiry seconds after the cached fetch; an empty prefix is not cached.  It is
 *              calculate_advanced_metrics(calculate_metrics(prefix)) plus regime_performance (per scored regime with
 *              records: trade_count, win_rate, profit_factor = net / |losses| or 1, and calculate_metrics' sharpe_ratio
 *              and max_drawdown of those records) and hourly_performance (per UTC hour: trade_count, wins = pnl > 0).
 *  scores      regime (the label of bar t_c in row 0 of labels), historical performance, risk, social 0.5, volatility
 *              (0.5 empty, else 0.6), feature importance 0.5; the weighted sum; the time adjustments; a clamp to [0, 1].
 *              float64 in the reference's order of operations, without contraction.
 *  rows        [n_checks][B200BT_SEL_ROW_WORDS]: merge = 0 first fills every row (no best) and zeroes check_locks; merge = 1
 *              merges into the rows of an earlier call over other candidates.  The best is the highest score, the lowest
 *              candidate index among equal ones, whatever the order of calls.  The ACTIVE columns are b200bt_selection_switch's.
 *  scores_or_null  [n_checks][K]: every candidate's final score (NaN for an invalid candidate).
 *  check_locks device int32 [n_checks] workspace.
 * A candidate with a lane whose n_records > event_cap (or a cand_row outside [0, n_indiv)) is invalid: never selected.
 * labels: device uint8 [S or 1][ld_labels] (ld_labels = 0: one row for every symbol; as b200bt_class_stats); a record's
 * regime is the label of its bar in its symbol's row.
 * Checked on the host, before the device: null pointers, the record-pass checks of b200bt_book_metrics (sizes, strides,
 * N < 2^30, the calendar clock; S > 64 is ELIMIT), event_cap < 1, ld_labels, 1 <= n_cand <= K, merge, check_bars not an
 * integer in [1, N], start_bar not an integer in [0, N), cache expiry not positive and finite, a zero risk threshold, a
 * volatility preference outside {0, 1, 2}, non-integer window hours, n_checks outside [1, (N - 1 - start_bar) / check_bars
 * + 1] (EINVAL). */
int b200bt_selection_replay(const float* price, int64_t ld_price, int S, int64_t N, const b200bt_individual* indiv,
                            int n_indiv, const b200bt_sweep_config* cfg, const b200bt_lane_stats* lane_stats,
                            const uint32_t* events, int64_t event_cap, const uint8_t* labels, int64_t ld_labels,
                            const int32_t* cand_row, const int32_t* cand_index, const double* genes, int n_cand, int K,
                            const double* params_host, int64_t n_checks, int merge, double* rows, double* scores_or_null,
                            int32_t* check_locks, b200bt_stream_t stream);

/* The switch rule over the rows in check order, one warp on the device: with (active, active score) starting at (-1, 0),
 * check c switches when its best is >= 0 and differs from the active one, score - active score > MIN_STRATEGY_IMPROVEMENT
 * and score > MIN_STRATEGY_CONFIDENCE; the best then becomes active with its score.  Writes the ACTIVE columns of every
 * row, the checks that switched in order (switch_checks, device int32 [n_checks]) and their count (n_switches, device
 * int32).  params_host: the slots of b200bt_selection_replay.  n_checks < 1 is EINVAL, >= 2^31 ELIMIT. */
int b200bt_selection_switch(double* rows, int64_t n_checks, const double* params_host, int32_t* switch_checks,
                            int32_t* n_switches, b200bt_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200BT_H_ */
