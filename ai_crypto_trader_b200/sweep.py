"""Population-fitness sweep: the GA hot path on the GPU.

Host side of `b200bt_sweep`, `b200bt_sweep_chunked` and `b200bt_sweep_tiled` (include/b200bt.h): three schedules of
the same computation, chosen by `PopulationSweep.plan`.  For every (individual, symbol) lane they evaluate what the
reference evaluates serially in Python:

    trades  = StrategyEvaluationSystem._simulate_trades(id, params, bars)   strategy_evaluation.py:746
    metrics = StrategyPerformanceMetrics.calculate_metrics(trades)          :32
    score   = StrategyEvaluationSystem._calculate_strategy_score(metrics)   :579

and reduces fitness(individual) = mean over symbols of score.  (The
composition simulate -> metrics -> score is the reference's own, see
cross_validate_strategy :682-691; the mean over symbols mirrors its mean over
folds, :1030-1060.)  With aggregation="book" the fitness is instead the score of the
individual's combined multi-symbol trade list (`b200bt_book_metrics`), the list
evaluate_strategy (:528-577) hands to calculate_metrics.

PyTorch is used for device memory and streams only; all arithmetic happens in
the hand-written sm_90a kernels behind the C-ABI.
"""
from __future__ import annotations

import ctypes as C
import inspect
import os
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .population import calendar_days, fitness_callable, unique_rows
from .synth import EPOCH_2024_MINUTES

DEFAULT_GOALS = {  # config.json: evolution.optimization_goals
    "primary": "sharpe_ratio",
    "secondary": ["max_drawdown", "win_rate", "profit_factor"],
}

INDIVIDUAL_DTYPE = np.dtype([("rsi_row", "<i4"), ("rsi_lo", "<f4"), ("rsi_hi", "<f4"), ("reserved", "<i4"),  # b200bt_individual
                             ("take_profit", "<f8"), ("stop_loss", "<f8"), ("position_size", "<f8")])


def _f32_up(x: float) -> np.float32:
    """Smallest float32 >= x."""
    f = np.float32(x)
    return f if float(f) >= x else np.nextafter(f, np.float32(np.inf))


def _f32_down(x: float) -> np.float32:
    """Largest float32 <= x."""
    f = np.float32(x)
    return f if float(f) <= x else np.nextafter(f, np.float32(-np.inf))


class MarketData:
    """Device-resident fp32 OHLCV, field-major SoA [5][S][N] (open, high, low, close, volume).
    `MarketData.from_close(close_dev, ...)` wraps device close prices alone (other fields zero).

    Mirrors the role of HistoricalDataManager.market_data_cache
    (backtesting/data_manager.py:218-220): load once, reuse across calls.

    From a PINNED host tensor only the close prices are uploaded at construction; open / high / low / volume are
    uploaded when first read (`materialise()` forces it), so the source must stay unchanged until then.
    """

    def __init__(self, ohlcv, symbols: Optional[Sequence[str]] = None,
                 minute0: int = EPOCH_2024_MINUTES, bar_minutes: int = 1,
                 device: Optional[torch.device] = None, pinned_source: bool = False):
        if not torch.cuda.is_available():
            raise RuntimeError("MarketData needs a CUDA device (sm_90); this engine has no CPU path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if isinstance(ohlcv, torch.Tensor):
            host = ohlcv
        else:
            host = torch.from_numpy(np.ascontiguousarray(ohlcv, dtype=np.float32))
        if host.dim() != 3 or host.shape[0] != 5:
            raise ValueError("ohlcv must have shape [5][S][N] (open, high, low, close, volume)")
        self.S = int(host.shape[1])
        self.N = int(host.shape[2])
        self._pending_host = None       # pinned source whose open / high / low / volume rows are not on the device yet
        self._close_parts = []
        self.h2d_bytes = 0              # bytes this object has copied host -> device so far
        if host.is_cuda or not host.is_pinned():
            self._ohlcv = host.to(self.device, non_blocking=True).contiguous()
            self.h2d_bytes = 0 if host.is_cuda else host.numel() * 4
        else:
            # pinned host source: only the close prices (all the sweep and the RSI bank read) are uploaded now, in four
            # concurrent quarter copies (one 40 MB copy reaches ~24 GB/s here, four ~33 GB/s: tools/h2d_bandwidth.py);
            # open / high / low / volume follow on first use (the indicator kernels), so a GA generation does not move them
            host = host.contiguous()
            self._ohlcv = torch.empty(host.shape, dtype=torch.float32, device=self.device)
            cur = torch.cuda.current_stream(self.device)
            parts = min(4, self.S)
            lanes = [_copy_stream(self.device, 1 + i) for i in range(parts)]
            rows = [(i * self.S) // parts for i in range(parts + 1)]
            self._close_parts = []      # (row lo, row hi, stream) of the quarter copies the current stream has not joined yet
            for st, lo, hi in zip(lanes, rows[:-1], rows[1:]):
                st.wait_stream(cur)                                          # (allocation order)
                with torch.cuda.stream(st):
                    self._ohlcv[3, lo:hi].copy_(host[3, lo:hi], non_blocking=True)
                self._close_parts.append((lo, hi, st))
            self._pending_host = host
            self.h2d_bytes = self.S * self.N * 4
        self.symbols = list(symbols) if symbols is not None else [f"SYN{i:03d}USDT" for i in range(self.S)]
        self.minute0 = int(minute0)
        self.bar_minutes = int(bar_minutes)

    @classmethod
    def from_close(cls, close: torch.Tensor, minute0: int = EPOCH_2024_MINUTES, bar_minutes: int = 1,
                   symbols: Optional[Sequence[str]] = None) -> "MarketData":
        if not (close.is_cuda and close.dtype == torch.float32 and close.dim() == 2):
            raise ValueError("close must be a device float32 tensor [S][N]")
        ohlcv = torch.zeros((5,) + tuple(close.shape), dtype=torch.float32, device=close.device)
        ohlcv[3] = close
        return cls(ohlcv, symbols=symbols, minute0=minute0, bar_minutes=bar_minutes, device=close.device)

    def materialise(self) -> "MarketData":
        """Make all five fields device-resident now (ordered before later work on the current stream)."""
        self._wait_others()
        self._join_close()
        return self

    def _wait_others(self) -> None:
        """Upload the fields that are still on the host (current stream)."""
        host = self._pending_host
        if host is not None:
            self._pending_host = None
            for f in (0, 1, 2, 4):
                self._ohlcv[f].copy_(host[f], non_blocking=True)
            self.h2d_bytes += 4 * self.S * self.N * 4

    @property
    def ohlcv(self) -> torch.Tensor:
        # all five rows, close included: a reader of the whole array (resample) must not overtake the close copies
        self._wait_others()
        self._join_close()
        return self._ohlcv

    def _join_close(self) -> None:
        """The current stream waits for the quarter copies of the close prices (once)."""
        if self._close_parts:
            cur = torch.cuda.current_stream(self.device)
            for _, _, st in self._close_parts:
                cur.wait_stream(st)
            self._close_parts = []

    @property
    def close(self) -> torch.Tensor:
        self._join_close()
        return self._ohlcv[3]

    @property
    def high(self) -> torch.Tensor:
        return self.ohlcv[1]

    @property
    def low(self) -> torch.Tensor:
        return self.ohlcv[2]

    @property
    def open(self) -> torch.Tensor:
        return self.ohlcv[0]

    @property
    def volume(self) -> torch.Tensor:
        return self.ohlcv[4]


_COPY_STREAMS: Dict[Tuple[int, int], "torch.cuda.Stream"] = {}


def _copy_stream(device: torch.device, which: int = 0) -> "torch.cuda.Stream":
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if (idx, which) not in _COPY_STREAMS:
        _COPY_STREAMS[(idx, which)] = torch.cuda.Stream(device=device)
    return _COPY_STREAMS[(idx, which)]


def rsi_bank(close: torch.Tensor, periods: Sequence[int], fill: bool = True,
             out: Optional[torch.Tensor] = None, zones: Optional[torch.Tensor] = None, zones_symbols: int = 0,
             first_symbol: int = 0) -> torch.Tensor:
    """RSI for every window in `periods`: close [S][N] fp32 -> [S][P][N] fp32.

    ta.momentum.RSIIndicator semantics as used at binance_ml_strategy.py:112.
    `zones`: a sweep zone map (zone_map_floats(P, zones_symbols, N) floats) whose rows of the symbols
    [first_symbol, first_symbol + S) are written in the same pass (b200bt_rsi_bank_zones; needs fill=True).
    A `close` whose bars are not consecutive in memory (a time-strided view) is copied to contiguous rows first.
    """
    if not (close.is_cuda and close.dtype == torch.float32 and close.dim() == 2):
        raise ValueError("close must be a device float32 tensor [S][N]")
    if close.stride(-1) != 1:
        close = close.contiguous()
    S, N = close.shape
    P = len(periods)
    if out is None:
        out = torch.empty((S, P, N), dtype=torch.float32, device=close.device)
    if not (out.device == close.device and out.dtype == torch.float32 and tuple(out.shape) == (S, P, N) and out.is_contiguous()):
        raise ValueError(f"out must be a contiguous float32 tensor [{S}][{P}][{N}] on the device of close")
    arr = (C.c_int * P)(*[int(p) for p in periods])
    with torch.cuda.device(close.device):
        if zones is not None:
            if not fill:
                raise ValueError("zones need fill=True: zone rows describe the NaN-filled bank")
            _lib.call("b200bt_rsi_bank_zones", close.data_ptr(), S, N, _lib.ld(close), arr, P, out.data_ptr(), zones.data_ptr(),
                      int(zones_symbols), int(first_symbol), _lib.current_stream())
        else:
            _lib.call("b200bt_rsi_bank", close.data_ptr(), S, N, _lib.ld(close), arr, P, 1 if fill else 0,
                      out.data_ptr(), _lib.current_stream())
    return out


def decode_population(population: List[Dict], period_row: Dict[int, int], n_timeframes: int = 1) -> np.ndarray:
    """List of GA parameter dicts -> packed b200bt_individual array (numpy structured).

    With `n_timeframes` > 1 the bank holds one block of len(period_row) rows per timeframe and the gene
    `rsi_timeframe` (an index into PopulationSweep.timeframes, default 0 = the base clock) selects the block."""
    out = np.zeros(len(population), dtype=INDIVIDUAL_DTYPE)
    g = lambda key, default: np.array([p.get(key, default) for p in population], dtype=np.float64)
    period = g("rsi_period", 14).astype(np.int64)
    # the table ends one entry (-1) past the bank's largest period: a larger period, however large, decodes to that entry
    rows = np.full(max((w for w in period_row if w >= 0), default=-1) + 2, -1, dtype=np.int64)
    for w, r in period_row.items():
        if w >= 0:
            rows[w] = r
    row = rows[np.clip(period, 0, len(rows) - 1)]
    if len(period) and (period.min() < 0 or row.min() < 0):
        bad = int(period[(row < 0) | (period < 0)][0])
        raise KeyError(f"rsi_period {bad} is not in the RSI bank {sorted(period_row)}")
    if n_timeframes > 1:
        tf = g("rsi_timeframe", 0).astype(np.int64)
        if len(tf) and (tf.min() < 0 or tf.max() >= n_timeframes):
            raise KeyError(f"rsi_timeframe {int(tf[(tf < 0) | (tf >= n_timeframes)][0])} is not an index into the {n_timeframes} timeframes of the bank")
        row = row + tf * len(period_row)
    out["rsi_row"] = row
    # thresholds rounded towards the side that keeps `rsi < oversold` / `rsi > overbought` exact in fp32
    lo, hi = g("rsi_oversold", 30), g("rsi_overbought", 70)
    lo32, hi32 = lo.astype(np.float32), hi.astype(np.float32)
    out["rsi_lo"] = np.where(lo32.astype(np.float64) >= lo, lo32, np.nextafter(lo32, np.float32(np.inf)))
    out["rsi_hi"] = np.where(hi32.astype(np.float64) <= hi, hi32, np.nextafter(hi32, np.float32(-np.inf)))
    # strategy_evaluation.py:762-764, :773-774 (same float64 expressions)
    out["take_profit"] = g("take_profit", 3) / 100
    out["stop_loss"] = g("stop_loss", 2) / 100
    out["position_size"] = 10000 * (np.minimum(g("max_position_size", 5), 20) / 100)
    return out


def lane_cost(p: Dict) -> float:
    """Fraction of bars on which RSI(w) sits outside [oversold, overbought] under the model
    RSI(w) ~ N(50, 44/sqrt(w)): the lane's trade-event rate is proportional to it (measured on the
    synthetic 1-minute data: events ~= 0.27 * cost * bars).  Scheduling only; never affects results."""
    from math import erf, sqrt
    w = int(p.get("rsi_period", 14))
    sd = 44.0 / sqrt(max(w, 1))
    phi = lambda x: 0.5 * (1.0 + erf(x / sqrt(2.0)))
    return phi((float(p.get("rsi_oversold", 30)) - 50.0) / sd) + 1.0 - phi((float(p.get("rsi_overbought", 70)) - 50.0) / sd)


EVENTS_PER_COST_BAR = 0.27


def predicted_events(population: List[Dict], n_bars: int) -> np.ndarray:
    """Expected trade records per (individual, symbol) lane under the lane_cost model."""
    return EVENTS_PER_COST_BAR * lane_costs(population) * n_bars


def _band_costs(period: np.ndarray, oversold: np.ndarray, overbought: np.ndarray) -> np.ndarray:
    """lane_cost's band model on arrays of RSI windows and float64 thresholds."""
    from scipy.special import ndtr
    sd = 44.0 / np.sqrt(np.maximum(period, 1))
    return ndtr((oversold - 50.0) / sd) + 1.0 - ndtr((overbought - 50.0) / sd)


def lane_costs(population: List[Dict]) -> np.ndarray:
    """lane_cost for a whole population (vectorised)."""
    g = lambda key, default: np.array([float(p.get(key, default)) for p in population], dtype=np.float64)
    return _band_costs(g("rsi_period", 14).astype(np.int64), g("rsi_oversold", 30), g("rsi_overbought", 70))


def _duplicate_classes(packed: np.ndarray):
    """(first index of each distinct record, class of every record) of decoded records, in population order, or None
    when all records are distinct (population.unique_rows)."""
    keep, expand = unique_rows(packed)
    return None if expand is None else (keep, expand)


def costs_from_packed(packed: np.ndarray, periods: Sequence[int], timeframes: Sequence[int] = (1,)) -> np.ndarray:
    """lane_cost of already decoded individuals (b200bt_individual records): no second pass over the dicts.  An RSI row
    of a k-times slower clock changes every k bars: its threshold crossings (events) are rarer by about sqrt(k)."""
    P = len(periods)
    w = np.asarray(periods, dtype=np.float64)[packed["rsi_row"] % P]
    c = _band_costs(w, packed["rsi_lo"].astype(np.float64), packed["rsi_hi"].astype(np.float64))
    if len(timeframes) > 1:
        k = np.asarray(timeframes, dtype=np.float64)[packed["rsi_row"] // P] / float(timeframes[0])
        c = c / np.sqrt(k)
    return c


_SM_COUNT: Dict[int, int] = {}


def _sm_count(device) -> int:
    idx = torch.device(device).index
    idx = torch.cuda.current_device() if idx is None else idx
    if idx not in _SM_COUNT:
        _SM_COUNT[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SM_COUNT[idx]


_PINNED_FLAGS = None
_FLAG_SLOTS = 256


def _pinned_flags() -> torch.Tensor:
    """Pinned int32 [256][5]: per plan (slice) of a sweep, [0] = the event pool overflowed, [1] = lanes that went through
    the exact fallback, [2] = pool blocks handed out, [3] = scan tiles that timed out, [4] = time chunks that set a new
    equity peak.  The kernels' flags are copied here asynchronously; the host looks at them only after a stream
    synchronisation it does anyway (page-locking memory is slow: one table shared by every plan)."""
    global _PINNED_FLAGS
    if _PINNED_FLAGS is None:
        _PINNED_FLAGS = torch.zeros((_FLAG_SLOTS, 5), dtype=torch.int32).pin_memory()
    return _PINNED_FLAGS


_NEXT_FLAG = [0]


def _flag_slot() -> torch.Tensor:
    i = _NEXT_FLAG[0] = (_NEXT_FLAG[0] + 1) % _FLAG_SLOTS
    return _pinned_flags()[i]


class _Plan:
    """What the plans of both time-chunked schedules share.  A plan covers the slice [lo, lo + pop) of the caller's
    population (individual indices inside it are slice-relative); `pred` = predicted_events of that slice when the caller
    already has it.  A plan sizes its workspace (`ws_bytes`); _allocate_plans gives it its device buffers."""

    def _start(self, population: List[Dict], n_bars: int, lo: int, pred: Optional[np.ndarray]) -> np.ndarray:
        self.lo, self.pop = int(lo), len(population)
        self.workspace = self.invalid = self.overflow = None
        return predicted_events(population, n_bars) if pred is None else np.asarray(pred, dtype=np.float64)

    def _size_pool(self, pred: np.ndarray, n_symbols: int, pool_scale: float, pool_blocks: Optional[int]) -> None:
        """Event pool in blocks of 256 events, once n_seg is known."""
        self.pred_blocks = float(pred.sum()) * n_symbols / 256
        # every segment owns at least one block, and a repaired segment abandons its first chain
        self.pool_blocks = (int(pool_scale * self.pred_blocks) + 2 * self.n_seg * n_symbols + 1024 if pool_blocks is None
                            else int(pool_blocks))


def _allocate_plans(plans: List[_Plan], n_symbols: int, device) -> List[_Plan]:
    """The device buffers of the plans of one call: one workspace, of the largest size any of them needs (their slices run
    one after the other on the same stream), then every plan's lane fallback flags and pinned flag row."""
    # keep this order: with the small buffers allocated before the workspace, the same lane_scan_kernel took 1.3 % longer
    # on the configs[1] workload (H100 80GB HBM3, 400 W power limit), from where the allocations landed in device memory
    shared = torch.empty(max(pl.ws_bytes for pl in plans), dtype=torch.uint8, device=device)
    for pl in plans:
        pl.workspace = shared
        pl.invalid = torch.zeros((pl.pop, n_symbols), dtype=torch.uint8, device=device)
        pl.overflow = _flag_slot()
    return plans


class ChunkPlan(_Plan):
    """Host-side plan of the time-chunked sweep for one population slice (device tensors inside)."""

    def __init__(self, population: List[Dict], n_bars: int, n_symbols: int, device, target_events: int = 16384,
                 warm: int = 8192, max_chunks: int = 64, pool_scale: float = 1.5, pool_blocks: Optional[int] = None,
                 max_repair_rounds: int = 8, lo: int = 0, pred: Optional[np.ndarray] = None):
        pred = self._start(population, n_bars, lo, pred)
        kmax = max(1, min(max_chunks, n_bars // max(8 * warm, 2048)))
        k = np.clip(np.ceil(pred / target_events), 1, kmax).astype(np.int32)
        self.n_chunks = k
        self.seg_base = np.concatenate([[0], np.cumsum(k)[:-1]]).astype(np.int32)
        self.n_seg = int(k.sum())
        items = np.zeros((self.n_seg, 4), dtype=np.int32)
        # most expensive work first (per-chunk cost), keeping one individual's chunks together
        per_chunk = pred / k
        row = 0
        for i in sorted(range(self.pop), key=lambda j: (-per_chunk[j], int(population[j].get("rsi_period", 14)))):
            for c in range(int(k[i])):
                items[row] = (i, c, k[i], self.seg_base[i] + c)
                row += 1
        self.warm = int(warm)
        self.max_repair_rounds = int(max_repair_rounds)
        self._size_pool(pred, n_symbols, pool_scale, pool_blocks)
        self.items = torch.from_numpy(items).to(device)
        self.seg_base_dev = torch.from_numpy(self.seg_base).to(device)
        self.n_chunks_dev = torch.from_numpy(self.n_chunks).to(device)
        self.ws_bytes = int(_lib.load().b200bt_sweep_chunked_workspace_bytes(self.pool_blocks, n_symbols, self.n_seg))

    def launch(self, sweep: "PopulationSweep", data: tuple, indiv: int, stats: torch.Tensor,
               events: Optional[torch.Tensor], event_cap: int, stream) -> None:
        """b200bt_sweep_chunked on this slice: `data` = PopulationSweep._data_args(), `indiv` = address of the slice's first
        record, `stats` / `events` = the slice's rows."""
        _lib.call("b200bt_sweep_chunked", *data, indiv, None, self.pop, self.items.data_ptr(), self.n_seg,
                  self.seg_base_dev.data_ptr(), self.n_chunks_dev.data_ptr(), self.n_seg, self.warm, self.max_repair_rounds,
                  self.pool_blocks, self.workspace.data_ptr(), self.workspace.numel(), C.byref(sweep.cfg), stats.data_ptr(),
                  _lib.ptr(events), event_cap, self.invalid.data_ptr(), self.overflow.data_ptr(), stream)


class TilePlan(_Plan):
    """Host-side plan of the thread-per-lane sweep (b200bt_sweep_tiled) for one population slice: every
    individual gets the same K time chunks, chosen so that the CTAs fill whole waves of the GPU."""

    THREADS = int(os.environ.get("B200BT_LS_THREADS", 256))     # individuals per CTA (csrc/sweep_chunked.cu LS_THREADS)
    CTAS_PER_SM = int(os.environ.get("B200BT_LS_CTAS", 3))     # resident CTAs of lane_scan_kernel per SM (__launch_bounds__(256, 3))
    WARM = 1536          # warm-up bars of a speculative chunk

    @classmethod
    def chunks_for(cls, pop: int, n_bars: int, n_symbols: int, device, warm: int = WARM, max_chunks: int = 64,
                   n_slots: Optional[int] = None) -> int:
        """About 2.5 work items per resident warp slot (the scan is persistent: warps take (warp-slot, chunk, symbol) items
        from a counter, the most expensive first; more chunks balance better but every chunk pays its warm-up and its share of
        the per-chunk metrics overhead), chunks at least 3 warm-ups long.  Measured on configs[1] (3 CTAs/SM): a plateau of
        7.15-7.25 ms for K = 26..30 and warm-ups of 1024..3072 bars; K = 34 +0.3 ms, K = 24 +0.15 ms.  A short warm-up is
        affordable because a mis-speculated chunk is re-scanned only until it meets its recorded trajectory again
        (chunk_scan_item, REPAIR): at 2048 bars ~10 % of the chunks start in the wrong state and take ~3500 bars each to come
        back (at 8192 bars: 2 % and ~7700 bars)."""
        kmax = max(1, min(max_chunks, n_bars // max(3 * warm, 2048)))
        slots = _sm_count(device) * cls.CTAS_PER_SM
        groups = -(-(n_slots if n_slots is not None else pop) // cls.THREADS) * n_symbols
        return min(kmax, max(1, round(2.5 * slots / groups)))

    def __init__(self, population: List[Dict], n_bars: int, n_symbols: int, device, warm: int = WARM,
                 max_chunks: int = 64, chunks: Optional[int] = None, pool_scale: float = 1.5,
                 pool_blocks: Optional[int] = None, max_repair_rounds: Optional[int] = None, lo: int = 0,
                 order_by: str = "row_cost", pred: Optional[np.ndarray] = None, rows: Optional[np.ndarray] = None):
        pred = self._start(population, n_bars, lo, pred)
        self.warm = int(warm)
        # thread slots: 32 consecutive slots = one warp, which stages its own tiles and may read two distinct RSI rows
        self.slots = pack_warps(population, pred, order_by, rows)
        if chunks is None:
            chunks = self.chunks_for(self.pop, n_bars, n_symbols, device, warm, max_chunks, n_slots=len(self.slots))
        self.K = int(chunks)
        # 0 = no repair, 1 = the bounded pass on the critical path, 2 = that and the unbounded pass beside the metrics
        self.max_repair_rounds = int(max_repair_rounds) if max_repair_rounds is not None else 2
        self.n_seg = self.pop * self.K
        self._size_pool(pred, n_symbols, pool_scale, pool_blocks)
        self.order = np.ascontiguousarray(self.slots[self.slots >= 0])      # individuals in dispatch order
        self.slots_dev = torch.from_numpy(np.concatenate([self.slots, self.order])).to(device)     # [slots | order]
        self.ws_bytes = int(_lib.load().b200bt_sweep_tiled_workspace_bytes(self.pool_blocks, n_symbols, self.pop, self.K))

    def launch(self, sweep: "PopulationSweep", data: tuple, indiv: int, stats: torch.Tensor,
               events: Optional[torch.Tensor], event_cap: int, stream) -> None:
        """b200bt_sweep_tiled on this slice (arguments as ChunkPlan.launch)."""
        n_slots = len(self.slots)
        _lib.call("b200bt_sweep_tiled", *data, _lib.ptr(sweep._zones_if_amortised()), indiv, self.slots_dev.data_ptr(),
                  n_slots, self.slots_dev.data_ptr() + 4 * n_slots, self.pop, self.K, self.warm, self.max_repair_rounds,
                  self.pool_blocks, self.workspace.data_ptr(), self.workspace.numel(), C.byref(sweep.cfg), stats.data_ptr(),
                  _lib.ptr(events), event_cap, self.invalid.data_ptr(), self.overflow.data_ptr(), stream)


WARP_RSI_ROWS = 2       # distinct RSI rows the machines of one warp may read (csrc/sweep_chunked.cu LS_RSI_ROWS)


def pack_warps(population: List[Dict], pred: np.ndarray, order_by: str = "row_cost", rows: Optional[np.ndarray] = None) -> np.ndarray:
    """Thread slots of the thread-per-lane scan: int32[n_warps * 32], the individual each slot runs, -1 = empty.

    A warp stages the price row and the RSI rows of its own 32 machines, at most WARP_RSI_ROWS of them, and its cost is
    the UNION of its machines' events.  So individuals are sorted by (RSI row, predicted cost) -- neighbours read the same
    row and fire at similar rates on the same bars -- and cut into warps that never span more than WARP_RSI_ROWS rows (a
    row's tail shares a warp with the head of the next row; slots stay empty only where a third row would enter).  Warps
    are then dispatched most expensive first, so that the warps resident together (and the 8 of a CTA) cost the same.
    order_by = "identity" keeps the population order (testing: warps that break the row rule are re-run by the exact
    fallback), "row_thresholds" sorts a row by (oversold, overbought) instead of cost.  `rows`: the bank row of every
    individual when it is not a function of `rsi_period` alone (several timeframes)."""
    n = len(population)
    if order_by == "identity":
        out = np.full(-(-n // 32) * 32, -1, dtype=np.int32)
        out[:n] = np.arange(n, dtype=np.int32)
        return out
    g = lambda key, default: np.array([float(p.get(key, default)) for p in population], dtype=np.float64)
    row = g("rsi_period", 14).astype(np.int64) if rows is None else np.asarray(rows, dtype=np.int64)    # (bank row when given)
    pred = np.asarray(pred, dtype=np.float64)
    rows, inv = np.unique(row, return_inverse=True)
    mean_cost = np.bincount(inv, weights=pred) / np.maximum(np.bincount(inv), 1)
    if order_by == "row_thresholds":
        idx = np.lexsort((np.arange(n), -g("rsi_overbought", 70), g("rsi_oversold", 30), -mean_cost[inv]))
    else:
        idx = np.lexsort((np.arange(n), -pred, -mean_cost[inv]))          # rows by mean cost, inside a row by cost
    counts = np.bincount(inv, minlength=len(rows))[np.argsort(-mean_cost, kind="stable")]    # members per row, in dispatch order
    warps, fill, used, pos = [], 0, 0, 0
    cur = np.full(32, -1, dtype=np.int32)
    for cnt in counts:
        left = int(cnt)
        while left:
            if fill == 32 or (fill and used == WARP_RSI_ROWS):
                warps.append(cur)
                cur, fill, used = np.full(32, -1, dtype=np.int32), 0, 0
            take = min(32 - fill, left)
            cur[fill:fill + take] = idx[pos:pos + take]
            fill, used, pos, left = fill + take, used + 1, pos + take, left - take
    if fill:
        warps.append(cur)
    warps = np.stack(warps)
    cost = np.where(warps >= 0, pred[np.maximum(warps, 0)], 0.0).sum(axis=1)
    return np.ascontiguousarray(warps[np.argsort(-cost, kind="stable")]).reshape(-1)


def evaluation_order(population: List[Dict]) -> np.ndarray:
    """Order in which the kernel dispatches individuals: same RSI period adjacent (the
    warps of a CTA then read the same RSI stream), most expensive first.

    Cost model: a lane's work is dominated by its trade events, whose rate follows the
    fraction of time RSI(w) spends outside [oversold, overbought]; RSI(w) is roughly
    N(50, 44/sqrt(w)) on 1-minute data.  Only scheduling depends on this, never results.
    """
    period = np.array([int(p.get("rsi_period", 14)) for p in population], dtype=np.int64)
    return np.lexsort((np.arange(len(population)), -lane_costs(population), period)).astype(np.int32)


BOOK_MAX_SYMBOLS = 64                  # b200bt_book_metrics: one 64-bit symbol mask per bar
# Event buffers of one book slice: 24 GiB holds configs[1] (1024 individuals x 10 symbols) unsliced up to 629 k records in
# its busiest lane (of 1M bars), beside the sweep's own event pool (plan_batches' 8 GiB), on an 80 GB H100.
BOOK_MAX_EVENT_BYTES = 24 << 30
BOOK_CAP_HEADROOM = 4                  # a learnt event cap is the last busiest lane + 1/4


def _stats_fields(raw: np.ndarray) -> Dict[str, np.ndarray]:
    """Stats records float64 [...][LANE_STATS_WORDS] (b200bt_lane_stats) as dict field -> [...] array, trade_hash as uint64."""
    out = {name: raw[..., i] for i, name in enumerate(_lib.LANE_STATS_FIELDS[:-1])}
    out["trade_hash"] = np.ascontiguousarray(raw[..., _lib.LANE_STATS_WORDS - 1]).view(np.uint64)
    return out


class PopulationSweep:
    """Evaluate a GA population against device-resident market data.

    `sweep.fitness_function` is a callable usable as GeneticAlgorithm's
    `fitness_function`; it carries a `.batch` attribute that evaluates the whole
    population in one kernel launch (see genetic_algorithm.GeneticAlgorithm).
    """

    def __init__(self, market: MarketData, rsi_periods: Iterable[int] = range(5, 31),
                 optimization_goals: Optional[Dict] = None, initial_capital: float = 10000.0,
                 event_cap: int = 0, mode: str = "auto", chunk_options: Optional[Dict] = None,
                 score_on_advanced: bool = False, timeframes: Sequence[int] = (), aggregation: str = "mean",
                 max_event_bytes: Optional[int] = None):
        """score_on_advanced: take the strategy score on calculate_advanced_metrics' dict (the composition of
        evaluate_strategy, strategy_evaluation.py:545-557: `expectancy`, `sortino_ratio`, ... exist as keys) instead of the
        plain calculate_metrics dict (cross_validate_strategy :683-691, the default).
        mode: "fused" (one warp per lane, serial in time), "chunked" (expensive lanes split into verified
        time chunks, one warp per chunk), "tiled" (every lane split into the same K verified chunks, one THREAD
        per chunk; csrc/sweep_chunked.cu) or "auto" (tiled from 131072 bars up, fused below).
        aggregation: how evaluate() turns an individual's symbols into one fitness: "mean" = the mean over symbols of the
        per-symbol scores, "book" = the score of the book, the individual's records on every symbol in one trade list
        (evaluate_strategy's composition, strategy_evaluation.py:528-577; see book_stats()).
        max_event_bytes: budget of the event buffers of a book evaluation (default BOOK_MAX_EVENT_BYTES); a population whose
        buffers exceed it is swept and booked in slices."""
        self._setup(market, sorted(set(int(p) for p in rsi_periods)), optimization_goals, initial_capital, event_cap, mode,
                    chunk_options, score_on_advanced, timeframes, aggregation=aggregation, max_event_bytes=max_event_bytes)

    def _setup(self, market: MarketData, periods: List[int], optimization_goals: Optional[Dict], initial_capital: float,
               event_cap: int, mode: str, chunk_options: Optional[Dict], score_on_advanced: bool, timeframes: Sequence[int],
               bank: Optional[torch.Tensor] = None, aggregation: str = "mean", max_event_bytes: Optional[int] = None) -> None:
        """The initialisation of both constructors: `periods` in bank-row order, `bank` = None computes the bank."""
        if aggregation not in ("mean", "book"):
            raise ValueError(f"aggregation must be 'mean' or 'book', not {aggregation!r}")
        if aggregation == "book" and market.S > BOOK_MAX_SYMBOLS:
            raise ValueError(f"aggregation='book' handles at most {BOOK_MAX_SYMBOLS} symbols ({market.S} given)")
        self.aggregation = aggregation
        self.max_event_bytes = int(BOOK_MAX_EVENT_BYTES if max_event_bytes is None else max_event_bytes)
        self._book_cap = 0                     # event_cap learnt from the previous book evaluation (0: count first)
        self._book = None                      # book stats [pop][20] float64 of the last book evaluation (host)
        self._book_dev = None                  # the same stats of its unique individuals, on the device
        self.book_resweeps = 0                 # slices of the last book evaluation swept again with the exact cap
        self.last_event_bytes = 0              # largest event buffer of the last book evaluation
        self.market = market
        self.periods = periods
        self.period_row = {p: i for i, p in enumerate(self.periods)}
        goals = optimization_goals or DEFAULT_GOALS
        primary, mask = _lib.score_codes(goals, advanced=score_on_advanced)
        self.cfg = _lib.SweepConfig(initial_capital=float(initial_capital), minute0=market.minute0,
                                    bar_minutes=market.bar_minutes, primary=primary, secondary_mask=mask, variant=0)
        self.event_cap = int(event_cap)
        # timeframes (minutes per bar, the first one = the market's own clock): BASELINE configs[3] evaluates the RSI rule on
        # 1m / 5m / 15m indicators (recipe: services/market_monitor_service.py:219-301); the bank then holds one block of rows
        # per timeframe, each higher-timeframe RSI brought back to the base clock by "last completed bar", and the gene
        # `rsi_timeframe` (index into `timeframes`) selects the block
        self.timeframes = tuple(int(k) for k in timeframes) or (market.bar_minutes,)
        if self.timeframes[0] != market.bar_minutes or any(k % market.bar_minutes for k in self.timeframes):
            raise ValueError("timeframes must start with the market's own bar spacing and be multiples of it")
        self.mode, self.chunk_min_bars, self.chunk_options = mode, 131072, dict(chunk_options or {})
        self._zones = None             # zone map of the bank: made with a computed one-clock bank, else on first use
        if bank is not None:
            self.bank = bank
        elif len(self.timeframes) == 1:
            self.bank, self._zones = self._bank_behind_the_upload(market)
        else:
            self.bank = self._multi_timeframe_bank(market)
        self._stats = self._events = None      # lane stats / event words of the last evaluation (_buffers)
        self._buffer_key = None                # (pop, event_cap) they were allocated for
        self._inverse = None                   # last evaluate(): its population -> row of its unique individuals
        self._last_plans = []                  # plans of the last evaluation, whose pinned flags _flags reads
        self._pool_factor = 1.0                # event-pool scale learnt from earlier sweeps (_pool_options)
        self._tiled_sweeps = 0                 # thread-per-lane slices swept so far (_zones_if_amortised)
        self._pinned_in = self._pinned_out = None
        self.last_unique = self.h2d_bytes = self.d2h_bytes = 0      # of the last evaluate()

    def _bank_behind_the_upload(self, market: MarketData) -> Tuple[torch.Tensor, torch.Tensor]:
        """RSI bank of the market and its zone map.  While the close prices are still arriving in quarter copies (MarketData
        from a pinned host tensor), each quarter's rows are computed on that quarter's copy stream, so the bank is ready one
        quarter of its kernel time after the last byte instead of one whole kernel."""
        parts = market._close_parts
        P = len(self.periods)
        # the zone map of the bank (ranges of every 32-bar block and 4-bar group) comes out of the same pass
        zones = torch.empty(int(_lib.load().b200bt_zone_map_floats(P, market.S, market.N)), dtype=torch.float32, device=market.device)
        if not parts:
            return rsi_bank(market.close, self.periods, zones=zones, zones_symbols=market.S), zones
        bank = torch.empty((market.S, P, market.N), dtype=torch.float32, device=market.device)
        cur = torch.cuda.current_stream(market.device)
        for lo, hi, st in parts:
            st.wait_stream(cur)                        # (the allocations of the bank and of the zone map)
            with torch.cuda.stream(st):
                rsi_bank(market._ohlcv[3, lo:hi], self.periods, out=bank[lo:hi], zones=zones, zones_symbols=market.S, first_symbol=lo)
        market._join_close()                           # the current stream now waits for copies AND bank rows
        return bank, zones

    def _multi_timeframe_bank(self, market: MarketData) -> torch.Tensor:
        """[S][T * P][N] bank: block 0 = RSI of the base clock, block i = RSI of the clock-aligned timeframes[i]-minute bars
        (b200bt_resample), NaN policy applied on that clock like the reference's analyzer does per kline series, then aligned
        to the base clock with the value of the last COMPLETED higher-timeframe bar (b200bt_align: no look-ahead; NaN before
        the first completed bar, where no threshold compare is true)."""
        from . import indicators as ind
        P, T = len(self.periods), len(self.timeframes)
        bank = torch.empty((market.S, T * P, market.N), dtype=torch.float32, device=market.device)
        bank[:, :P] = rsi_bank(market.close, self.periods)
        for i, k in enumerate(self.timeframes[1:], start=1):
            hi = ind.resample(market, k)
            rows = rsi_bank(hi.close, self.periods)                                        # [S][P][M]
            aligned = ind.align_to_base(rows.view(market.S * P, hi.N), market, k)          # [S * P][N]
            bank[:, i * P:(i + 1) * P] = aligned.view(market.S, P, market.N)
            del hi, rows, aligned
        return bank

    @classmethod
    def from_bank(cls, market: MarketData, bank: torch.Tensor, periods, optimization_goals=None,
                  initial_capital: float = 10000.0, event_cap: int = 0, mode: str = "fused",
                  score_on_advanced: bool = False, aggregation: str = "mean",
                  max_event_bytes: Optional[int] = None) -> "PopulationSweep":
        """Sweep over a caller-supplied RSI bank [S][P][N] (e.g. the 'rsi' field of the reference's
        market-data points) instead of one computed from the close prices."""
        periods = [int(p) for p in periods]
        if not (bank.is_cuda and bank.dtype == torch.float32 and tuple(bank.shape) == (market.S, len(periods), market.N)):
            raise ValueError(f"bank must be a device float32 tensor [{market.S}][{len(periods)}][{market.N}]")
        self = cls.__new__(cls)
        self._setup(market, periods, optimization_goals, initial_capital, event_cap, mode, None, score_on_advanced, (),
                    bank=bank.contiguous(), aggregation=aggregation, max_event_bytes=max_event_bytes)
        return self

    # -- device-side evaluation (inputs already resident) -------------------
    def evaluate_device(self, indiv_dev: torch.Tensor, order_dev: Optional[torch.Tensor], pop: int,
                        fitness_dev: torch.Tensor, plan: Optional[List[_Plan]] = None,
                        event_cap: Optional[int] = None) -> None:
        """Sweep + fitness reduction on the current stream.  Without a plan the fused kernel runs (in `order_dev` order);
        with the TilePlan / ChunkPlan slices of `plan` the time-chunked kernels run, and lanes whose chunk boundaries failed
        verification go through the fused kernel inside the same call.  `event_cap`: event words kept per lane (default:
        the instance's)."""
        m = self.market
        cap = self.event_cap if event_cap is None else int(event_cap)
        stats, events = self._buffers(pop, cap)
        self._inverse = None
        self._last_plans = [] if plan is None else plan if isinstance(plan, (list, tuple)) else [plan]
        with torch.cuda.device(m.device):
            st = _lib.current_stream()
            data = self._data_args()
            if plan is None:
                _lib.call("b200bt_sweep", *data, indiv_dev.data_ptr(), _lib.ptr(order_dev), pop, C.byref(self.cfg),
                          stats.data_ptr(), _lib.ptr(events), cap, st)
            for pl in self._last_plans:
                part = slice(pl.lo, pl.lo + pl.pop)
                pl.launch(self, data, indiv_dev.data_ptr() + pl.lo * C.sizeof(_lib.Individual), stats[part],
                          None if events is None else events[part], cap, st)
            _lib.call("b200bt_fitness_reduce", stats.data_ptr(), pop, m.S, fitness_dev.data_ptr(), st)

    def _data_args(self) -> tuple:
        """The leading arguments of every sweep entry point: price rows, RSI bank, P, S, N."""
        m = self.market
        return (m.close.data_ptr(), _lib.ld(m.close), self.bank.data_ptr(), _lib.ld(self.bank), self.bank.shape[1], m.S, m.N)

    def _buffers(self, pop: int, event_cap: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """Lane stats [pop][S] and event words [pop][S][event_cap] of an evaluation, kept while pop and event_cap stay."""
        if self._buffer_key != (pop, event_cap):
            m = self.market
            self._stats = torch.empty((pop, m.S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=m.device)
            self._events = torch.zeros((pop, m.S, event_cap), dtype=torch.int32, device=m.device) if event_cap else None
            self._buffer_key = (pop, event_cap)
        return self._stats, self._events

    # Lanes the time-chunked kernels flagged (a boundary still inconsistent after the repair passes, a full event pool, a warp
    # not packed for the thread-per-lane scan) are re-evaluated by the fused kernel ON THE DEVICE, inside b200bt_sweep_chunked /
    # b200bt_sweep_tiled: an evaluation reads nothing back.  _flags looks at the flags of the last evaluation afterwards.
    def _flags(self) -> Tuple[np.ndarray, int, float]:
        """After synchronising the stream: the last evaluation's int[5] flags (_pinned_flags) summed over its plans, the
        pool blocks they used net of the 2 * n_seg * S floor of _Plan._size_pool, and the blocks their cost model predicted."""
        torch.cuda.current_stream(self.market.device).synchronize()
        flags = np.zeros(5, dtype=np.int64)
        used, predicted = 0, 0
        for pl in self._last_plans:
            f = pl.overflow.numpy()
            flags += f
            used += int(f[2]) - 2 * pl.n_seg * self.market.S
            predicted += pl.pred_blocks
        return flags, used, predicted

    @property
    def last_invalid_lanes(self) -> int:
        """(individual, symbol) lanes of the last evaluation that went through the exact fallback."""
        return int(self._flags()[0][1])

    @property
    def last_scan_stalls(self) -> int:
        """Tiles of the last thread-per-lane scan whose bulk copy did not complete in time (their chunks were re-scanned by the
        repair pass or their lanes re-run by the exact fallback; 0 in normal operation)."""
        return int(self._flags()[0][3])

    @property
    def last_peak_chunks(self) -> int:
        """(individual, symbol, chunk) time chunks of the last time-chunked evaluation that set a new equity peak: only those
        take the record-by-record drawdown pass (chunk_peak_kernel); the others' drawdown comes from three per-chunk sums."""
        return int(self._flags()[0][4])

    @property
    def last_pool_overflow(self) -> bool:
        """The event pool of the last evaluation was too small (its lanes were re-run exactly; the next plan is larger)."""
        return bool(self._flags()[0][0])

    def set_gap(self, gap_bar: int, gap_minutes: int) -> None:
        """Declare the series as two pieces glued at `gap_bar`, the second one `gap_minutes` later on the calendar
        (training folds of cross_validate_strategy): only the daily buckets of the metrics see it.  A gap is refused on a
        multi-timeframe sweep: its derived clocks were bucketed on the unbroken clock minute0 + t * bar_minutes."""
        if len(self.timeframes) > 1 and int(gap_minutes) != 0:
            raise ValueError("set_gap: a multi-timeframe bank is bucketed on the unbroken clock and cannot see a gap")
        self.cfg.gap_bar, self.cfg.gap_minutes = int(gap_bar), int(gap_minutes)

    def zone_map(self) -> torch.Tensor:
        """(min, max) per 32-bar block of the price rows and of the RSI bank (b200bt_zone_map), built on first use."""
        if self._zones is None:
            m = self.market
            n = int(_lib.load().b200bt_zone_map_floats(self.bank.shape[1], m.S, m.N))
            z = torch.empty(n, dtype=torch.float32, device=m.device)
            with torch.cuda.device(m.device):
                _lib.call("b200bt_zone_map", m.close.data_ptr(), _lib.ld(m.close), self.bank.data_ptr(), _lib.ld(self.bank),
                          self.bank.shape[1], m.S, m.N, z.data_ptr(), _lib.current_stream())
            self._zones = z
        return self._zones

    use_zones = True

    def _zones_if_amortised(self) -> Optional[torch.Tensor]:
        """The zone map costs about as much as it saves in ONE sweep (0.8 ms against ~0.2 ms at C2): it is built
        when this bank is swept a second time (a GA sweeps it every generation), not for a one-off evaluation."""
        self._tiled_sweeps += 1
        if not self.use_zones or (self._tiled_sweeps < 2 and self._zones is None):
            return None
        return self.zone_map()

    def plan(self, population: List[Dict], pred: Optional[np.ndarray] = None, rows: Optional[np.ndarray] = None) -> Optional[List]:
        """The kernel path `evaluate` takes for this population under self.mode: None = fused kernel, else the
        list of TilePlan / ChunkPlan slices to pass to evaluate_device(plan=...).  `pred`: predicted_events of the
        population when the caller already has it (evaluate derives it from the decoded records)."""
        long_enough = self.market.N >= self.chunk_min_bars
        tiled = self.mode == "tiled"
        if self.mode == "auto" and long_enough:
            # thread-per-lane needs many machines: enough chunks per lane, or enough lanes (tools/mode_crossover.py:
            # at 200k bars the warp-per-chunk path is faster below ~2000 individuals x 10 symbols)
            k = TilePlan.chunks_for(len(population), self.market.N, self.market.S, self.market.device,
                                    self.chunk_options.get("warm", TilePlan.WARM), self.chunk_options.get("max_chunks", 64))
            tiled = k >= 16 or len(population) * self.market.S * k >= 100_000
        if not (tiled or self.mode == "chunked" or (self.mode == "auto" and long_enough)):
            return None
        options = dict(self.chunk_options)
        if not tiled and self.mode == "auto":
            options.setdefault("target_events", 8192)
        self._pool_options(options)
        if tiled and rows is None and len(self.timeframes) > 1:
            rows = decode_population(population, self.period_row, len(self.timeframes))["rsi_row"]
        return self.plan_batches(population, tiled=tiled, pred=pred, rows=rows, **options)

    def _pool_options(self, options: Dict) -> None:
        """Event-pool sizing learns from the previous sweep of this bank: the cost model behind `pred` is calibrated on random
        populations, while the populations a GA evolves write several times more records.  The pool is scaled by the
        measured blocks-per-predicted-block ratio (never below the model), and by 4x more whenever it still overflowed (a
        fixed `pool_blocks` is then dropped).  Synchronises the stream when there is a previous sweep to learn from."""
        if self._last_plans:
            flags, used, predicted = self._flags()
            if flags[0]:
                self._pool_factor *= 4.0
                options.pop("pool_blocks", None)
            elif predicted > 0:
                self._pool_factor = max(1.0, 1.2 * used / predicted)
        if self._pool_factor > 1.0:
            options["pool_scale"] = self._pool_factor * options.get("pool_scale", 1.5)

    def plan_tiles(self, population: List[Dict], **kw) -> "TilePlan":
        m = self.market
        return _allocate_plans([TilePlan(population, m.N, m.S, m.device, **kw)], m.S, m.device)[0]

    def plan_chunks(self, population: List[Dict], **kw) -> "ChunkPlan":
        m = self.market
        return _allocate_plans([ChunkPlan(population, m.N, m.S, m.device, **kw)], m.S, m.device)[0]

    def plan_batches(self, population: List[Dict], max_pool_bytes: int = 8 << 30, tiled: bool = False,
                     pred: Optional[np.ndarray] = None, rows: Optional[np.ndarray] = None, **kw) -> List:
        """Plans for contiguous slices of the population whose event pools each stay below `max_pool_bytes`
        and share one workspace: large populations (BASELINE configs[4]: 10 000 x 50 symbols) record more
        events than fit in HBM at once, so they go through the chunked kernels slice by slice."""
        cls = TilePlan if tiled else ChunkPlan
        accepted = inspect.signature(cls.__init__).parameters     # chunk_options may carry the other path's knobs
        kw = {k: v for k, v in kw.items() if k in accepted}
        if pred is None:
            pred = predicted_events(population, self.market.N)
        rows_of = (lambda lo, hi: {"rows": None if rows is None else rows[lo:hi]}) if tiled else (lambda lo, hi: {})
        pool_bytes = None if kw.get("pool_blocks") is not None else pred * (self.market.S * 8 * kw.get("pool_scale", 1.5))
        if pool_bytes is None or float(pool_bytes.sum()) <= max_pool_bytes:
            plans = [cls(population, self.market.N, self.market.S, self.market.device, pred=pred, **rows_of(0, None), **kw)]
        else:
            cuts, acc = [0], 0.0
            for i, b in enumerate(pool_bytes):
                if acc + b > max_pool_bytes and i > cuts[-1]:
                    cuts.append(i)
                    acc = 0.0
                acc += b
            cuts.append(len(population))
            plans = [cls(population[lo:hi], self.market.N, self.market.S, self.market.device, lo=lo, pred=pred[lo:hi],
                         **rows_of(lo, hi), **kw) for lo, hi in zip(cuts[:-1], cuts[1:])]
        return _allocate_plans(plans, self.market.S, self.market.device)

    # -- host-facing evaluation --------------------------------------------
    def _unique(self, population: List[Dict]) -> Tuple[np.ndarray, List[Dict], Optional[np.ndarray]]:
        """Decoded records of the individuals of `population` that decode differently, in population order, their dicts,
        and the index that expands per-unique results back to `population` (None when all are distinct).  Individuals
        that decode to the same kernel parameters (the reference rule reads 6 of the 18 genes, and elitism / crossover
        copy individuals) are evaluated once."""
        packed = decode_population(population, self.period_row, len(self.timeframes))
        dup = _duplicate_classes(packed)
        if dup is None:
            return packed, population, None
        keep, expand = dup
        return np.ascontiguousarray(packed[keep]), [population[i] for i in keep], expand

    def evaluate(self, population: List[Dict]) -> np.ndarray:
        """fitness (float64[pop]) of a list of parameter dicts; H2D of the decoded
        population and D2H of the fitness vector happen inside this call."""
        if not population:
            return np.zeros(0, dtype=np.float64)
        if self.aggregation == "book":
            return self._evaluate_book(*self._unique(population))
        return self._evaluate_unique(*self._unique(population), self.event_cap)

    def evaluate_objectives_device(self, population: List[Dict], objectives) -> torch.Tensor:
        """Objective matrix float64 [pop][M] on the device: one evaluate() (same deduplication, schedules and book slicing),
        then b200bt_objective_matrix on its stats -- the lane stats averaged over the symbols under aggregation="mean", the
        book stats under "book".  objectives: [(lane-stat field, maximize)] (pareto.objectives_from_goals); the values are
        in the metric's own sense, so ("score", True) under "mean" gives evaluate()'s fitness bit for bit."""
        from . import pareto
        objectives = list(objectives)
        for name, _ in objectives:
            pareto._field(name)
        if not population:
            return torch.zeros((0, len(objectives)), dtype=torch.float64, device=self.market.device)
        self.evaluate(population)
        stats = self._book_dev if self.aggregation == "book" else self._stats
        out = pareto.objective_matrix(stats, objectives)
        if self._inverse is not None:
            out = out.index_select(0, torch.from_numpy(self._inverse).to(out.device))
        return out

    def evaluate_objectives(self, population: List[Dict], objectives) -> np.ndarray:
        """evaluate_objectives_device on the host: float64 [pop][M]."""
        return self.evaluate_objectives_device(population, objectives).cpu().numpy()

    def _evaluate_book(self, packed: np.ndarray, population: List[Dict], expand: Optional[np.ndarray]) -> np.ndarray:
        """evaluate() under aggregation="book": sweep with event buffers, then b200bt_book_metrics.

        The event cap of the first book evaluation is exact: a sweep without events counts every lane's records first.
        Later evaluations reuse the largest lane of the previous one with BOOK_CAP_HEADROOM; a slice in which some book
        lost records to a too-small guess is swept again with its exact cap (the lane counts are exact either way), so the
        results never depend on the guess.  Slices of the population keep their event buffers within max_event_bytes."""
        m = self.market
        U = len(packed)
        book = torch.empty((U, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=m.device)
        fit = torch.empty(U, dtype=torch.float64, device=m.device)

        def launch(indiv: torch.Tensor, lo: int, hi: int, cap: int) -> None:
            _lib.call("b200bt_book_metrics", m.close.data_ptr(), _lib.ld(m.close), m.S, m.N, indiv.data_ptr(), hi - lo,
                      C.byref(self.cfg), self._stats.data_ptr(), self._events.data_ptr(), cap, book[lo:hi].data_ptr(),
                      fit[lo:hi].data_ptr(), _lib.current_stream())

        self._record_pass(packed, population, expand, self._book_cap, launch)
        busiest = self._exact_cap(self._stats)
        self._book_cap = busiest + busiest // BOOK_CAP_HEADROOM + 2
        self._book_dev = book
        self._book = book.cpu().numpy()
        if expand is not None:
            self._book = self._book[expand]
        res = fit.cpu().numpy()
        return res if expand is None else res[expand]

    def _record_pass(self, packed: np.ndarray, population: List[Dict], expand: Optional[np.ndarray], cap: int,
                     launch: Callable[[torch.Tensor, int, int, int], None]) -> None:
        """Run a pass over the records of the decoded individuals `packed` (their dicts `population`, the output of _unique):
        with cap <= 0 a sweep without events counts every lane's records first and gives the exact cap; then _event_slices
        sweeps slices of the population with event buffers and launch(indiv[lo:hi], lo, hi, event cap) runs the pass on
        each slice's lane stats and event words (self._stats / self._events), on the current stream of the market's device.
        Afterwards lane_stats() describes every slice (_keep_slice_stats)."""
        m = self.market
        U = len(packed)
        if cap <= 0:
            self._evaluate_unique(packed, population, None, 0)
            cap = self._exact_cap(self._stats)
        stats = torch.empty((U, m.S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=m.device)
        indiv = torch.from_numpy(packed.view(np.uint8)).to(m.device).view(U, -1)
        for lo, hi, c in self._event_slices(packed, population, cap):
            with torch.cuda.device(m.device):
                launch(indiv[lo:hi], lo, hi, c)
            stats[lo:hi] = self._stats
        self._keep_slice_stats(stats, expand)

    def _event_slices(self, packed: np.ndarray, population: List[Dict], cap: int):
        """Sweep the decoded individuals `packed` with event buffers, in slices whose buffers keep within max_event_bytes,
        and yield (lo, hi, event cap) once the slice [lo, hi) is swept: its lane stats and event words are then
        self._stats / self._events, every record of every lane held.  `cap` is a guess (a learnt cap) or exact; a slice in
        which some lane lost records to a too-small guess is swept again with its exact cap (the lane counts are exact
        either way), cut again so that every piece keeps within the budget."""
        U, S = len(packed), self.market.S
        per_row = lambda c: max(1, self.max_event_bytes // (S * c * 4))     # individuals whose event buffers fit the budget
        self.book_resweeps, self.last_event_bytes = 0, 0
        rows = per_row(cap)
        todo = [(lo, min(U, lo + rows), cap, False) for lo in range(0, U, rows)]      # (lo, hi, event cap, cap is exact)
        while todo:
            lo, hi, c, exact = todo.pop(0)
            self._evaluate_unique(packed[lo:hi], population[lo:hi], None, c)
            self.last_event_bytes = max(self.last_event_bytes, (hi - lo) * S * c * 4)
            if not exact and int(self._stats[:, :, 0].max().item()) > c:
                self.book_resweeps += 1
                need = self._exact_cap(self._stats)
                self._stats = self._events = self._buffer_key = None       # the guessed buffers are freed first
                step = per_row(need)
                todo[:0] = [(a, min(hi, a + step), need, True) for a in range(lo, hi, step)]
                continue
            yield lo, hi, c

    def _keep_slice_stats(self, lanes: torch.Tensor, expand: Optional[np.ndarray]) -> None:
        """After _event_slices: lane_stats() describes every slice (`lanes`, assembled by the caller); the event words are
        kept only when one slice held the whole population."""
        if self._stats.shape[0] != lanes.shape[0]:     # the event words of the slices were not kept together
            self._events, self._buffer_key = None, None
        self._stats, self._inverse = lanes, expand

    @staticmethod
    def _exact_cap(stats: torch.Tensor) -> int:
        """Event cap that holds every record of every lane of `stats` (n_records of the busiest lane, at least 2)."""
        return max(2, int(stats[:, :, 0].max().item()))

    def book_stats(self) -> Dict[str, np.ndarray]:
        """Book metrics of the last aggregation="book" evaluation: the lane_stats() fields as [pop] arrays, computed on each
        individual's records on every symbol as one trade list (b200bt_book_metrics), plus
          return_pct          net_profit / initial_capital * 100
          avg_trade_duration  minutes, over the merged record pairs (2k, 2k+1) (calculate_metrics :166-178, whose pairs may
                              mix symbols); bars * bar_minutes, so a pair across the seam of a glued series (set_gap)
                              does not count the gap
          profitable_symbols  bool [pop][S]: the symbol's records net a profit (symbol_pnl > 0, :190-199); a symbol without
                              records is in neither of the reference's symbol dicts, so test it with n_records of lane_stats()
        lane_stats() still describes the per-symbol lanes of the same evaluation."""
        if self._book is None:
            raise RuntimeError("book_stats() needs an evaluate() under aggregation='book' first")
        out = _stats_fields(self._book)
        out["return_pct"] = out["net_profit"] / self.cfg.initial_capital * 100
        pairs = np.floor(out["n_records"] / 2)
        with np.errstate(divide="ignore", invalid="ignore"):
            out["avg_trade_duration"] = np.where(pairs > 0, out["sum_duration_bars"] * self.market.bar_minutes / pairs, 0.0)
        lanes = self.lane_stats()
        out["profitable_symbols"] = (lanes["n_records"] > 0) & (lanes["net_profit"] > 0)
        return out

    def _evaluate_unique(self, packed: np.ndarray, population: List[Dict], expand: Optional[np.ndarray],
                         event_cap: int) -> np.ndarray:
        """evaluate() on the output of _unique, keeping `event_cap` event words per lane."""
        dev = self.market.device
        self.last_unique = pop = len(population)
        pred = EVENTS_PER_COST_BAR * costs_from_packed(packed, self.periods, self.timeframes) * self.market.N
        plan = self.plan(population, pred=pred, rows=packed["rsi_row"])
        if plan is None:       # the fused kernel dispatches in this order: same RSI period adjacent, most expensive first
            order = np.lexsort((np.arange(pop), -pred, packed["rsi_row"])).astype(np.int32)
        else:
            order = np.zeros(0, dtype=np.int32)
        nbytes = packed.nbytes
        if self._pinned_in is None or self._pinned_in.numel() < nbytes + order.nbytes:
            self._pinned_in = torch.empty(nbytes + order.nbytes, dtype=torch.uint8, pin_memory=True)
        if self._pinned_out is None or self._pinned_out.numel() < pop:
            self._pinned_out = torch.empty(pop, dtype=torch.float64, pin_memory=True)
        hin = self._pinned_in.numpy()
        hin[:nbytes] = packed.view(np.uint8)
        hin[nbytes:nbytes + order.nbytes] = order.view(np.uint8)
        staged = self._pinned_in[:nbytes + order.nbytes].to(dev, non_blocking=True)
        indiv_dev = staged[:nbytes]
        order_dev = staged[nbytes:].view(torch.int32) if order.size else None
        fit = torch.empty(pop, dtype=torch.float64, device=dev)
        self.evaluate_device(indiv_dev, order_dev, pop, fit, plan=plan, event_cap=event_cap)
        self._inverse = expand
        out = self._pinned_out[:pop]
        out.copy_(fit, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        self.h2d_bytes = nbytes + order.nbytes
        self.d2h_bytes = pop * 8
        res = out.numpy().copy()
        return res if expand is None else res[expand]

    TRADE_PNL_MAX_BYTES = 4 << 30

    def trade_pnl(self, population: List[Dict], max_bytes: int = TRADE_PNL_MAX_BYTES):
        """Round-trip PnL of every (individual, symbol) lane, on the device, in the order of `population`:
        (trip_pnl float64 [pop][S][T_max], n_trips int32 [pop][S], fee float64 [pop][S]).  Lane (i, s) holds n_trips[i, s]
        round trips; its records are, in time order, an entry with pnl -fee and an exit with pnl trip_pnl[i, s, j] --
        bit-identical to the pnl of StrategyEvaluationSystem._simulate_trades' records (b200bt_trade_pnl).

        Two sweeps of this bank under this schedule: the first counts each lane's records, the second writes their event
        words with event_cap = the largest count.  Individuals that decode alike are swept once.  Meant for the top of a
        population: a ValueError names the bytes when the event and PnL buffers would exceed `max_bytes`.  Afterwards
        lane_stats() / events() describe this population (the next evaluate() allocates its own buffers)."""
        if not population:
            raise ValueError("trade_pnl needs at least one individual")
        m = self.market
        packed, unique, expand = self._unique(population)
        U, P, S = len(packed), len(population), m.S
        self._evaluate_unique(packed, unique, expand, 0)
        cap = int(self._stats[:, :, 0].max().item())           # n_records of the busiest lane (always even)
        cap = max(2, cap + (cap & 1))
        T = cap // 2
        need = U * S * cap * 4 + (U + P) * S * T * 8
        if need > max_bytes:
            raise ValueError(f"trade_pnl: {need} bytes of event and trip PnL buffers for {P} individuals x {S} symbols "
                             f"(up to {cap} records per lane) exceed the budget of {max_bytes} bytes; pass the top "
                             f"of the population, not all of it")
        self._evaluate_unique(packed, unique, expand, cap)
        indiv = torch.from_numpy(packed.view(np.uint8)).to(m.device)
        trip = torch.empty((U, S, T), dtype=torch.float64, device=m.device)
        n_trips = torch.empty((U, S), dtype=torch.int32, device=m.device)
        fee = torch.empty((U, S), dtype=torch.float64, device=m.device)
        with torch.cuda.device(m.device):
            _lib.call("b200bt_trade_pnl", m.close.data_ptr(), _lib.ld(m.close), S, m.N, indiv.data_ptr(), U,
                      self._stats.data_ptr(), self._events.data_ptr(), cap, trip.data_ptr(), T, n_trips.data_ptr(),
                      fee.data_ptr(), _lib.current_stream())
        if expand is not None:
            inv = torch.from_numpy(expand).to(m.device)
            trip, n_trips, fee = trip.index_select(0, inv), n_trips.index_select(0, inv), fee.index_select(0, inv)
        if bool((n_trips < 0).any()):
            raise RuntimeError("trade_pnl: a lane wrote more records than its event buffer held")
        return trip, n_trips, fee

    DAILY_PNL_MAX_BYTES = 8 << 30

    def calendar_days(self) -> Tuple[int, int]:
        """(first_day, D): the calendar day of bar 0 (days since 1970-01-01 of the market's minute clock) and the number of
        days from it to the day of the last bar, the skipped days of a glued series (set_gap) included."""
        c = self.cfg
        return calendar_days(c.minute0, c.bar_minutes, self.market.N, c.gap_bar, c.gap_minutes)

    def daily_pnl(self, population: List[Dict], max_bytes: int = DAILY_PNL_MAX_BYTES):
        """Per-day PnL of every individual's book and of its lanes, on the device, in the order of `population`:
        (book float64 [pop][D], lanes float64 [pop][S][D], first_day).  Column d is calendar day first_day + d (days since
        1970-01-01); lanes[i, s, d] is the sum of the pnl of the records of individual i on symbol s dated on that day,
        book[i, d] their sum over symbols -- the daily buckets of calculate_metrics (strategy_evaluation.py:141-159) on the
        book, kept for every calendar day of the series (a day without records is 0.0).  b200bt_daily_pnl.

        A counting sweep gives the exact event cap, then slices of the population whose event buffers keep within
        max_event_bytes are swept and bucketed.  Individuals that decode alike are swept once.  A ValueError names the
        bytes when the output rows alone exceed `max_bytes`.  Afterwards lane_stats() describes this population."""
        if not population:
            raise ValueError("daily_pnl needs at least one individual")
        m = self.market
        packed, unique, expand = self._unique(population)
        U, P, S = len(packed), len(population), m.S
        first_day, D = self.calendar_days()
        need = (U + (P if expand is not None else 0)) * (S + 1) * D * 8
        if need > max_bytes:
            raise ValueError(f"daily_pnl: {need} bytes of per-day rows for {P} individuals x {S} symbols x {D} days exceed "
                             f"the budget of {max_bytes} bytes")
        lanes = torch.empty((U, S, D), dtype=torch.float64, device=m.device)
        book = torch.empty((U, D), dtype=torch.float64, device=m.device)

        def launch(indiv: torch.Tensor, lo: int, hi: int, cap: int) -> None:
            _lib.call("b200bt_daily_pnl", m.close.data_ptr(), _lib.ld(m.close), S, m.N, indiv.data_ptr(), hi - lo,
                      C.byref(self.cfg), self._stats.data_ptr(), self._events.data_ptr(), cap, lanes[lo:hi].data_ptr(), D,
                      book[lo:hi].data_ptr(), _lib.current_stream())

        self._record_pass(packed, unique, expand, 0, launch)
        if expand is not None:
            inv = torch.from_numpy(expand).to(m.device)
            book, lanes = book.index_select(0, inv), lanes.index_select(0, inv)
        return book, lanes, int(first_day)

    def class_stats(self, population: List[Dict], labels: torch.Tensor, n_classes: int):
        """Trade metrics of every lane split by the label of each record's bar (b200bt_class_stats), in the order of
        `population`: (stats float64 [R][pop][S][20] on the device, [R dicts field -> [pop][S] array]).  Block r holds
        calculate_metrics and the score on the records of lane (i, s) whose bar carries label r; labels >= R belong to no
        class.  labels: device uint8 [S][N]; [1][N] (or a row expanded to [S][N]) is one row shared by every symbol.

        A counting sweep gives the exact event cap, then slices of the population whose event buffers keep within
        max_event_bytes are swept and split.  Individuals that decode alike are swept once.  Afterwards lane_stats()
        describes this population."""
        if not population:
            raise ValueError("class_stats needs at least one individual")
        m = self.market
        R = int(n_classes)
        if not 1 <= R <= 8:
            raise ValueError(f"class_stats: n_classes must be 1..8, not {R}")
        from .regime import label_rows
        labels, ld_labels = label_rows(labels, m.S, m.N, "class_stats: labels")
        packed, unique, expand = self._unique(population)
        U, S = len(packed), m.S
        out = torch.empty((R, U, S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=m.device)
        part = torch.empty_like(out)

        def launch(indiv: torch.Tensor, lo: int, hi: int, cap: int) -> None:
            piece = part.view(-1)[:R * (hi - lo) * S * _lib.LANE_STATS_WORDS].view(R, hi - lo, S, -1)   # [R][slice][S]
            _lib.call("b200bt_class_stats", m.close.data_ptr(), _lib.ld(m.close), S, m.N, indiv.data_ptr(), hi - lo,
                      C.byref(self.cfg), self._stats.data_ptr(), self._events.data_ptr(), cap, labels.data_ptr(),
                      ld_labels, R, piece.data_ptr(), _lib.current_stream())
            out[:, lo:hi] = piece

        self._record_pass(packed, unique, expand, 0, launch)
        if expand is not None:
            out = out.index_select(1, torch.from_numpy(expand).to(m.device))
        raw = out.cpu().numpy()
        return out, [_stats_fields(raw[r]) for r in range(R)]

    def lane_stats(self) -> Dict[str, np.ndarray]:
        """Per-lane metrics of the last evaluation: dict field -> [pop][S] array."""
        raw = self._stats.cpu().numpy()
        if self._inverse is not None:
            raw = raw[self._inverse]
        return _stats_fields(raw)

    def advanced_stats(self) -> Dict[str, np.ndarray]:
        """calculate_advanced_metrics (strategy_evaluation.py:231-319) for every lane of the last evaluation,
        [pop][S] arrays: the Sortino ingredients come out of the kernels' daily buckets, the rest is arithmetic on
        the lane stats (same expressions as the reference, including its fixed 10 000 in the recovery factor)."""
        st = self.lane_stats()
        with np.errstate(divide="ignore", invalid="ignore"):
            dd, net, n = st["max_drawdown"], st["net_profit"], st["n_records"]
            ret_pct = net / self.cfg.initial_capital * 100
            avg_p = np.where(st["n_wins"] > 0, st["total_profit"] / st["n_wins"], 0.0)
            avg_l = np.where(st["n_losses"] > 0, st["total_loss"] / st["n_losses"], 0.0)
            return {
                "calmar_ratio": np.where(dd > 0, (ret_pct / 100) / dd, np.inf),
                "sortino_ratio": st["sortino_ratio"],
                "recovery_factor": np.where(dd > 0, net / (dd * 10000), np.inf),
                "expectancy": np.where(n > 0, st["win_rate"] * avg_p - (1 - st["win_rate"]) * np.abs(avg_l), 0.0),
                "profit_per_day": st["mean_daily_pnl"],
            }

    def events(self) -> Optional[np.ndarray]:
        """First `event_cap` event words per lane, uint32 [pop][S][cap] (see B200BT_EVENT_*)."""
        if self._events is None:
            return None
        ev = self._events.cpu().numpy().view(np.uint32)
        return ev if self._inverse is None else ev[self._inverse]

    @property
    def fitness_function(self):
        return fitness_callable(self.evaluate)
