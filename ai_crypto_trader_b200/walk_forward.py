"""Walk-forward analysis of the strategy-evolution loop on the GPU engine.

Reference: services/strategy_evolution_service.py.  The service's loop (:1584-1711) checks the deployed strategy, asks
`_needs_improvement` (:1571-1582) against the risk level's thresholds (:119-142) and, when that fires, re-optimises it with
a GA seeded with the current parameters (:655) and hot-swaps the winner in (:349).  A walk-forward analysis replays that on
history: fit on an in-sample window, trade the fitted parameters on the out-of-sample bars that follow, move on.

Windows are cut on the market's own calendar.  Boundary k is the first bar of day d0 + in_sample_days + k * out_of_sample_days
(d0 = the day of bar 0); window k fits on the in_sample_days days before it (or everything from bar 0, anchored) and trades
the bars up to the next boundary (the last window up to N).

reoptimize="always" runs W independent GAs in lockstep over one [W][pop][genes] device matrix: each generation is one
decode launch (b200bt_decode_individuals), one b200bt_sweep_segments launch over W * pop one-segment schedules, one
b200bt_fitness_reduce, a per-window stable argsort and W calls of b200bt_ga_next_generation.  Only the [W][pop] fitness comes
back to the host.  Window w's trajectory is the one DeviceGeneticAlgorithm(random_seed = seed + w) produces alone on that
window.  reoptimize="when_needed" is the reference loop: at each boundary the deployed parameters are scored on the
in-sample window and re-optimised only when the gate fires.

A final b200bt_sweep_segments call scores, in one launch, the stitched out-of-sample schedule (segment k = window k's
out-of-sample bars traded by window k's deployed parameters) and every window's in-sample and out-of-sample lanes.  Each
segment is a fresh _simulate_trades call: an open position does not carry across a hot swap.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .genetic_algorithm import _is_int_range
from .population import iso_minute
from .sweep import PopulationSweep, _stats_fields, decode_population

# decode_population's genes, in the column order of b200bt_decode_individuals
DECODE_GENES = ("rsi_period", "rsi_oversold", "rsi_overbought", "take_profit", "stop_loss", "max_position_size")
DECODE_MAX_PERIODS = 256                      # entries of b200bt_decode_individuals' period table
SEED_MASK = 0xFFFFFFFFFFFFFFFF
# config.json evolution block: the keys the risk thresholds (:119-142) read, where the caller's block lacks them
EVOLUTION_DEFAULTS = {"min_win_rate": 0.52, "max_drawdown": 15.0, "min_sharpe_ratio": 1.2,
                      "risk_management": {"max_position_size": 0.4}}
STAT_FIELDS = _lib.LANE_STATS_FIELDS[:-1]     # the lane-stat fields a mean is taken of (not trade_hash)


# -- window plan ----------------------------------------------------------------------------------------------------------
def first_bar_of_day(day: int, minute0: int, bar_minutes: int) -> int:
    """First bar t >= 0 with (minute0 + t * bar_minutes) // 1440 >= day."""
    return max(0, -((minute0 - day * 1440) // bar_minutes))


def plan_windows(minute0: int, bar_minutes: int, N: int, in_sample_days: int, out_of_sample_days: int,
                 anchored: bool = False) -> List[Tuple[int, int, int, int]]:
    """[(is_start, is_end, oos_start, oos_end)] of the walk-forward windows of an N-bar series (bar t at Unix minute
    minute0 + t * bar_minutes).  is_end == oos_start is boundary k; a boundary whose next one falls on the same bar (a day
    without bars) opens no window.  Raises ValueError when no out-of-sample bar exists."""
    if in_sample_days < 1 or out_of_sample_days < 1:
        raise ValueError("in_sample_days and out_of_sample_days must be >= 1")
    if bar_minutes < 1 or minute0 < 0 or N < 1:
        raise ValueError("bar_minutes must be >= 1, minute0 >= 0 and N >= 1")
    d0 = minute0 // 1440
    out = []
    k = 0
    while True:
        day = d0 + in_sample_days + k * out_of_sample_days
        b = first_bar_of_day(day, minute0, bar_minutes)
        if b >= N:
            break
        nxt = min(N, first_bar_of_day(day + out_of_sample_days, minute0, bar_minutes))
        start = 0 if anchored else first_bar_of_day(day - in_sample_days, minute0, bar_minutes)
        if nxt > b and b > start:
            out.append((start, b, b, nxt))
        k += 1
    if not out:
        raise ValueError(f"no out-of-sample bar: {N} bars of {bar_minutes} minutes do not reach past the first "
                         f"{in_sample_days} in-sample days")
    return out


def segment_tables(schedules: Sequence[Sequence[Tuple[int, int, int]]]) -> Tuple[np.ndarray, np.ndarray]:
    """The segment records (_lib.SEGMENT_DTYPE [n], reserved = 0) and seg_begin int32 [J + 1] of b200bt_sweep_segments
    for schedules [[(start, end, individual)]]."""
    seg = np.array([(a, b, k, 0) for sched in schedules for a, b, k in sched], dtype=_lib.SEGMENT_DTYPE)
    begin = np.zeros(len(schedules) + 1, dtype=np.int32)
    np.cumsum([len(s) for s in schedules], out=begin[1:])
    return seg, begin


def ga_schedules(ranges: Sequence[Tuple[int, int]], pop: int) -> List[List[Tuple[int, int, int]]]:
    """One generation of the lockstep GA: schedule w * pop + i trades individual w * pop + i on window w's in-sample
    range ranges[w] = (start, end)."""
    return [[(a, b, w * pop + i)] for w, (a, b) in enumerate(ranges) for i in range(pop)]


def scoring_schedules(windows: Sequence[Tuple[int, int, int, int]]) -> List[List[Tuple[int, int, int]]]:
    """The final scoring launch, individual k = window k's deployed parameters: schedule 0 is the stitched out-of-sample
    run (segment k = window k's out-of-sample bars), schedules 1 .. K each window's out-of-sample lane, K + 1 .. 2K each
    window's in-sample lane."""
    out = [[(c, d, k) for k, (_, _, c, d) in enumerate(windows)]]
    out += [[(c, d, k)] for k, (_, _, c, d) in enumerate(windows)]
    out += [[(a, b, k)] for k, (a, b, _, _) in enumerate(windows)]
    return out


def generation_best(fitness: np.ndarray, best: np.ndarray):
    """One generation's fitness [W][pop] against the best so far [W], as DeviceGeneticAlgorithm takes them row by row.
    -> (improved [W] bool, the row index it keeps [W], the new best [W], and the history's max, min and mean [W]).

    DeviceGeneticAlgorithm walks a row in order and keeps an individual that beats the best so far (NaN never does): the
    one it keeps last is the first holding the row's maximum, when that maximum beats the best.  The history's max / min /
    mean are Python's max(), min() and sum() / len over the row: a NaN in first place is what max() and min() return, a
    later NaN is passed over, and the mean is Python's sum() over the row."""
    W = fitness.shape[0]
    nan = np.isnan(fitness)
    key = np.where(nan, -np.inf, fitness)
    top_i = key.argmax(axis=1)
    top = key[np.arange(W), top_i]
    improved = top > best
    hi = np.where(nan[:, 0], np.nan, key.max(axis=1))
    lo = np.where(nan[:, 0], np.nan, np.where(nan, np.inf, fitness).min(axis=1))
    mean = np.array([sum(row) / len(row) for row in fitness.tolist()])     # Python's own float sum (compensated from 3.12)
    return improved, top_i, np.where(improved, top, best), hi, lo, mean


def window_seed(random_seed: Optional[int], w: int) -> int:
    """Seed of window w's GA: (random_seed + w) mod 2^64 (random_seed None counts as 0, as DeviceGeneticAlgorithm's)."""
    return (int(random_seed or 0) + int(w)) & SEED_MASK


# -- the reference's gate -------------------------------------------------------------------------------------------------
def risk_thresholds(evolution_config: Optional[Dict] = None, leverage_trading: bool = False) -> Dict[str, Dict]:
    """The risk levels' thresholds as strategy_evolution_service.py:119-142 builds them from the evolution config block
    (keys it lacks take config.json's values, EVOLUTION_DEFAULTS)."""
    ev = dict(EVOLUTION_DEFAULTS, **(evolution_config or {}))
    base_position_size = dict(EVOLUTION_DEFAULTS["risk_management"], **ev.get("risk_management", {}))["max_position_size"]
    leverage_multiplier = 0.5 if leverage_trading else 1.0
    return {
        "LOW": {"min_win_rate": ev["min_win_rate"] + 0.05, "max_drawdown": ev["max_drawdown"] - 5,
                "min_sharpe_ratio": ev["min_sharpe_ratio"] + 0.3,
                "position_size_pct": base_position_size * 0.5 * leverage_multiplier},
        "MEDIUM": {"min_win_rate": ev["min_win_rate"], "max_drawdown": ev["max_drawdown"],
                   "min_sharpe_ratio": ev["min_sharpe_ratio"], "position_size_pct": base_position_size * leverage_multiplier},
        "HIGH": {"min_win_rate": ev["min_win_rate"] - 0.05, "max_drawdown": ev["max_drawdown"] + 5,
                 "min_sharpe_ratio": ev["min_sharpe_ratio"] - 0.3,
                 "position_size_pct": base_position_size * 1.5 * leverage_multiplier},
    }


def needs_improvement(performance: Dict, risk_params: Dict) -> bool:
    """_needs_improvement (:1571-1582) verbatim.  Note the reference reads a "drawdown" key (in percent, against
    max_drawdown 15.0) that calculate_metrics never writes: fed a metrics dict as it is, the default 100 always fires the
    gate.  gate_performance() supplies the key."""
    if not performance:
        return False
    return (
        performance.get("sharpe_ratio", 0) < risk_params["min_sharpe_ratio"] or
        performance.get("drawdown", 100) > risk_params["max_drawdown"] or
        performance.get("win_rate", 0) < risk_params["min_win_rate"]
    )


def gate_performance(stats: Dict[str, np.ndarray]) -> Dict[str, float]:
    """The performance dict the gate reads, from one schedule's lane stats [S]: the means over symbols of sharpe_ratio and
    win_rate, and drawdown = 100 x the mean max_drawdown (a percentage, as the thresholds state it)."""
    return {"sharpe_ratio": float(np.mean(stats["sharpe_ratio"])), "win_rate": float(np.mean(stats["win_rate"])),
            "drawdown": 100.0 * float(np.mean(stats["max_drawdown"]))}


def efficiency(oos_net: float, oos_days: float, is_net: float, is_days: float) -> float:
    """Walk-forward efficiency: out-of-sample net profit per day over in-sample net profit per day; NaN when the in-sample
    net profit is not positive (or a span is empty)."""
    if not (is_net > 0) or not (is_days > 0) or not (oos_days > 0):
        return math.nan
    return (oos_net / oos_days) / (is_net / is_days)


def _fitness_of(scores: Sequence[float]) -> float:
    """b200bt_fitness_reduce's expression on the host: the sequential sum over symbols from +0.0, divided by S."""
    acc = 0.0
    for x in scores:
        acc += float(x)
    return acc / len(scores)


class WalkForward:
    """Walk-forward evaluation of the evolution loop on a PopulationSweep's market, RSI bank and score rule (aggregation
    "mean", one bar clock, no glued series)."""

    def __init__(self, sweep: PopulationSweep, param_ranges: Dict[str, Tuple], population_size: int = 20,
                 generations: int = 10, mutation_rate: float = 0.2, crossover_rate: float = 0.8,
                 elitism_pct: float = 0.1, tournament_size: int = 3, random_seed: Optional[int] = None):
        if sweep.aggregation != "mean":
            raise ValueError("walk-forward scores each symbol's lane: aggregation must be 'mean'")
        if len(sweep.timeframes) > 1:
            raise ValueError("walk-forward decodes one bar clock's RSI bank (no rsi_timeframe gene)")
        if sweep.cfg.gap_bar:
            raise ValueError("walk-forward runs on one contiguous series (no glued cross-validation fold)")
        self.sweep, self.market = sweep, sweep.market
        self.param_ranges = dict(param_ranges)
        self.population_size, self.generations = int(population_size), int(generations)
        self.mutation_rate, self.crossover_rate = float(mutation_rate), float(crossover_rate)
        self.elitism_pct, self.tournament_size = float(elitism_pct), int(tournament_size)
        self.random_seed = random_seed
        self.names = list(self.param_ranges)
        G = len(self.names)
        self._lo = (C.c_double * G)(*[float(self.param_ranges[n][0]) for n in self.names])
        self._hi = (C.c_double * G)(*[float(self.param_ranges[n][1]) for n in self.names])
        self._is_int = (C.c_int * G)(*[1 if _is_int_range(*self.param_ranges[n]) else 0 for n in self.names])
        self._cols = (C.c_int * 6)(*[self.names.index(g) if g in self.names else -1 for g in DECODE_GENES])
        rows = np.full(max(sweep.period_row) + 1, -1, dtype=np.int32)
        for p, r in sweep.period_row.items():
            rows[p] = r
        if len(rows) > DECODE_MAX_PERIODS:
            raise ValueError(f"the device decode takes periods below {DECODE_MAX_PERIODS}")
        self._period_row = (C.c_int32 * len(rows))(*rows.tolist())
        self.device = self.market.device

    # -- matrix <-> parameter dicts -----------------------------------------------------------------------------------
    def _to_dicts(self, matrix: np.ndarray) -> List[Dict]:
        """DeviceGeneticAlgorithm's conversion: integer genes as int (truncated), the rest as float."""
        cols = [matrix[:, g].astype(np.int64).tolist() if self._is_int[g] else matrix[:, g].tolist()
                for g in range(len(self.names))]
        return [dict(zip(self.names, row)) for row in zip(*cols)]

    def _row(self, params: Dict) -> List[float]:
        return [float(params.get(n, self.param_ranges[n][0])) for n in self.names]

    # -- device calls -------------------------------------------------------------------------------------------------
    def _tables(self, schedules: List[List[Tuple[int, int, int]]]) -> Tuple[torch.Tensor, torch.Tensor]:
        """segment_tables(schedules) on the device."""
        seg, begin = segment_tables(schedules)
        return torch.from_numpy(seg.view(np.int64)).to(self.device), torch.from_numpy(begin).to(self.device)

    def sweep_segments(self, indiv: torch.Tensor, n_indiv: int, segments: torch.Tensor, seg_begin: torch.Tensor,
                       stats: torch.Tensor, events: Optional[torch.Tensor] = None, event_cap: int = 0) -> None:
        """b200bt_sweep_segments on the sweep's market and bank (current stream): stats [J][S][LANE_STATS_WORDS]."""
        J = int(seg_begin.numel()) - 1
        with torch.cuda.device(self.device):
            _lib.call("b200bt_sweep_segments", *self.sweep._data_args(), indiv.data_ptr(), int(n_indiv),
                      segments.data_ptr(), seg_begin.data_ptr(), J, C.byref(self.sweep.cfg), stats.data_ptr(),
                      _lib.ptr(events), int(event_cap), _lib.current_stream())

    def decode(self, params: torch.Tensor, out: torch.Tensor) -> None:
        """b200bt_decode_individuals of the rows of the contiguous float64 matrix `params` [..][genes] into `out`."""
        n = params.numel() // len(self.names)
        with torch.cuda.device(self.device):
            _lib.call("b200bt_decode_individuals", params.data_ptr(), len(self.names), n, self._cols, self._period_row,
                      len(self._period_row), out.data_ptr(), _lib.current_stream())

    def score(self, schedules: List[List[Tuple[int, int, int]]], params: List[Dict]) -> Dict[str, np.ndarray]:
        """Lane stats {field: [J][S]} of schedules [[(start, end, index into params)]] in one launch."""
        packed = decode_population(params, self.sweep.period_row)
        indiv = torch.from_numpy(packed.view(np.uint8)).to(self.device, non_blocking=True)
        segments, seg_begin = self._tables(schedules)
        stats = torch.empty((len(schedules), self.market.S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=self.device)
        self.sweep_segments(indiv, len(params), segments, seg_begin, stats)
        return _stats_fields(stats.cpu().numpy())

    # -- the lockstep GA ------------------------------------------------------------------------------------------------
    def evolve(self, ranges: Sequence[Tuple[int, int]], seeds: Sequence[int], seeded: Optional[Dict] = None):
        """One GA per in-sample range [(start, end)], all in lockstep; GA w draws from seeds[w] and is seeded with `seeded`.
        -> (winners [W] dicts, best fitness [W], history [W][generations + 1] dicts, final parameter matrix [W][pop][G])."""
        W, pop, G = len(ranges), self.population_size, len(self.names)
        dev = self.device
        params = torch.zeros((W, pop, G), dtype=torch.float64, device=dev)
        nxt = torch.empty_like(params)
        sel = torch.empty((W, pop), dtype=torch.int32, device=dev)
        indiv = torch.empty(W * pop * C.sizeof(_lib.Individual), dtype=torch.uint8, device=dev)
        stats = torch.empty((W * pop, self.market.S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=dev)
        fit = torch.empty(W * pop, dtype=torch.float64, device=dev)
        segments, seg_begin = self._tables(ga_schedules(ranges, pop))
        self.last_fitness: List[np.ndarray] = []      # [W][pop] fitness of every generation of this call
        n_seeded = 0
        if seeded:
            n_seeded = 1
            params[:, 0] = torch.tensor(self._row(seeded), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            st = _lib.current_stream()
            for w in range(W):
                _lib.call("b200bt_ga_init", params[w].data_ptr(), pop, G, n_seeded, self._lo, self._hi, self._is_int,
                          int(seeds[w]), st)
        # best so far (DeviceGeneticAlgorithm: strictly greater wins, NaN never); until something beats -inf the winner is
        # row 0 of the initial population (the seeded parameters, when given)
        best_fit = np.full(W, -math.inf)
        best_rows = params[:, 0].clone()
        history: List[List[Dict]] = [[] for _ in range(W)]
        for generation in range(self.generations + 1):
            if generation:
                key = torch.where(torch.isnan(fit), torch.full_like(fit, -math.inf), fit).view(W, pop)
                ranked = torch.argsort(key, dim=1, descending=True, stable=True).to(torch.int32)
                with torch.cuda.device(dev):
                    st = _lib.current_stream()
                    for w in range(W):
                        _lib.call("b200bt_ga_next_generation", params[w].data_ptr(), key[w].data_ptr(), ranked[w].data_ptr(),
                                  pop, G, self._lo, self._hi, self._is_int, self.elitism_pct, self.tournament_size,
                                  self.crossover_rate, self.mutation_rate, int(seeds[w]), generation, sel[w].data_ptr(),
                                  nxt[w].data_ptr(), st)
                params, nxt = nxt, params
            self.decode(params, indiv)
            self.sweep_segments(indiv, W * pop, segments, seg_begin, stats)
            with torch.cuda.device(dev):
                _lib.call("b200bt_fitness_reduce", stats.data_ptr(), W * pop, self.market.S, fit.data_ptr(),
                          _lib.current_stream())
            host = fit.cpu().numpy().reshape(W, pop)
            self.last_fitness.append(host)
            improved, top_i, best_fit, hi, lo, mean = generation_best(host, best_fit)
            for w in range(W):
                history[w].append({"generation": generation, "best_fitness": float(hi[w]), "avg_fitness": float(mean[w]),
                                   "min_fitness": float(lo[w])})
            if improved.any():
                ws = torch.from_numpy(np.nonzero(improved)[0]).to(dev)
                best_rows[ws] = params[ws, torch.from_numpy(top_i[improved]).to(dev)]
        winners = self._to_dicts(best_rows.cpu().numpy())
        return winners, best_fit.tolist(), history, params

    # -- the walk-forward run -------------------------------------------------------------------------------------------
    def run(self, current_params: Optional[Dict], in_sample_days: int = 30, out_of_sample_days: int = 7,
            anchored: bool = False, reoptimize: str = "always", risk_level: str = "MEDIUM",
            evolution_config: Optional[Dict] = None, leverage_trading: bool = False) -> Dict:
        """The walk-forward report (see the module docstring).  reoptimize: "always" (every window re-fitted, all at once)
        or "when_needed" (the reference loop: the deployed parameters, starting as current_params, are re-fitted at a
        boundary only when the gate fires on their in-sample performance)."""
        if reoptimize not in ("always", "when_needed"):
            raise ValueError(f"reoptimize must be 'always' or 'when_needed', not {reoptimize!r}")
        m = self.market
        windows = plan_windows(m.minute0, m.bar_minutes, m.N, in_sample_days, out_of_sample_days, anchored)
        K = len(windows)
        seeds = [window_seed(self.random_seed, k) for k in range(K)]
        deployed: List[Dict] = []
        reoptimized: List[bool] = []
        histories: List[List[Dict]] = []
        gates: List[Optional[Dict]] = []
        if reoptimize == "always":
            winners, _, hist, _ = self.evolve([(a, b) for a, b, _, _ in windows], seeds, current_params)
            deployed, reoptimized, histories, gates = winners, [True] * K, hist, [None] * K
        else:
            if not current_params:
                raise ValueError("reoptimize='when_needed' starts from current_params")
            thresholds = risk_thresholds(evolution_config, leverage_trading)[risk_level]
            current = dict(current_params)
            for k, (a, b, _, _) in enumerate(windows):
                perf = gate_performance({f: v[0] for f, v in self.score([[(a, b, 0)]], [current]).items()})
                fire = needs_improvement(perf, thresholds)
                hist: List[Dict] = []
                if fire:
                    winners, _, hist_all, _ = self.evolve([(a, b)], [seeds[k]], current)
                    current, hist = winners[0], hist_all[0]
                deployed.append(dict(current))
                reoptimized.append(fire)
                histories.append(hist)
                gates.append(perf)
        st = self.score(scoring_schedules(windows), deployed)
        return self._report(windows, deployed, reoptimized, histories, gates, st)

    def _report(self, windows, deployed, reoptimized, histories, gates, st) -> Dict:
        m = self.market
        K = len(windows)
        day_of = lambda bars: bars * m.bar_minutes / 1440.0
        stamp = lambda t: iso_minute(m.minute0 + int(t) * m.bar_minutes)
        mean = lambda j: {f: float(np.mean(st[f][j])) for f in STAT_FIELDS}
        rows = []
        sums = np.zeros(4)
        for k, (a, b, c, d) in enumerate(windows):
            oos, ins = mean(1 + k), mean(1 + K + k)
            is_days, oos_days = day_of(b - a), day_of(d - c)
            sums += (oos["net_profit"], oos_days, ins["net_profit"], is_days)
            rows.append({
                "window": k, "in_sample": (a, b), "out_of_sample": (c, d),
                "in_sample_time": (stamp(a), stamp(b - 1)), "out_of_sample_time": (stamp(c), stamp(d - 1)),
                "reoptimized": bool(reoptimized[k]), "parameters": dict(deployed[k]),
                "in_sample_fitness": _fitness_of(st["score"][1 + K + k]),
                "in_sample_stats": ins, "out_of_sample_stats": oos,
                "efficiency": efficiency(oos["net_profit"], oos_days, ins["net_profit"], is_days),
                "gate_performance": gates[k], "history": histories[k]})
        stitched = {f: st[f][0] for f in st}
        return {
            "windows": rows,
            "stitched_stats": stitched,
            "stitched_mean": {f: float(np.mean(stitched[f])) for f in STAT_FIELDS},
            "efficiency": efficiency(*sums),
            "n_reoptimizations": int(sum(reoptimized)),
            "history": [r["history"] for r in rows],
        }
