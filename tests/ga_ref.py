"""Float64 NumPy restatement of the device GA operators (csrc/ga_ops.cu), draw for draw, for the tests.

  * `Words`: the kernels' GaRng for many (slot, stream) pairs at once -- one CONTINUOUS word stream per pair on
    oracle/mc_ref's Philox4x32-10, words handed out x[3], x[2], x[1], x[0] per block, and `below` / `uniform` on it.
    Calls take a lane mask, as a warp whose lanes take different branches draws only in the active lanes.
  * `init`, `select`, `breed`: ga_init_kernel, ga_select_kernel and ga_breed_kernel; `next_generation` is
    b200bt_ga_next_generation (elite count, select, breed) on host arrays.
  * `fma`: the correctly rounded fused multiply-add the kernels write out explicitly, computed exactly with Fraction.
  * `run`: DeviceGeneticAlgorithm.run around them -- NaN fitness ranks as -inf, stable descending rank, the dict view of
    the matrix (`to_dicts`) and the seeded rows of initialize_population.

`Stats` counts the events a test needs to know were exercised: uniforms that straddle two Philox blocks, rejected
repeated contenders, and fused results that differ from the twice-rounded expression.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from fractions import Fraction
from typing import Callable, Dict, List, Optional

import numpy as np

from oracle import mc_ref

SELECT, PARENTS, COINS, MUTATION, INIT = 0, 1, 2, 3, 4        # stream ids (counter word 2)
_2P26, _2M53 = 67108864.0, 1.0 / 9007199254740992.0


@dataclass
class Stats:
    straddles: int = 0              # uniform() whose two words come from two Philox blocks
    rejections: int = 0             # tournament draws rejected as a repeated contender
    fma_mutation: int = 0           # mutated float genes where the fused result differs from the twice-rounded one
    fma_init: int = 0               # initial float genes where the fused result differs from the twice-rounded one
    mutated: int = 0                # mutated genes, all kinds

    def add(self, other: "Stats") -> None:
        for k in self.__dataclass_fields__:
            setattr(self, k, getattr(self, k) + getattr(other, k))


def fma(a: float, b: float, c: float) -> float:
    """a * b + c rounded once (IEEE 754 fusedMultiplyAdd, round to nearest even)."""
    a, b, c = float(a), float(b), float(c)
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return a * b + c                                   # inf / NaN propagate as in the unfused expression
    exact = Fraction(a) * Fraction(b) + Fraction(c)
    if exact == 0:                                         # sign of an exact zero: -0 only if a*b and c are both -0
        return (a * b) + c if (a == 0 or b == 0) else 0.0
    try:
        return float(exact)                                # Fraction -> float rounds to nearest even
    except OverflowError:
        return float("inf") if exact > 0 else float("-inf")


def fma_array(a, b, c) -> np.ndarray:
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    return np.array([fma(x, y, z) for x, y, z in zip(a.ravel().tolist(), b.ravel().tolist(), c.ravel().tolist())],
                    dtype=np.float64).reshape(a.shape)


def clamp(v, lo, hi):
    """fmax(lo, fmin(hi, v)): a NaN operand yields the other one."""
    return np.fmax(lo, np.fmin(hi, v))


class Words:
    """GaRng(seed, generation, slot, stream) for every slot in `slots`: counter = (slot, generation, stream, block)."""

    def __init__(self, seed: int, generation: int, slots, stream: int, stats: Optional[Stats] = None):
        self.k0, self.k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
        self.c0 = np.asarray(slots, dtype=np.uint32)
        self.c1, self.c2 = np.uint32(generation), np.uint32(stream)
        n = len(self.c0)
        self.blk = np.zeros(n, dtype=np.uint32)
        self.have = np.zeros(n, dtype=np.int64)
        self.x = np.zeros((n, 4), dtype=np.uint32)
        self.stats = stats

    def _mask(self, active):
        return np.ones(len(self.c0), dtype=bool) if active is None else np.asarray(active, dtype=bool)

    def next(self, active=None) -> np.ndarray:
        """One word per active lane (0 in the others, whose streams do not move)."""
        active = self._mask(active)
        refill = np.nonzero(active & (self.have == 0))[0]
        if len(refill):
            x = mc_ref.philox4x32_10(self.c0[refill], self.c1, self.c2, self.blk[refill], self.k0, self.k1)
            self.x[refill] = np.stack(x, axis=1)
            self.blk[refill] += np.uint32(1)
            self.have[refill] = 4
        lanes = np.nonzero(active)[0]
        self.have[lanes] -= 1
        w = np.zeros(len(self.c0), dtype=np.uint32)
        w[lanes] = self.x[lanes, self.have[lanes]]
        return w

    def uniform(self, active=None) -> np.ndarray:
        """[0, 1) with 53 bits: the high 27 from the first word drawn, the low 26 from the second."""
        active = self._mask(active)
        if self.stats is not None:
            self.stats.straddles += int(np.count_nonzero(active & (self.have == 1)))
        hi = (self.next(active) >> np.uint32(5)).astype(np.float64)
        lo = (self.next(active) >> np.uint32(6)).astype(np.float64)
        return (hi * _2P26 + lo) * _2M53

    def below(self, n: int, active=None) -> np.ndarray:
        """(word * n) >> 32: an integer in [0, n)."""
        return ((self.next(active).astype(np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def _ranges(lo, hi, is_int):
    return np.asarray(lo, np.float64), np.asarray(hi, np.float64), np.asarray(is_int, dtype=bool)


def init(params, n_seeded: int, lo, hi, is_int, seed: int, stats: Optional[Stats] = None) -> np.ndarray:
    """ga_init_kernel: rows < n_seeded are params clamped to the ranges; the others are drawn from stream INIT at
    generation 0, gene by gene: integer genes lo + below(int(hi - lo) + 1), float genes fma(hi - lo, u, lo)."""
    lo, hi, is_int = _ranges(lo, hi, is_int)
    params = np.asarray(params, dtype=np.float64)
    pop, genes = params.shape
    out = params.copy()
    out[:n_seeded] = clamp(params[:n_seeded], lo, hi)
    rng = Words(seed, 0, np.arange(n_seeded, pop), INIT, stats)
    for g in range(genes):
        span = hi[g] - lo[g]
        if is_int[g]:
            out[n_seeded:, g] = lo[g] + rng.below(int(span) + 1).astype(np.float64)
        else:
            u = rng.uniform()
            v = fma_array(span, u, lo[g])
            if stats is not None:
                stats.fma_init += int(np.count_nonzero(v != lo[g] + span * u))
            out[n_seeded:, g] = v
    return out


def elite_count(elitism_pct: float, pop: int) -> int:
    return min(pop, max(1, int(elitism_pct * pop)))


def tournaments(fitness, pop: int, n_elite: int, tournament: int, seed: int, generation: int,
                stats: Optional[Stats] = None):
    """Contenders [pop - n_elite][tournament] of slots n_elite.. and the winners: rejection-sampled distinct
    contenders from stream SELECT, the first maximum wins (strict >)."""
    fitness = np.asarray(fitness, dtype=np.float64)
    m = pop - n_elite
    rng = Words(seed, generation, np.arange(n_elite, pop), SELECT, stats)
    picks = np.full((m, tournament), -1, dtype=np.int64)
    best = np.full(m, -1, dtype=np.int64)
    best_fit = np.zeros(m)
    for t in range(tournament):
        pending = np.ones(m, dtype=bool)
        cand = np.zeros(m, dtype=np.int64)
        while pending.any():
            c = rng.below(pop, pending)
            cand = np.where(pending, c, cand)
            repeated = (picks[:, :t] == cand[:, None]).any(axis=1)
            if stats is not None:
                stats.rejections += int(np.count_nonzero(pending & repeated))
            pending &= repeated
        picks[:, t] = cand
        f = fitness[cand]
        take = (best < 0) | (f > best_fit)
        best = np.where(take, cand, best)
        best_fit = np.where(take, f, best_fit)
    return picks, best


def select(fitness, ranked, pop: int, n_elite: int, tournament: int, seed: int, generation: int,
           stats: Optional[Stats] = None) -> np.ndarray:
    """ga_select_kernel: sel[j] = ranked[j] for j < n_elite, else the slot's tournament winner."""
    sel = np.empty(pop, dtype=np.int32)
    sel[:n_elite] = np.asarray(ranked)[:n_elite]
    sel[n_elite:] = tournaments(fitness, pop, n_elite, tournament, seed, generation, stats)[1]
    return sel


def breed(params, sel, n_elite: int, lo, hi, is_int, crossover_rate: float, mutation_rate: float, seed: int,
          generation: int, stats: Optional[Stats] = None) -> np.ndarray:
    """ga_breed_kernel: elites copied; pair q makes slots n_elite + 2q (child a) and n_elite + 2q + 1 (child b, dropped
    past pop).  Stream PARENTS of q: p1, p2 = sel[below(pop)] twice, then cross = !(u > crossover_rate).  Both children
    read the coin stream COINS of q (child a takes p1 where the coin is < 0.5, b the other parent); each child mutates
    from the stream MUTATION of its own slot."""
    lo, hi, is_int = _ranges(lo, hi, is_int)
    params = np.asarray(params, dtype=np.float64)
    sel = np.asarray(sel, dtype=np.int64)
    pop, genes = params.shape
    out = np.empty_like(params)
    out[:n_elite] = params[sel[:n_elite]]
    n_pairs = (pop - n_elite + 1) // 2
    q = np.arange(n_pairs)
    pr = Words(seed, generation, q, PARENTS, stats)
    p1 = params[sel[pr.below(pop)]]
    p2 = params[sel[pr.below(pop)]]
    cross = ~(pr.uniform() > crossover_rate)
    for child in (0, 1):
        slots = n_elite + 2 * q + child
        keep = slots < pop
        qs, slots, a, b, cx = q[keep], slots[keep], p1[keep], p2[keep], cross[keep]
        coin = Words(seed, generation, qs, COINS, stats)
        mut = Words(seed, generation, slots, MUTATION, stats)
        for g in range(genes):
            first = coin.uniform() < 0.5
            own = a[:, g] if child == 0 else b[:, g]
            v = np.where(~cx, own, np.where(first == (child == 0), a[:, g], b[:, g]))
            m = mut.uniform() < mutation_rate
            if is_int[g]:
                step = max(1.0, float(np.floor((hi[g] - lo[g]) * 0.1)))
                up = (mut.next(m) & np.uint32(1)) != 0
                new = v + np.where(up, step, -step)
            else:
                scale = mut.uniform(m) < 0.5
                u = mut.uniform(m)
                span = hi[g] - lo[g]
                new = v.copy()
                for lanes, fused, plain in (
                        (m & scale, lambda i: v[i] * fma_array(u[i], 0.4, 0.8), lambda i: v[i] * (0.8 + 0.4 * u[i])),
                        (m & ~scale, lambda i: fma_array((2.0 * u[i] - 1.0) * 0.1, span, v[i]),
                         lambda i: v[i] + (2.0 * u[i] - 1.0) * 0.1 * span)):
                    i = np.nonzero(lanes)[0]
                    new[i] = fused(i)
                    if stats is not None:
                        stats.fma_mutation += int(np.count_nonzero(clamp(new[i], lo[g], hi[g]) !=
                                                                   clamp(plain(i), lo[g], hi[g])))
            if stats is not None:
                stats.mutated += int(np.count_nonzero(m))
            out[slots, g] = np.where(m, clamp(new, lo[g], hi[g]), v)
    return out


def next_generation(params, fitness, ranked, lo, hi, is_int, elitism_pct: float, tournament: int,
                    crossover_rate: float, mutation_rate: float, seed: int, generation: int,
                    stats: Optional[Stats] = None):
    """b200bt_ga_next_generation -> (sel int32 [pop], params_out float64 [pop][genes])."""
    params = np.asarray(params, dtype=np.float64)
    pop = params.shape[0]
    n_elite = elite_count(elitism_pct, pop)
    sel = select(fitness, ranked, pop, n_elite, tournament, seed, generation, stats)
    return sel, breed(params, sel, n_elite, lo, hi, is_int, crossover_rate, mutation_rate, seed, generation, stats)


def rank(scores) -> np.ndarray:
    """DeviceGeneticAlgorithm's ranking: NaN -> -inf, then a stable descending argsort.  -> (key, ranked)"""
    key = np.asarray(scores, dtype=np.float64)
    key = np.where(np.isnan(key), -np.inf, key)
    return key, np.argsort(-key, kind="stable").astype(np.int32)


def _is_int_range(lo, hi) -> bool:
    return isinstance(lo, int) and isinstance(hi, int)


@dataclass
class Run:
    params: List[np.ndarray] = field(default_factory=list)      # generation 0..G, as evaluated
    sel: List[np.ndarray] = field(default_factory=list)         # generation 1..G
    fitness: List[List[float]] = field(default_factory=list)    # generation 0..G
    history: List[Dict] = field(default_factory=list)           # generation_history without the timestamps
    best_individual: Optional[Dict] = None
    best_fitness: float = float("-inf")


def run(param_ranges: Dict, batch_fitness: Callable, population_size: int = 20, generations: int = 10,
        mutation_rate: float = 0.2, crossover_rate: float = 0.8, elitism_pct: float = 0.1, tournament_size: int = 3,
        random_seed: Optional[int] = None, seeded_individuals: Optional[List[Dict]] = None,
        stats: Optional[Stats] = None) -> Run:
    """DeviceGeneticAlgorithm(param_ranges, batch_fitness, ...).run(seeded_individuals), restated."""
    seed = int(random_seed or 0) & 0xFFFFFFFFFFFFFFFF
    names = list(param_ranges)
    lo = np.array([float(param_ranges[n][0]) for n in names])
    hi = np.array([float(param_ranges[n][1]) for n in names])
    is_int = np.array([_is_int_range(*param_ranges[n]) for n in names])
    pop = int(population_size)
    params = np.zeros((pop, len(names)))
    seeded = list(seeded_individuals or [])[:pop]
    if seeded:
        params[:len(seeded)] = [[float(ind.get(n, param_ranges[n][0])) for n in names] for ind in seeded]
    params = init(params, len(seeded), lo, hi, is_int, seed, stats)
    out = Run()

    def to_dicts(matrix):
        cols = [matrix[:, g].astype(np.int64).tolist() if is_int[g] else matrix[:, g].tolist() for g in range(len(names))]
        return [dict(zip(names, row)) for row in zip(*cols)]

    def evaluate_and_record(generation):
        population = to_dicts(params)
        scores = [float(x) for x in batch_fitness(population)]
        for ind, fit in zip(population, scores):
            if fit > out.best_fitness:
                out.best_fitness, out.best_individual = fit, dict(ind)
        top = max(scores)
        spans = hi - lo
        keep = spans != 0
        diversity = 0.0 if pop < 2 or not keep.any() else \
            float(np.mean(np.var((params[:, keep] - lo[keep]) / spans[keep], axis=0)))
        out.params.append(params.copy())
        out.fitness.append(scores)
        out.history.append({"generation": generation, "best_fitness": top, "avg_fitness": sum(scores) / len(scores),
                            "min_fitness": min(scores), "best_individual": dict(population[scores.index(top)]),
                            "diversity": diversity})
        return scores

    scores = evaluate_and_record(0)
    for generation in range(1, generations + 1):
        key, ranked = rank(scores)
        sel, params = next_generation(params, key, ranked, lo, hi, is_int, elitism_pct, tournament_size,
                                      crossover_rate, mutation_rate, seed, generation, stats)
        out.sel.append(sel)
        scores = evaluate_and_record(generation)
    return out
