"""GeneticAlgorithm with the reference's call surface and a batched fitness hook.

Reference: services/genetic_algorithm.py (class GeneticAlgorithm, :27-393).  Same
constructor, attributes (`population`, `fitness_scores`, `best_individual`,
`best_fitness`, `generation_history`) and methods.  The operators draw from the
global `random` module in exactly the reference's order, so a seeded run
reproduces the reference's trajectory individual for individual (pinned by
tests/golden/ga_run.json, produced by running the reference class).

New, backward compatible: if `fitness_function` has a `.batch` attribute (or
`batch_fitness_function=` is given), `evaluate_population` calls it ONCE with the
whole population (List[Dict] -> sequence of floats) instead of looping over
individuals (:124) -- that one call is the GPU population sweep.
"""
from __future__ import annotations

import logging
import random
from datetime import datetime
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

logger = logging.getLogger("b200bt.genetic_algorithm")


def _is_int_range(lo, hi) -> bool:
    return isinstance(lo, int) and isinstance(hi, int)


class GeneticAlgorithm:
    def __init__(self, param_ranges: Dict[str, Tuple], fitness_function: Callable, population_size: int = 20,
                 generations: int = 10, mutation_rate: float = 0.2, crossover_rate: float = 0.8,
                 elitism_pct: float = 0.1, tournament_size: int = 3, random_seed: Optional[int] = None,
                 batch_fitness_function: Optional[Callable[[List[Dict]], Sequence[float]]] = None):
        self.param_ranges = param_ranges
        self.fitness_function = fitness_function
        self.batch_fitness_function = batch_fitness_function or getattr(fitness_function, "batch", None)
        self.population_size = population_size
        self.generations = generations
        self.mutation_rate = mutation_rate
        self.crossover_rate = crossover_rate
        self.elitism_pct = elitism_pct
        self.tournament_size = tournament_size
        if random_seed is not None:           # :65-67
            random.seed(random_seed)
            np.random.seed(random_seed)
        self.population: List[Dict] = []
        self.fitness_scores: List[float] = []
        self.best_individual: Optional[Dict] = None
        self.best_fitness = -float("inf")
        self.generation_history: List[Dict] = []

    # -- population ---------------------------------------------------------------
    def initialize_population(self, seeded_individuals: List[Dict] = None) -> None:
        self.population = []
        for given in seeded_individuals or []:       # clamp seeds into range (:94-104)
            clamped = {}
            for name, value in given.items():
                if name in self.param_ranges:
                    lo, hi = self.param_ranges[name]
                    clamped[name] = max(lo, min(hi, value))
                else:
                    clamped[name] = value
            self.population.append(clamped)
        for _ in range(self.population_size - len(self.population)):
            self.population.append({name: (random.randint(lo, hi) if _is_int_range(lo, hi) else random.uniform(lo, hi))
                                    for name, (lo, hi) in self.param_ranges.items()})

    def evaluate_population(self) -> None:
        if self.batch_fitness_function is not None:
            scores = [float(x) for x in self.batch_fitness_function(self.population)]
            if len(scores) != len(self.population):
                raise ValueError("batch fitness returned %d scores for %d individuals" % (len(scores), len(self.population)))
        else:
            scores = [self.fitness_function(ind) for ind in self.population]      # :124 serial form
        self.fitness_scores = scores
        for ind, fit in zip(self.population, scores):                             # strict '>' keeps the first best (:129)
            if fit > self.best_fitness:
                self.best_fitness = fit
                self.best_individual = dict(ind)

    # -- operators (random-call order identical to the reference) ----------------------
    def _elites_count(self) -> int:
        return max(1, int(self.elitism_pct * self.population_size))

    def selection(self) -> List[Dict]:
        ranked = sorted(range(len(self.fitness_scores)), key=lambda i: self.fitness_scores[i], reverse=True)
        chosen = [dict(self.population[i]) for i in ranked[:self._elites_count()]]
        n = len(self.population)
        while len(chosen) < self.population_size:
            contenders = random.sample(range(n), self.tournament_size)
            fits = [self.fitness_scores[i] for i in contenders]
            chosen.append(dict(self.population[contenders[fits.index(max(fits))]]))   # first max wins (:158)
        return chosen

    def crossover(self, parent1: Dict, parent2: Dict) -> Tuple[Dict, Dict]:
        if random.random() > self.crossover_rate:
            return dict(parent1), dict(parent2)
        a, b = {}, {}
        for name in self.param_ranges:               # uniform crossover, one draw per gene (:180-186)
            if random.random() < 0.5:
                a[name], b[name] = parent1[name], parent2[name]
            else:
                a[name], b[name] = parent2[name], parent1[name]
        return a, b

    def mutation(self, individual: Dict) -> Dict:
        out = dict(individual)
        for name, (lo, hi) in self.param_ranges.items():
            if random.random() < self.mutation_rate:
                if _is_int_range(lo, hi):
                    step = max(1, int((hi - lo) * 0.1))
                    out[name] = max(lo, min(hi, out[name] + random.choice([-step, step])))
                elif random.random() < 0.5:
                    out[name] = max(lo, min(hi, out[name] * random.uniform(0.8, 1.2)))
                else:
                    span = hi - lo
                    out[name] = max(lo, min(hi, out[name] + random.uniform(-0.1 * span, 0.1 * span)))
        return out

    def evolve_generation(self) -> None:
        selected = self.selection()
        nxt = list(selected[:self._elites_count()])
        while len(nxt) < self.population_size:
            p1 = random.choice(selected)
            p2 = random.choice(selected)
            c1, c2 = self.crossover(p1, p2)
            c1 = self.mutation(c1)
            c2 = self.mutation(c2)
            nxt.append(c1)
            if len(nxt) < self.population_size:
                nxt.append(c2)
        self.population = nxt

    # -- driver -------------------------------------------------------------------
    def run(self, seeded_individuals: List[Dict] = None) -> Dict:
        self.initialize_population(seeded_individuals)
        self.evaluate_population()
        self.record_generation(0)
        for generation in range(1, self.generations + 1):
            self.evolve_generation()
            self.evaluate_population()
            self.record_generation(generation)
        return self.best_individual

    def record_generation(self, generation: int) -> None:
        scores = self.fitness_scores
        top = max(scores)
        self.generation_history.append({
            "generation": generation,
            "timestamp": datetime.now().isoformat(),
            "best_fitness": top,
            "avg_fitness": sum(scores) / len(scores),
            "min_fitness": min(scores),
            "best_individual": dict(self.population[scores.index(top)]),
            "diversity": self.calculate_diversity(),
        })

    def _normalised_variances(self) -> Dict[str, float]:
        out = {}
        for name, (lo, hi) in self.param_ranges.items():
            span = hi - lo
            if span == 0:
                continue
            out[name] = float(np.var([(ind[name] - lo) / span for ind in self.population]))
        return out

    def calculate_diversity(self) -> float:
        if not self.population or len(self.population) < 2:
            return 0.0
        return float(np.mean(list(self._normalised_variances().values())))

    def get_generation_history(self) -> List[Dict]:
        return self.generation_history

    def get_best_individual(self) -> Dict:
        return dict(self.best_individual)

    def get_population_diversity(self) -> Dict:
        per_param = self._normalised_variances()
        for name, (lo, hi) in self.param_ranges.items():
            if hi - lo == 0:
                per_param[name] = 0.0
        return {"overall": self.calculate_diversity(), "parameters": {k: per_param[k] for k in self.param_ranges}}


class DeviceGeneticAlgorithm:
    """The same GA with its operators on the GPU (csrc/ga_ops.cu, SURVEY 8-f2): one launch per generation instead of
    a Python loop over individuals (0.1 s per generation at 10 000 individuals on the host).

    Same constructor arguments, attributes and `run()` contract as GeneticAlgorithm; the fitness must be a BATCH
    callable (List[Dict] -> sequence of floats, e.g. `PopulationSweep.evaluate` or `ShardedFitness(...).batch`).
    Differences a caller can see: the random stream is Philox keyed by `random_seed` (default 0), so trajectories
    are reproducible but not equal to the reference's Mersenne-twister ones -- the operators and their probabilities
    are (genetic_algorithm.py:83-252); NaN fitness ranks below every number.
    """

    def __init__(self, param_ranges: Dict[str, Tuple], batch_fitness_function: Callable[[List[Dict]], List[float]],
                 population_size: int = 20, generations: int = 10, mutation_rate: float = 0.2,
                 crossover_rate: float = 0.8, elitism_pct: float = 0.1, tournament_size: int = 3,
                 random_seed: Optional[int] = None, device=None):
        import torch
        from . import _lib
        self._torch, self._lib = torch, _lib
        if not torch.cuda.is_available():
            raise RuntimeError("DeviceGeneticAlgorithm needs a CUDA device (sm_90); use GeneticAlgorithm on the host")
        self.param_ranges = param_ranges
        self.batch_fitness_function = getattr(batch_fitness_function, "batch", batch_fitness_function)
        self.population_size, self.generations = int(population_size), int(generations)
        self.mutation_rate, self.crossover_rate = float(mutation_rate), float(crossover_rate)
        self.elitism_pct, self.tournament_size = float(elitism_pct), int(tournament_size)
        self.seed = int(random_seed or 0) & 0xFFFFFFFFFFFFFFFF
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.names = list(param_ranges)
        G = len(self.names)
        import ctypes as C
        self._lo = (C.c_double * G)(*[float(param_ranges[n][0]) for n in self.names])
        self._hi = (C.c_double * G)(*[float(param_ranges[n][1]) for n in self.names])
        self._is_int = (C.c_int * G)(*[1 if _is_int_range(*param_ranges[n]) else 0 for n in self.names])
        self.params = torch.zeros((self.population_size, G), dtype=torch.float64, device=self.device)
        self._next = torch.empty_like(self.params)
        self._sel = torch.empty(self.population_size, dtype=torch.int32, device=self.device)
        self.population: List[Dict] = []
        self.fitness_scores: List[float] = []
        self.best_individual: Optional[Dict] = None
        self.best_fitness = float("-inf")
        self.generation_history: List[Dict] = []

    # -- matrix <-> reference representation --------------------------------------------------------
    def _to_dicts(self, matrix: np.ndarray) -> List[Dict]:
        cols = [matrix[:, g].astype(np.int64).tolist() if self._is_int[g] else matrix[:, g].tolist()
                for g in range(len(self.names))]
        return [dict(zip(self.names, row)) for row in zip(*cols)]

    def initialize_population(self, seeded_individuals: Optional[List[Dict]] = None) -> None:
        torch, lib = self._torch, self._lib
        seeded = list(seeded_individuals or [])[:self.population_size]
        if seeded:
            rows = np.array([[float(ind.get(n, self.param_ranges[n][0])) for n in self.names] for ind in seeded])
            self.params[:len(seeded)] = torch.from_numpy(rows).to(self.device)
        with torch.cuda.device(self.device):
            lib.call("b200bt_ga_init", self.params.data_ptr(), self.population_size, len(self.names), len(seeded),
                     self._lo, self._hi, self._is_int, self.seed, lib.current_stream())

    def evaluate_population(self) -> None:
        host = self.params.cpu().numpy()
        self.population = self._to_dicts(host)
        scores = [float(x) for x in self.batch_fitness_function(self.population)]
        if len(scores) != self.population_size:
            raise ValueError("batch fitness returned %d scores for %d individuals" % (len(scores), self.population_size))
        self.fitness_scores = scores
        for ind, fit in zip(self.population, scores):
            if fit > self.best_fitness:
                self.best_fitness, self.best_individual = fit, dict(ind)

    def evolve_generation(self, generation: int) -> None:
        torch, lib = self._torch, self._lib
        fit = torch.tensor(self.fitness_scores, dtype=torch.float64, device=self.device)
        key = torch.where(torch.isnan(fit), torch.full_like(fit, float("-inf")), fit)
        ranked = torch.argsort(key, descending=True, stable=True).to(torch.int32)
        with torch.cuda.device(self.device):
            lib.call("b200bt_ga_next_generation", self.params.data_ptr(), key.data_ptr(), ranked.data_ptr(),
                     self.population_size, len(self.names), self._lo, self._hi, self._is_int, self.elitism_pct,
                     self.tournament_size, self.crossover_rate, self.mutation_rate, self.seed, int(generation),
                     self._sel.data_ptr(), self._next.data_ptr(), lib.current_stream())
        self.params, self._next = self._next, self.params

    def record_generation(self, generation: int) -> None:
        scores = self.fitness_scores
        top = max(scores)
        self.generation_history.append({
            "generation": generation, "timestamp": datetime.now().isoformat(), "best_fitness": top,
            "avg_fitness": sum(scores) / len(scores), "min_fitness": min(scores),
            "best_individual": dict(self.population[scores.index(top)]), "diversity": self.calculate_diversity()})

    def calculate_diversity(self) -> float:
        if self.population_size < 2:
            return 0.0
        host = self.params.cpu().numpy()
        spans = np.array([self._hi[g] - self._lo[g] for g in range(len(self.names))])
        keep = spans != 0
        if not keep.any():
            return 0.0
        norm = (host[:, keep] - np.array(list(self._lo))[keep]) / spans[keep]
        return float(np.mean(np.var(norm, axis=0)))

    def run(self, seeded_individuals: Optional[List[Dict]] = None) -> Dict:
        self.initialize_population(seeded_individuals)
        self.evaluate_population()
        self.record_generation(0)
        for generation in range(1, self.generations + 1):
            self.evolve_generation(generation)
            self.evaluate_population()
            self.record_generation(generation)
        return self.best_individual

    def get_generation_history(self) -> List[Dict]:
        return self.generation_history

    def get_best_individual(self) -> Dict:
        return dict(self.best_individual)
