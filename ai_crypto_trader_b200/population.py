"""Population plumbing shared by the GA-facing sweeps.

    unique_rows        first occurrences of a population's decoded records, and the index that expands results back
    calendar_days      the calendar days a series spans (the per-day row length of b200bt_cscv)
    fitness_callable   GeneticAlgorithm's fitness_function of a batch evaluator
    StrategySweep      the evaluator of the grid and DCA sweeps: dedup and upload, objectives, stats views, day rows
"""
from __future__ import annotations

from datetime import datetime, timedelta, timezone
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

_HASH_MULTIPLIERS = np.array([0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x27D4EB2F165667C5,
                              0x85EBCA77C2B2AE63], dtype=np.uint64)


def unique_rows(records: np.ndarray) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """(keep, expand) of C-contiguous records, one per row, each a multiple of 8 bytes: keep = the index of the first
    occurrence of every distinct row, in population order; expand[i] = the position in keep of row i's first occurrence,
    or None when every row is distinct.  Rows are equal when their bytes are.  They are compared through a 64-bit
    multiplicative hash of their uint64 words (much faster than sorting wide rows); a hash class is only trusted after
    every member is compared with its first, and a collision falls back to sorting the rows."""
    n = len(records)
    words = records.view(np.uint8).reshape(n, -1).view(np.uint64)
    mult = np.resize(_HASH_MULTIPLIERS, words.shape[1])
    with np.errstate(over="ignore"):
        key = (words * mult).sum(axis=1, dtype=np.uint64)
    _, first, inverse = np.unique(key, return_index=True, return_inverse=True)
    if len(first) < n and not np.array_equal(words[first][inverse.reshape(-1)], words):     # a collision: exact path
        _, first, inverse = np.unique(words, axis=0, return_index=True, return_inverse=True)
    if len(first) == n:
        return np.arange(n), None
    rank = np.empty(len(first), dtype=np.int64)
    rank[np.argsort(first)] = np.arange(len(first))
    return np.sort(first), rank[inverse.reshape(-1)]


def calendar_days(minute0: int, bar_minutes: int, N: int, gap_bar: int = 0, gap_minutes: int = 0) -> Tuple[int, int]:
    """(first_day, D): the calendar day of bar 0 (days since 1970-01-01 of the minute clock) and the number of days from
    it to the day of bar N - 1, the skipped days of a glued series (gap_minutes skipped before bar gap_bar > 0) included."""
    last = N - 1
    first = minute0 // 1440
    gap = gap_minutes if (gap_bar > 0 and last >= gap_bar) else 0
    return first, (minute0 + last * bar_minutes + gap) // 1440 - first + 1


def fitness_callable(evaluate: Callable[[List[Dict]], np.ndarray]) -> Callable[[Dict], float]:
    """fitness(individual) -> float through a batch evaluator, with a .batch attribute that evaluates a whole population
    in one call (GeneticAlgorithm uses it when present)."""

    def fitness(individual: Dict) -> float:
        return float(evaluate([individual])[0])

    fitness.batch = lambda population: [float(x) for x in evaluate(population)]
    return fitness


def iso_minute(minute: int) -> str:
    """The naive ISO timestamp of a Unix minute, as the services print their times."""
    return (datetime(1970, 1, 1, tzinfo=timezone.utc) + timedelta(minutes=int(minute))).replace(tzinfo=None).isoformat()


class StrategySweep:
    """The population evaluator of a strategy whose kernel writes a 20-word stats record per (individual, symbol) and,
    as a service, one service record per individual.  A subclass sets

        FIELDS, SERVICE_FIELDS        the names of the stats and service record words
        OBJECTIVE_FIELDS              the stats fields an objective may name (mean over the symbols)
        SERVICE_OBJECTIVE_FIELDS      the service fields an objective may name
        service                       whether the sweep writes service records

    and implements _inputs(population) -> ([per-individual arrays, first axis the population], {launch keywords}) and
    launch(*device arrays, stats, service, rows, **keywords), its entry point on the current stream.  The sweep
    uploads and evaluates each distinct individual once: individuals whose arrays are byte-equal decode alike."""

    SERVICE_OBJECTIVE_FIELDS: Tuple[str, ...] = ()
    service = False
    _stats = _service = _inverse = None

    def _column(self, name: str) -> Tuple[str, int]:
        if name in self.OBJECTIVE_FIELDS:
            return "stats", self.OBJECTIVE_FIELDS.index(name)
        if name in self.SERVICE_OBJECTIVE_FIELDS:
            return "service", self.SERVICE_FIELDS.index(name)
        names = [*self.OBJECTIVE_FIELDS, *self.SERVICE_OBJECTIVE_FIELDS]
        raise ValueError(f"{name!r} is not an objective of {type(self).__name__}; one of {', '.join(names)}")

    def _run(self, population: List[Dict], day: bool = False):
        if not population:
            raise ValueError("an empty population")
        m = self.market
        arrays, extra = self._inputs(population)
        keep, expand = unique_rows(np.concatenate([a.reshape(len(population), -1).view(np.uint8) for a in arrays], axis=1))
        U = len(keep)
        inputs = [torch.from_numpy(np.ascontiguousarray(a[keep])).to(m.device) for a in arrays]
        stats = torch.empty((U, m.S, len(self.FIELDS)), dtype=torch.float64, device=m.device)
        service = torch.empty((U, len(self.SERVICE_FIELDS)), dtype=torch.float64, device=m.device) if self.service else None
        rows = torch.empty((U, self.calendar_days()[1]), dtype=torch.float64, device=m.device) if day else None
        with torch.cuda.device(m.device):
            self.launch(*inputs, stats, service, rows, **extra)
        self._stats, self._service, self._inverse = stats, service, expand
        return stats, service, rows

    def calendar_days(self) -> Tuple[int, int]:
        """(first_day, D): the calendar day of bar 0 (days since 1970-01-01) and the days from it to the last bar's."""
        m = self.market
        return calendar_days(m.minute0, m.bar_minutes, m.N)

    def _expand(self, t: torch.Tensor) -> torch.Tensor:
        return t if self._inverse is None else t.index_select(0, torch.from_numpy(self._inverse).to(t.device))

    def evaluate(self, population: List[Dict]) -> np.ndarray:
        """fitness float64 [pop]: the `objective` (a stats field's mean over the symbols, or a service field)."""
        if not population:
            return np.zeros(0, dtype=np.float64)
        return self.evaluate_objectives_device(population, [(self.objective, True)])[:, 0].cpu().numpy()

    def evaluate_objectives_device(self, population: List[Dict], objectives) -> torch.Tensor:
        """Objective matrix float64 [pop][M] on the device for ParetoGeneticAlgorithm: per objective (field, maximize)
        a stats field's mean over the symbols (b200bt_objective_matrix, which reads the 20-word stats records as it reads
        lane stats) or a service field, in the field's own sense."""
        from .pareto import objective_matrix
        objectives = list(objectives)
        cols = [self._column(name) for name, _ in objectives]
        M = len(cols)
        if not 1 <= M <= 8:
            raise ValueError("1..8 objectives")
        if not population:
            return torch.zeros((0, M), dtype=torch.float64, device=self.market.device)
        stats, service, _ = self._run(population)
        means = [(name, True) for (name, _), (kind, _) in zip(objectives, cols) if kind == "stats"]
        if means:
            means = objective_matrix(stats, means, fields=self.OBJECTIVE_FIELDS)
        out, j = [], 0
        for kind, f in cols:
            if kind == "stats":
                out.append(means[:, j])
                j += 1
            else:
                out.append(service[:, f])
        return self._expand(torch.stack(out, dim=1))

    def evaluate_objectives(self, population: List[Dict], objectives) -> np.ndarray:
        return self.evaluate_objectives_device(population, objectives).cpu().numpy()

    def stats_dict(self, population: Optional[List[Dict]] = None) -> Dict[str, np.ndarray]:
        """dict field -> [pop][S] float64 of `population` (evaluated now) or of the last evaluation."""
        if population is not None:
            self._run(population)
        if self._stats is None:
            raise RuntimeError("nothing evaluated yet")
        raw = self._expand(self._stats).cpu().numpy()
        return {name: raw[:, :, f] for f, name in enumerate(self.FIELDS)}

    def service_stats(self, population: Optional[List[Dict]] = None) -> Dict[str, np.ndarray]:
        """dict field -> [pop] float64 of the service records of `population` (evaluated now) or of the last
        evaluation."""
        if not self.service:
            raise RuntimeError(f"service_stats() needs {type(self).__name__}(..., service=True)")
        if population is not None:
            self._run(population)
        if self._service is None:
            raise RuntimeError("nothing evaluated yet")
        raw = self._expand(self._service).cpu().numpy()
        return {name: raw[:, f] for f, name in enumerate(self.SERVICE_FIELDS)}

    def stats_device(self) -> torch.Tensor:
        """The last evaluation's stats float64 [pop][S][20] on the device, in population order."""
        return self._expand(self._stats)

    def day_rows(self, population: List[Dict]) -> Tuple[torch.Tensor, int]:
        """(rows float64 [pop][D] on the device, first_day): the kernel's per-day rows of `population`, column d =
        calendar day first_day + d -- the row shape b200bt_cscv takes."""
        _, _, rows = self._run(population, day=True)
        return self._expand(rows), self.calendar_days()[0]

    @property
    def fitness_function(self):
        return fitness_callable(self.evaluate)
