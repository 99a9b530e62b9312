"""Multi-objective ranking on the GPU: non-dominated fronts, crowding distance and the crowded order (NSGA-II; Deb,
Pratap, Agarwal, Meyarivan 2002), and the objectives of the reference's optimisation goals.

The reference states its goal as several metrics (config.json evolution.optimization_goals: a primary metric and
secondary ones) and multiplies them into one score (_calculate_strategy_score, services/strategy_evaluation.py:579-633).
A Pareto front keeps the trade-off instead: every strategy that no other beats in all the metrics at once.

pareto_rank            b200bt_pareto_rank on a device [n][M] float64 matrix (contract: include/b200bt.h)
objectives_from_goals  goals dict -> [(lane-stat field, maximize)]
objective_matrix       b200bt_objective_matrix: the per-individual mean over symbols of lane-stat (or other stats) fields
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib

MAX_POINTS = 65536
MAX_OBJECTIVES = 8

# lane-stat fields where smaller is better; every other field is maximised
MINIMISED = frozenset({"max_drawdown", "n_losses", "n_negative_days", "downside_deviation"})
OBJECTIVE_FIELDS = _lib.LANE_STATS_FIELDS[:-1]          # trade_hash is a hash, not a metric

Objective = Tuple[str, bool]


def _field(name: str, fields: Sequence[str] = OBJECTIVE_FIELDS) -> int:
    if name not in fields:
        raise ValueError(f"{name!r} is not a stats field; objectives are one of {', '.join(fields)}")
    return fields.index(name)


def objectives_from_goals(goals: Union[Dict, Sequence]) -> List[Objective]:
    """[(field, maximize)] of an optimisation-goals dict ({"primary": name, "secondary": [names]}, the keys
    _lib.score_codes reads): the primary first, then the secondaries in their order, duplicates dropped.  A minimised
    field (MINIMISED) gets maximize = False, every other one True.  A sequence of names and (name, "min" | "max") pairs
    is accepted too; an explicit direction overrides the mapping.  A name that is not a lane-stat field raises
    ValueError: unlike the scalar score, a missing metric is never silently 0."""
    if isinstance(goals, dict):
        items = [goals.get("primary", "sharpe_ratio"), *goals.get("secondary", [])]
    else:
        items = list(goals)
    out: List[Objective] = []
    seen = set()
    for item in items:
        if isinstance(item, str):
            name, maximize = item, item not in MINIMISED
        else:
            name, sense = item
            if sense not in ("min", "max"):
                raise ValueError(f"direction of {name!r} must be 'min' or 'max', not {sense!r}")
            maximize = sense == "max"
        _field(name)
        if name in seen:
            continue
        seen.add(name)
        out.append((name, maximize))
    if not out:
        raise ValueError("no objectives")
    if len(out) > MAX_OBJECTIVES:
        raise ValueError(f"at most {MAX_OBJECTIVES} objectives ({len(out)} given)")
    return out


def objective_matrix(stats: torch.Tensor, objectives: Sequence[Objective], out: Optional[torch.Tensor] = None,
                     fields: Sequence[str] = OBJECTIVE_FIELDS) -> torch.Tensor:
    """b200bt_objective_matrix: [pop][M] float64 on the device, out[i][j] = mean over the S symbols of stats[i][s].<field j>
    (the ascending sum of b200bt_fitness_reduce), in the metric's own sense.  stats: device [pop][S][20] float64 lane stats,
    or [pop][20] book stats; `fields` names the record's words (another 20-word stats record, such as the grid's or the
    DCA's, passes its own names)."""
    if not (isinstance(stats, torch.Tensor) and stats.is_cuda and stats.dtype == torch.float64):
        raise TypeError("objective_matrix: stats must be a float64 CUDA tensor")
    if stats.dim() == 2:
        stats = stats.unsqueeze(1)
    if stats.dim() != 3 or stats.shape[-1] != _lib.LANE_STATS_WORDS:
        raise ValueError(f"objective_matrix: stats must be [pop][S][{_lib.LANE_STATS_WORDS}] or [pop][{_lib.LANE_STATS_WORDS}], "
                         f"not {tuple(stats.shape)}")
    stats = stats.contiguous()
    pop, S = stats.shape[0], stats.shape[1]
    M = len(objectives)
    index = (C.c_int * M)(*[_field(name, fields) for name, _ in objectives])
    if out is None:
        out = torch.empty((pop, M), dtype=torch.float64, device=stats.device)
    elif not (isinstance(out, torch.Tensor) and out.device == stats.device and out.dtype == torch.float64 and
              tuple(out.shape) == (pop, M) and (pop == 1 or out.stride(1) == 1)):
        raise ValueError(f"objective_matrix: out must be a float64 [{pop}][{M}] tensor with unit column stride on "
                         f"{stats.device}")
    with torch.cuda.device(stats.device):
        _lib.call("b200bt_objective_matrix", stats.data_ptr(), pop, S, index, M, out.data_ptr(), _lib.ld(out),
                  _lib.current_stream())
    return out


class ParetoRanker:
    """b200bt_pareto_rank with its workspace kept between calls of the same size."""

    def __init__(self):
        self._ws = None
        self._ws_key = None

    def workspace(self, n: int, M: int, device) -> torch.Tensor:
        need = int(_lib.load().b200bt_pareto_workspace_bytes(n, M))
        if need == 0:
            raise ValueError(f"pareto_rank: 1 <= n <= {MAX_POINTS} and 1 <= M <= {MAX_OBJECTIVES} (n = {n}, M = {M})")
        key = (need, torch.device(device))
        if self._ws_key != key:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=device)       # the caching allocator aligns to 512
            self._ws_key = key
        return self._ws

    def rank(self, obj: torch.Tensor, maximize: Sequence[bool], with_key: bool = False):
        """(front int32 [n], crowding float64 [n], order int32 [n], key float64 [n] or None), all on obj's device."""
        if not (isinstance(obj, torch.Tensor) and obj.is_cuda and obj.dtype == torch.float64):
            raise TypeError("pareto_rank: obj must be a float64 CUDA tensor")
        if obj.dim() != 2:
            raise ValueError(f"pareto_rank: obj must be a [n][M] matrix, not {tuple(obj.shape)}")
        if obj.stride(1) != 1:
            obj = obj.contiguous()
        n, M = obj.shape
        if len(maximize) != M:
            raise ValueError(f"{len(maximize)} directions for {M} objectives")
        ws = self.workspace(n, M, obj.device)
        dev = obj.device
        front = torch.empty(n, dtype=torch.int32, device=dev)
        crowding = torch.empty(n, dtype=torch.float64, device=dev)
        order = torch.empty(n, dtype=torch.int32, device=dev)
        key = torch.empty(n, dtype=torch.float64, device=dev) if with_key else None
        mx = (C.c_int * M)(*[1 if m else 0 for m in maximize])
        with torch.cuda.device(dev):
            _lib.call("b200bt_pareto_rank", obj.data_ptr(), _lib.ld(obj), n, M, mx, ws.data_ptr(), ws.numel(),
                      front.data_ptr(), crowding.data_ptr(), order.data_ptr(), _lib.ptr(key), _lib.current_stream())
        return front, crowding, order, key


def pareto_rank(obj: torch.Tensor, maximize: Sequence[bool], with_key: bool = False):
    """Fronts, crowding distance and crowded order of the rows of a device float64 [n][M] matrix (b200bt_pareto_rank).
    -> (front, crowding, order, key or None); key[p] = -(position of p in order).  Each call allocates its own workspace
    (n^2 / 8 bytes, 512 MB at n = 65 536); a caller that ranks repeatedly keeps one ParetoRanker, which reuses it."""
    return ParetoRanker().rank(obj, maximize, with_key)
