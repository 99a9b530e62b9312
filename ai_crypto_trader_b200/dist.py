"""Multi-GPU sharding of the population sweep: one process per GPU (torchrun),
individuals partitioned contiguously across ranks, market data replicated, ONE
all-gather of the fitness vector per generation (SURVEY.md 8e).  NCCL on GPUs;
the same code runs over gloo on CPU tensors for the host-logic tests.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence

import numpy as np
import torch
import torch.distributed as dist


def shard_bounds(n: int, world: int, rank: int):
    """Contiguous shard [lo, hi) of n items for `rank`; every rank holds ceil(n/world) slots."""
    per = (n + world - 1) // world
    lo = min(rank * per, n)
    return lo, min(lo + per, n), per


def population_fingerprint(population: List[Dict]) -> int:
    """63-bit digest of a population (gene names and values in order): equal on two ranks iff they hold the same
    individuals in the same order (up to hash collisions)."""
    import hashlib
    h = hashlib.blake2b(digest_size=8)
    if population:
        keys = sorted(population[0])
        h.update("\0".join(keys).encode())
        h.update(np.array([[float(p.get(k, np.nan)) for k in keys] for p in population], dtype=np.float64).tobytes())
    return int.from_bytes(h.digest(), "little") & ((1 << 63) - 1)


class PopulationMismatch(RuntimeError):
    """The ranks of a sharded fitness evaluation do not hold the same population."""


class ShardedFitness:
    """Batched fitness callable: evaluates this rank's shard with `evaluate_local`
    (List[Dict] -> float64 array) and all-gathers the per-rank results.

    `fitness = ShardedFitness(sweep.evaluate)`; `GeneticAlgorithm(..., fitness_function=fitness)`
    then calls `fitness.batch(population)` once per generation on every rank.  The GA operators run replicated, so
    every rank must hold the SAME population (same `random_seed`; evolution.StrategyEvolutionService broadcasts one when
    none is given).  That is enforced, not assumed: the gather carries each rank's population fingerprint and an error
    flag next to its fitness shard, and every rank raises together -- PopulationMismatch when the fingerprints differ,
    RuntimeError when any rank's local evaluation failed -- so a bad rank can neither poison the fitness vector
    silently nor leave the others waiting in the collective.  Still ONE collective per generation.
    """

    def __init__(self, evaluate_local: Callable[[List[Dict]], Sequence[float]], device=None, group=None):
        self.evaluate_local = evaluate_local
        self.group = group
        self.device = device
        self.batch = self.__call_batch

    def _world(self):
        if dist.is_available() and dist.is_initialized():
            return dist.get_world_size(self.group), dist.get_rank(self.group)
        return 1, 0

    def __call_batch(self, population: List[Dict]) -> List[float]:
        world, rank = self._world()
        n = len(population)
        lo, hi, per = shard_bounds(n, world, rank)
        if world == 1:
            return np.asarray(self.evaluate_local(population[lo:hi]) if hi > lo else [], dtype=np.float64).tolist()
        error = None
        try:
            local = np.asarray(self.evaluate_local(population[lo:hi]) if hi > lo else [], dtype=np.float64)
            if local.shape != (hi - lo,):
                raise ValueError(f"evaluate_local returned {local.shape} values for {hi - lo} individuals")
        except Exception as e:          # joins the collective anyway, so that every rank fails together
            error, local = e, np.full(hi - lo, np.nan)
        dev = self.device
        if dev is None:
            dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        # [per fitness slots | population fingerprint (int64 bits) | error flag]
        host = np.full(per + 2, np.nan, dtype=np.float64)
        host[:hi - lo] = local
        host[per:per + 1].view(np.int64)[0] = population_fingerprint(population)
        host[per + 1] = 0.0 if error is None else 1.0
        send = torch.from_numpy(host).to(dev)
        recv = torch.empty((per + 2) * world, dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(recv, send, group=self.group)   # the one collective per generation
        full = recv.cpu().numpy().reshape(world, per + 2)
        failed = [r for r in range(world) if full[r, per + 1] != 0.0]
        if failed:
            raise RuntimeError(f"sharded fitness: local evaluation failed on rank(s) {failed}"
                               + (f" (this rank: {error!r})" if error is not None else "")) from error
        prints = np.ascontiguousarray(full[:, per]).view(np.int64)
        if not (prints == prints[0]).all():
            raise PopulationMismatch(f"sharded fitness: ranks hold different populations (fingerprints {prints.tolist()}); "
                                     "run the GA with the same random_seed on every rank")
        out = np.concatenate([full[r, :shard_bounds(n, world, r)[1] - shard_bounds(n, world, r)[0]] for r in range(world)])
        return out.tolist()

    def __call__(self, individual: Dict) -> float:
        return float(self.evaluate_local([individual])[0])


def broadcast_seed(seed=None, group=None) -> int:
    """The GA seed every rank uses: rank 0's `seed` (a fresh one when None), broadcast when torch.distributed is up."""
    import random
    if seed is None:
        seed = random.SystemRandom().randrange(1 << 31)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        box = [int(seed)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        seed = box[0]
    return int(seed)


def gather_paths(local_finals: torch.Tensor, local_maxdd: torch.Tensor, n_total: int, group=None):
    """All-gather the per-rank shards of a Monte-Carlo run (paths sharded contiguously by shard_bounds, the kernels
    keyed by the GLOBAL path index, so the gathered arrays equal a single-GPU run bit for bit).  One collective of
    8 bytes per path; every rank then holds all finals / drawdowns and computes the same order statistics."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_finals, local_maxdd
    finals, maxdd = gather_path_rows(torch.stack([local_finals, local_maxdd]), n_total, group)
    return finals, maxdd


def gather_path_rows(local_rows: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """All-gather a [K][n_local] block of per-path rows (finals and drawdowns, the per-asset finals of a joint run),
    sharded as gather_paths' arrays: one collective, and the gathered [K][n_total] equals a single-GPU run bit for bit."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_rows
    world = dist.get_world_size(group)
    per = -(-n_total // world)
    K = local_rows.shape[0]
    send = torch.full((K, per), float("nan"), dtype=local_rows.dtype, device=local_rows.device)
    send[:, :local_rows.shape[1]] = local_rows
    recv = torch.empty((world, K, per), dtype=local_rows.dtype, device=local_rows.device)
    dist.all_gather_into_tensor(recv.view(-1), send.view(-1), group=group)
    counts = [shard_bounds(n_total, world, r)[1] - shard_bounds(n_total, world, r)[0] for r in range(world)]
    return torch.cat([recv[r, :, :counts[r]] for r in range(world)], dim=1)
