"""GA optimisation loop of the strategy-evolution service on the GPU engine.

Reference: services/strategy_evolution_service.py.
  param_ranges                       :98-117  (synth.param_ranges)
  optimize_with_genetic_algorithm    :525-694 (GA construction :644-655)
  optimize_with_reinforcement_learning :696-791 (rl.py: the agent on the device, trained on the market's bars)
The reference's fitness closure (:542-641) is a data-free placeholder that raises
NameError (SURVEY.md 0); the fitness wired in here is the reference's own
simulate -> metrics -> score composition (strategy_evaluation.py:682-691) evaluated for
the whole population by the sweep kernel.  LLM / Redis / regime plumbing is out of scope.
"""
from __future__ import annotations

import logging
import os
import secrets
import uuid
from datetime import datetime
from typing import Dict, List, Optional

from .dist import ShardedFitness, broadcast_seed
from .genetic_algorithm import GeneticAlgorithm, ParetoGeneticAlgorithm
from .pareto import objectives_from_goals
from .rl import ACTIONS, SERVICE_AGENT, RLPopulation, adjust_params_from_q_values, rl_states
from .sweep import DEFAULT_GOALS, MarketData, PopulationSweep
from .synth import param_ranges

logger = logging.getLogger("b200bt.evolution")


class StrategyEvolutionService:
    def __init__(self, market: MarketData, config: Optional[Dict] = None, leverage_trading: Optional[bool] = None,
                 random_seed: Optional[int] = None, aggregation: Optional[str] = None):
        """aggregation: the GA fitness of a multi-symbol strategy, "mean" of the per-symbol scores or the score of its
        "book" (all symbols as one trade list, PopulationSweep); default: config key evolution.fitness_aggregation,
        else "mean"."""
        self.config = config or {}
        if leverage_trading is None:
            leverage_trading = os.getenv("LEVERAGE_TRADING", "false").lower() == "true"     # :62
        self.leverage_trading = leverage_trading
        self.ga_population_size = int(os.getenv("GA_POPULATION_SIZE", 20))                  # :78
        self.ga_generations = int(os.getenv("GA_GENERATIONS", 10))                          # :79
        self.param_ranges = param_ranges(leverage_trading)
        goals = self.config.get("evolution", {}).get("optimization_goals") or DEFAULT_GOALS
        self.goals = goals
        self.market = market
        rsi_lo, rsi_hi = self.param_ranges["rsi_period"]
        self.aggregation = aggregation or self.config.get("evolution", {}).get("fitness_aggregation") or "mean"
        self.sweep = PopulationSweep(market, rsi_periods=range(int(rsi_lo), int(rsi_hi) + 1), optimization_goals=goals,
                                     aggregation=self.aggregation)
        self.fitness = ShardedFitness(self.sweep.evaluate, device=market.device)
        self.random_seed = random_seed
        self.evolution_records: List[Dict] = []
        self._rl_states = None
        self.rl_agents: Dict[int, RLPopulation] = {}      # the persistent agent of each symbol trained so far

    async def optimize_with_genetic_algorithm(self, current_params: Dict, performance_data: Optional[Dict] = None,
                                              historical_trades: Optional[List[Dict]] = None) -> Optional[Dict]:
        try:
            # under torch.distributed the GA operators run replicated: every rank needs the same seed (rank 0's;
            # a fresh one is drawn there when none was configured) -- ShardedFitness checks the populations agree
            import torch.distributed as dist
            seed = self.random_seed
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                seed = broadcast_seed(seed)
            ga = GeneticAlgorithm(param_ranges=self.param_ranges, fitness_function=self.fitness,
                                  population_size=self.ga_population_size, generations=self.ga_generations,
                                  mutation_rate=0.2, crossover_rate=0.8, elitism_pct=0.1,
                                  random_seed=seed)
            seeds = [dict(current_params)] if current_params else None
            optimized = ga.run(seeded_individuals=seeds)
            history = ga.get_generation_history()
            self.evolution_records.append({                       # the reference stores this record in Redis (:670-688)
                "id": str(uuid.uuid4()), "algorithm": "genetic", "timestamp": datetime.now().isoformat(),
                "improvement": history[-1]["best_fitness"] - history[0]["best_fitness"],
                "initial_fitness": history[0]["best_fitness"], "final_fitness": history[-1]["best_fitness"],
                "generations": len(history), "population_size": self.ga_population_size,
                "old_params": current_params, "new_params": optimized})
            self.last_ga = ga
            return optimized
        except Exception as e:        # reference convention (:692-694): log, return None
            logger.error("Error in genetic algorithm optimization: %s", e)
            return None

    async def optimize_pareto(self, current_params: Dict) -> Optional[List[Dict]]:
        """NSGA-II over the optimisation goals (ParetoGeneticAlgorithm): the objectives are the goals' primary and secondary
        metrics, each in its own direction (pareto.objectives_from_goals), instead of their product.  Returns the final
        Pareto front, [{"parameters": dict, "objectives": {name: value}}], and appends an evolution record whose new_params
        is the front's member with the best primary metric.  Single process: the objective matrix is not gathered over
        ranks, so under a torch.distributed world of more than one process this logs an error and returns None."""
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                logger.error("optimize_pareto runs in a single process (world size %d)", dist.get_world_size())
                return None
            objectives = objectives_from_goals(self.goals)
            sweep = self.sweep
            ga = ParetoGeneticAlgorithm(param_ranges=self.param_ranges,
                                        objective_function=lambda pop: sweep.evaluate_objectives_device(pop, objectives),
                                        objectives=objectives, population_size=self.ga_population_size,
                                        generations=self.ga_generations, mutation_rate=0.2, crossover_rate=0.8,
                                        random_seed=self.random_seed, device=self.market.device)
            seeds = [dict(current_params)] if current_params else None
            front = ga.run(seeded_individuals=seeds)
            history = ga.generation_history
            self.evolution_records.append({
                "id": str(uuid.uuid4()), "algorithm": "nsga2", "timestamp": datetime.now().isoformat(),
                "objectives": [{"name": n, "maximize": m} for n, m in objectives],
                "initial_best": history[0]["best_objectives"], "final_best": history[-1]["best_objectives"],
                "front_size": len(front), "generations": len(history), "population_size": self.ga_population_size,
                "old_params": current_params, "new_params": ga.best_individual})
            self.last_pareto = ga
            return front
        except Exception as e:        # reference convention (:692-694): log, return None
            logger.error("Error in Pareto optimization: %s", e)
            return None

    def _states(self):
        if self._rl_states is None:
            self._rl_states = rl_states(self.market)
        return self._rl_states

    async def optimize_with_reinforcement_learning(self, current_params: Dict, end_bar: int,
                                                   symbol: int = 0) -> Optional[Dict]:
        """One RL optimisation call (strategy_evolution_service.py:696-791) on the 20 bars of `symbol` ending at end_bar:
        the persistent agent (the service's hyperparameters, :213-224; one agent per symbol, created on first use) acts,
        remembers and replays on the device, and the Q-values of the last bar adjust the parameters (:901-975).  Appends
        the reference's evolution record; on error logs and returns None, as the reference does."""
        try:
            agent = self.rl_agents.get(symbol)
            if agent is None:
                seed = self.random_seed if self.random_seed is not None else secrets.randbits(63)
                agent = RLPopulation(self._states(), [dict(SERVICE_AGENT, seed=seed, symbol=symbol)])
                self.rl_agents[symbol] = agent
            agent.train([int(end_bar)], points_per_call=20)
            q = agent.q_values[0, -1]
            q_values = {a: float(q[i]) for i, a in enumerate(ACTIONS)}
            adjusted = adjust_params_from_q_values(current_params, q_values, self.param_ranges)
            self.evolution_records.append({                       # the reference stores this record in Redis (:770-785)
                "id": str(uuid.uuid4()), "algorithm": "reinforcement_learning", "timestamp": datetime.now().isoformat(),
                "avg_reward": float(agent.avg_reward[0, -1]), "q_values": q_values, "old_params": current_params,
                "new_params": adjusted, "epsilon": float(agent.epsilon[0])})
            return adjusted
        except Exception as e:        # reference convention (:789-791): log, return None
            logger.error("Error in reinforcement learning optimization: %s", e)
            return None

    def optimize_rl_population(self, current_params: Dict, call_end_bars, agents: List[Dict],
                               points_per_call: int = 20) -> Optional[List[Dict]]:
        """Train a fresh population of agents (dicts of seed, symbol and any of the reference constructor's
        hyperparameters; SERVICE_AGENT fills the rest) over the calls ending at call_end_bars, all at once on the device.
        Returns per agent {"agent", "new_params", "avg_reward", "q_values", "epsilon"} from its last call; the population
        stays in `last_rl_population`.  On error logs and returns None."""
        try:
            pop = RLPopulation(self._states(), agents).train(call_end_bars, points_per_call=points_per_call)
            self.last_rl_population = pop
            eps = pop.epsilon
            out = []
            for i, a in enumerate(pop.agents):
                q_values = {name: float(pop.q_values[i, -1, k]) for k, name in enumerate(ACTIONS)}
                out.append({"agent": a, "new_params": adjust_params_from_q_values(current_params, q_values, self.param_ranges),
                            "avg_reward": float(pop.avg_reward[i, -1]), "q_values": q_values, "epsilon": float(eps[i])})
            return out
        except Exception as e:
            logger.error("Error in reinforcement learning population optimization: %s", e)
            return None
