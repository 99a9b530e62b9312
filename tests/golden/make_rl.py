"""Generate the reinforcement-learning fixture by EXECUTING the reference's own code.

Run where a copy of the reference tree exists (as for make_golden.py):

    python tests/golden/make_rl.py

Writes tests/golden/rl_reference.json.  services/reinforcement_learning.py's TradingRLAgent runs unmodified on its NumPy
path (TensorFlow absent), and services/strategy_evolution_service.py is imported with the packages it imports but these
functions do not use replaced by empty stubs; three of its methods run unmodified on an instance built without __init__:
    optimize_with_reinforcement_learning  :696-791  per call, on the points of that call (Redis: a recorder)
    _convert_market_data_to_state         :793-847  (through it, and on its own for the state cases)
    _calculate_reward, _adjust_params_from_q_values  (through it; the latter also with the leverage parameter ranges)
The agent starts from given weights (a PCG64 standard normal draw x 0.1, platform independent), and its module's `random`
is replaced by an object that serves the restatement's Philox draws (tests/rl_ref.py: ACT stream for random() and
randrange(3), SAMPLE stream for random.sample, distinct positions with repeats rejected), so every action and minibatch
is the one the kernel draws.  The points are the wiring of include/b200bt.h: price = close, the analyzer's columns, the
price changes over 1 and 24 hours of the clock (0 before the first full hour and day), get_trend's rule per bar.
"""
from __future__ import annotations

import asyncio
import base64
import json
import sys
import types
from collections import deque
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
OUT = Path(__file__).resolve().parent / "rl_reference.json"
TOL = 1e-9


def _load():
    from oracle import ref_runner
    ref_runner._prepare()
    stubs = {"aiohttp": {}, "openai": {"AsyncOpenAI": object}, "dotenv": {"load_dotenv": lambda *a, **k: None},
             "services.genetic_algorithm": {"GeneticAlgorithm": object},
             "services.strategy_evaluation": {"StrategyPerformanceMetrics": object, "StrategyEvaluationSystem": object},
             "services.market_regime_service": {"MarketRegimeService": object},
             "services.social_strategy_integrator": {"SocialStrategyIntegrator": object}}
    for name, attrs in stubs.items():
        mod = sys.modules.setdefault(name, types.ModuleType(name))
        for k, v in attrs.items():
            setattr(mod, k, v)
    import importlib
    import logging
    rl = importlib.import_module("services.reinforcement_learning")
    ses = importlib.import_module("services.strategy_evolution_service")
    logging.getLogger().setLevel(logging.ERROR)
    logging.getLogger("reinforcement_learning").setLevel(logging.ERROR)
    for h in list(logging.getLogger().handlers):
        logging.getLogger().removeHandler(h)
    return rl, ses


class DrawServer:
    """Stands in for the `random` module of reinforcement_learning.py: the restatement's streams."""

    def __init__(self, seed: int):
        import rl_ref
        self.act = rl_ref.Stream(seed, 0, rl_ref.STREAM_ACT)
        self.smp = rl_ref.Stream(seed, 0, rl_ref.STREAM_SAMPLE)

    def random(self):
        return self.act.uniform()

    def randrange(self, n):
        return self.act.below(n)

    def sample(self, population, k):
        picks = []
        while len(picks) < k:
            c = self.smp.below(len(population))
            if c not in picks:
                picks.append(c)
        return [population[j] for j in picks]


class Recorder:
    def __init__(self):
        self.records = []

    async def set(self, key, value):
        self.records.append(json.loads(value))


def market(rng, N, bar_minutes, flat=None):
    """fp32 close / volume and analyzer-like columns with reachable features (zero Bollinger range on `flat`)."""
    close = (100.0 * np.exp(np.cumsum(0.01 * rng.standard_normal(N)))).astype(np.float32)
    vol = rng.uniform(2e5, 2e6, N).astype(np.float32)
    c = close.astype(np.float64)
    cols = {
        "sma_20": c * (1 + 0.01 * rng.standard_normal(N)), "sma_50": c * (1 + 0.01 * rng.standard_normal(N)),
        "ema_12": c * (1 + 0.005 * rng.standard_normal(N)), "ema_26": c * (1 + 0.005 * rng.standard_normal(N)),
        "macd": 0.5 * rng.standard_normal(N), "macd_signal": 0.5 * rng.standard_normal(N),
        "rsi": rng.uniform(10, 90, N), "atr": c * rng.uniform(0.001, 0.03, N),
    }
    width = c * rng.uniform(0.002, 0.05, N)
    mid = c * (1 + 0.01 * rng.standard_normal(N))
    cols["bb_mid"], cols["bb_high"], cols["bb_low"] = mid, mid + width * rng.uniform(0, 1, N), mid - width * rng.uniform(0, 1, N)
    if flat is not None:
        cols["bb_high"][flat] = cols["bb_low"][flat] = cols["bb_mid"][flat]
    cols = {k: v.astype(np.float32) for k, v in cols.items()}
    return close, vol, cols


def points_of(close, vol, cols, bar_minutes):
    """The wiring: one point dict per bar (Python floats of the fp32 values)."""
    c = close.astype(np.float64)
    pcs = []
    for minutes in (60, 1440):
        h = minutes // bar_minutes
        pc = np.zeros(len(c))
        pc[h:] = (100.0 * (c[h:] - c[:-h])) / c[:-h]
        pcs.append(pc)
    f = {k: v.astype(np.float64) for k, v in cols.items()}
    pts = []
    for t in range(len(c)):
        p, s20, s50 = c[t], f["sma_20"][t], f["sma_50"][t]
        trend = "uptrend" if p > s20 and s20 > s50 else "downtrend" if p < s20 and s20 < s50 else "sideways"
        pts.append({"price": float(p), "rsi": float(f["rsi"][t]), "macd": float(f["macd"][t]),
                    "macd_signal": float(f["macd_signal"][t]), "bb_upper": float(f["bb_high"][t]),
                    "bb_middle": float(f["bb_mid"][t]), "bb_lower": float(f["bb_low"][t]),
                    "ema_short": float(f["ema_12"][t]), "ema_long": float(f["ema_26"][t]), "atr": float(f["atr"][t]),
                    "volume": float(vol[t]), "price_change_1h": float(pcs[0][t]), "price_change_24h": float(pcs[1][t]),
                    "trend": trend})
    return pts


def run_case(rl, ses, name, seed, agent_kw, N, bar_minutes, call_ends, leverage=False, flat=None, with_weights=True):
    rng = np.random.default_rng(seed)
    close, vol, cols = market(rng, N, bar_minutes, flat)
    pts = points_of(close, vol, cols, bar_minutes)
    svc = object.__new__(ses.StrategyEvolutionService)
    svc.leverage_trading = leverage
    svc.enable_reinforcement_learning = True
    svc.redis = Recorder()
    svc.param_ranges = {
        "rsi_period": (5, 30), "rsi_overbought": (65, 85), "rsi_oversold": (15, 35),
        "social_sentiment_threshold": (50, 80),
        "stop_loss": (1, 5) if not leverage else (0.5, 2.5), "take_profit": (1, 10) if not leverage else (2, 20)}
    svc._initialize_rl_agent()
    agent = svc.rl_agent
    for k, v in agent_kw.items():
        setattr(agent, k, v)
    agent.memory = deque(maxlen=agent.memory_size)
    rl.random = DrawServer(seed)
    import rl_ref
    w0 = rl_ref.fixture_weights(seed)
    parts = rl_ref.split(w0.copy())
    agent.weights1, agent.bias1, agent.weights2, agent.bias2, agent.weights3, agent.bias3 = [p.copy() for p in parts]
    agent._update_target_network()
    actions, rewards, copies = [], [], []
    remember, update = agent.remember, agent._update_target_network
    agent.remember = lambda s, a, r, ns, d: (actions.append(a), rewards.append(r), remember(s, a, r, ns, d))
    agent._update_target_network = lambda: (copies.append(agent.step_counter), update())
    params = {"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30, "take_profit": 5, "stop_loss": 2,
              "social_sentiment_threshold": 60}
    calls = []
    for end in call_ends:
        new = asyncio.run(svc.optimize_with_reinforcement_learning(params, pts[max(0, end - 19):end + 1]))
        rec = svc.redis.records[-1]
        calls.append({"avg_reward": rec["avg_reward"], "q_values": [rec["q_values"][a] for a in ("BUY", "HOLD", "SELL")],
                      "new_params": new, "epsilon": rec["epsilon"]})
        params = new
    states = [[svc._convert_market_data_to_state(p)[f] for f in agent.state_features] for p in pts]
    final = np.concatenate([getattr(agent, n).reshape(-1) for n in
                            ("weights1", "bias1", "weights2", "bias2", "weights3", "bias3")])
    hist = [[h["loss"], h["mean_q"]] for h in agent.training_history]
    out = {
        "name": name, "seed": seed, "bar_minutes": bar_minutes, "leverage": leverage, "points": 20,
        "agent": {k: agent_kw.get(k, getattr(agent, k)) for k in ("learning_rate", "gamma", "epsilon_end", "epsilon_decay",
                                                                   "memory_size", "batch_size", "update_target_every")}
        | {"epsilon_start": 1.0},
        "close": enc(close, np.float32), "volume": enc(vol, np.float32), "cols": {k: enc(v, np.float32) for k, v in cols.items()},
        "states": enc(states), "call_ends": list(call_ends), "calls": calls,
        "actions": "".join(str(("BUY", "HOLD", "SELL").index(a)) for a in actions), "rewards": enc(rewards),
        "target_copies": copies, "step_counter": agent.step_counter, "epsilon": agent.epsilon,
        "history_loss_mean_q": enc(hist),
    }
    if with_weights:
        out["final_weights"] = enc(final)
    return out


def enc(a, dtype=np.float64) -> str:
    """Little-endian bytes of the array, base64 (tests/rl_ref.py decode)."""
    return base64.b64encode(np.ascontiguousarray(a, dtype=np.dtype(dtype).newbyteorder("<")).tobytes()).decode()


def main():
    rl, ses = _load()
    cases = [
        run_case(rl, ses, "service defaults, 20 calls of 20 points", 101, {}, 48, 60,
                 [19 + (28 * k) // 19 for k in range(20)]),
        run_case(rl, ses, "memory 100, batch 16: deque eviction", 102, {"memory_size": 100, "batch_size": 16}, 48, 60,
                 [19 + (28 * k) // 11 for k in range(12)], flat=slice(30, 34), with_weights=False),
        run_case(rl, ses, "target period 5, epsilon at its floor, leverage ranges", 103,
                 {"update_target_every": 5, "batch_size": 8, "memory_size": 50, "epsilon_decay": 0.9,
                  "epsilon_end": 0.3}, 48, 60, [5, 19, 30, 47, 47, 33], leverage=True),
        run_case(rl, ses, "30-minute clock: states before the first full hour and day", 104, {"batch_size": 4},
                 60, 30, [2, 3, 4, 50, 59], with_weights=False),
    ]
    text = json.dumps({"tolerance": TOL, "cases": cases}, separators=(",", ":"))
    OUT.write_text(text + "\n")
    print(f"wrote {OUT} ({len(text) / 1024:.0f} KB, {len(cases)} cases)")


if __name__ == "__main__":
    main()
