"""Reinforcement-learning agents of the strategy-evolution service on the GPU.

Reference: services/reinforcement_learning.py (TradingRLAgent, NumPy path) as the strategy-evolution service builds and
trains it (services/strategy_evolution_service.py):
  agent hyperparameters              :213-224  (SERVICE_AGENT)
  state features                     :203-207  (RL_STATE_FEATURES), _convert_market_data_to_state :793-847 (rl_states)
  one RL optimisation call           :696-791  (RLPopulation.train, one call per end bar)
  _adjust_params_from_q_values       :901-975  (adjust_params_from_q_values)
The reference trains on a Redis key nothing writes; the points here are the market's bars (our wiring, include/b200bt.h
b200bt_rl_*, DESIGN.md 3.15).  Training runs on the device for a whole population of agents, one warp each; the agents'
weights, replay memory, epsilon and RNG positions stay on the device between calls, so `train` can be called once per
evolution step and continues where the last call ended.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch

from . import _lib

RL_STATE_FEATURES = [
    "rsi", "macd", "macd_signal", "bb_upper", "bb_lower", "bb_middle", "ema_short", "ema_long", "atr", "volume",
    "price_change_1h", "price_change_24h", "social_sentiment", "social_volume", "social_engagement", "market_trend",
]
ACTIONS = ("BUY", "HOLD", "SELL")
SERVICE_AGENT = dict(learning_rate=0.001, gamma=0.95, epsilon_start=1.0, epsilon_end=0.01, epsilon_decay=0.995,
                     memory_size=10000, batch_size=64, update_target_every=100)
_WEIGHT_NAMES = ("weights1", "bias1", "weights2", "bias2", "weights3", "bias3")
_SHAPES = ((16, 24), (24,), (24, 24), (24,), (24, 3), (3,))


def rl_states(market) -> torch.Tensor:
    """Device float64 state table [S][N][16] of a MarketData on its own clock (whose bar length must divide 60 minutes):
    b200bt_analyzer's columns, then b200bt_rl_states.  Resample first (indicators.resample) for an hourly agent."""
    lib = _lib.load()
    S, N = market.S, market.N
    h, l, c, v = market.high, market.low, market.close, market.volume
    cols = torch.empty((len(_lib.ANALYZER_COLUMNS), S, N), dtype=torch.float32, device=c.device)
    ws = torch.empty(int(lib.b200bt_analyzer_workspace_floats(S, N)), dtype=torch.float32, device=c.device)
    out = torch.empty((S, N, _lib.RL_FEATURES), dtype=torch.float64, device=c.device)
    with torch.cuda.device(c.device):
        _lib.call("b200bt_analyzer", h.data_ptr(), l.data_ptr(), c.data_ptr(), v.data_ptr(), S, N, _lib.ld(c),
                  cols.data_ptr(), ws.data_ptr(), _lib.current_stream())
        _lib.call("b200bt_rl_states", cols.data_ptr(), c.data_ptr(), v.data_ptr(), _lib.ld(c), S, N, market.bar_minutes,
                  out.data_ptr(), _lib.current_stream())
    return out


def adjust_params_from_q_values(params: Mapping, q, param_ranges: Mapping) -> Dict:
    """_adjust_params_from_q_values (strategy_evolution_service.py:901-975).  q: {action: value} or the three Q-values
    in ACTIONS order.  Quirks kept: take_profit * 0.9 turns an integer into a float, and stop_loss * (1 - 0.2 max_q)
    widens the stop when every Q-value is negative (only the lower bound is clamped)."""
    q_values = dict(q) if isinstance(q, Mapping) else {a: float(q[i]) for i, a in enumerate(ACTIONS)}
    adjusted = dict(params)
    max_action = max(q_values.items(), key=lambda x: x[1])[0]
    buy, sell, hold = q_values.get("BUY", 0), q_values.get("SELL", 0), q_values.get("HOLD", 0)
    if max_action == "BUY":
        if "rsi_oversold" in adjusted:
            adjusted["rsi_oversold"] = min(adjusted["rsi_oversold"] + 5, param_ranges["rsi_oversold"][1])
        if "social_sentiment_threshold" in adjusted:
            adjusted["social_sentiment_threshold"] = max(adjusted["social_sentiment_threshold"] - 5,
                                                         param_ranges["social_sentiment_threshold"][0])
    elif max_action == "SELL":
        if "rsi_overbought" in adjusted:
            adjusted["rsi_overbought"] = max(adjusted["rsi_overbought"] - 5, param_ranges["rsi_overbought"][0])
        if "take_profit" in adjusted:
            adjusted["take_profit"] = max(adjusted["take_profit"] * 0.9, param_ranges["take_profit"][0])
    elif max_action == "HOLD":
        if "rsi_period" in adjusted:
            adjusted["rsi_period"] = min(adjusted["rsi_period"] + 2, param_ranges["rsi_period"][1])
    confidence = max(buy, sell, hold)
    if "stop_loss" in adjusted:
        adjusted["stop_loss"] = max(adjusted["stop_loss"] * (1 - confidence * 0.2), param_ranges["stop_loss"][0])
    return adjusted


class RLPopulation:
    """A population of TradingRLAgents trained on the device over a state table (rl_states).

    agents: dicts with the reference constructor's names (learning_rate, gamma, epsilon_start, epsilon_end, epsilon_decay,
    memory_size, batch_size, update_target_every; SERVICE_AGENT fills the missing ones) plus `seed` and `symbol`.
    agent_offset: global index of the first agent (its RNG counter), so an agent trains the same alone, in any
    population or shard.  init_weights: optional [A][1083] canonical weights replacing the initial draw."""

    def __init__(self, states: torch.Tensor, agents: Sequence[Mapping], agent_offset: int = 0,
                 init_weights: Optional[np.ndarray] = None):
        if states.dtype != torch.float64 or states.dim() != 3 or states.shape[2] != _lib.RL_FEATURES:
            raise ValueError("states must be rl_states' float64 [S][N][16] table")
        self.states = states.contiguous()
        self.S, self.N = int(states.shape[0]), int(states.shape[1])
        self.device = states.device
        self.agents = [dict(SERVICE_AGENT, **a) for a in agents]
        A = len(self.agents)
        if A < 1:
            raise ValueError("a population needs at least one agent")
        self._abi = (_lib.RlAgent * A)()
        for rec, a in zip(self._abi, self.agents):
            rec.seed = int(a["seed"]) & (2 ** 64 - 1)
            rec.symbol = int(a.get("symbol", 0))
            for k in ("batch_size", "memory_size", "update_target_every"):
                setattr(rec, k, int(a[k]))
            for k in ("learning_rate", "gamma", "epsilon_start", "epsilon_end", "epsilon_decay"):
                setattr(rec, k, float(a[k]))
        self.agent_offset = int(agent_offset)
        self.memory_max = max(int(a["memory_size"]) for a in self.agents)
        nbytes = int(_lib.load().b200bt_rl_workspace_bytes(A, self.memory_max))
        if nbytes <= 0:
            raise ValueError(f"memory_size must be in [1, {_lib.RL_MAX_MEMORY}]")
        self._state = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        self._stride = nbytes // A
        self._init = None
        if init_weights is not None:
            self._init = torch.as_tensor(np.asarray(init_weights, dtype=np.float64).reshape(A, _lib.RL_PARAMS),
                                         device=self.device).contiguous()
        self._history: List[List[np.ndarray]] = [[] for _ in range(A)]      # per agent: [replays][4] blocks
        self.q_values: Optional[np.ndarray] = None        # [A][n_calls][3] of the last train()
        self.avg_reward: Optional[np.ndarray] = None      # [A][n_calls]

    def __len__(self) -> int:
        return len(self.agents)

    def train(self, call_end_bars, points_per_call: int = 20, history: bool = False) -> "RLPopulation":
        """One optimisation call per end bar, in order, for every agent (one launch).  Continues from the state the last
        call left.  history: also record the reference's training_history rows (and compute the loss)."""
        ends = np.ascontiguousarray(np.atleast_1d(np.asarray(call_end_bars, dtype=np.int64)))
        A, n = len(self), len(ends)
        avg = torch.empty((A, n), dtype=torch.float64, device=self.device)
        q = torch.empty((A, n, 3), dtype=torch.float64, device=self.device)
        rows = int(np.minimum(ends + 1, points_per_call).sum()) if n else 0
        hist = torch.empty((A, max(rows, 1), 4), dtype=torch.float64, device=self.device) if history else None
        before = self.replays if history else None
        with torch.cuda.device(self.device):
            _lib.call("b200bt_rl_train", self.states.data_ptr(), self.S, self.N, self._abi, A, self.agent_offset,
                      self.memory_max, self._state.data_ptr(), self._state.numel(),
                      ends.ctypes.data_as(C.POINTER(C.c_int64)), n, int(points_per_call), _lib.ptr(self._init),
                      avg.data_ptr(), q.data_ptr(), _lib.ptr(hist), max(rows, 1) if history else 0,
                      _lib.current_stream())
        self.avg_reward = avg.cpu().numpy()
        self.q_values = q.cpu().numpy()
        if history:
            h = hist.cpu().numpy()
            for i, k in enumerate(self.replays - before):
                self._history[i].append(h[i, :k])
        return self

    def _headers(self) -> np.ndarray:
        raw = self._state.view(len(self), self._stride)[:, :64].cpu().numpy()
        return raw.copy().view(np.dtype(_lib.RL_STATE_DTYPE)).reshape(-1)

    @property
    def epsilon(self) -> np.ndarray:
        return self._headers()["epsilon"].copy()

    @property
    def replays(self) -> np.ndarray:
        """step_counter of every agent."""
        return self._headers()["replays"].astype(np.int64)

    @property
    def mean_q(self) -> np.ndarray:
        """mean_q of each agent's last replay (NaN before the first)."""
        return self._headers()["mean_q"].copy()

    def weight_vector(self, i: int, target: bool = False) -> np.ndarray:
        """Agent i's canonical 1083-double weights (online or target)."""
        off = 64 + (8 * _lib.RL_PARAMS if target else 0)
        raw = self._state[i * self._stride + off: i * self._stride + off + 8 * _lib.RL_PARAMS]
        return raw.cpu().numpy().view(np.float64).copy()

    def weights(self, i: int) -> Dict[str, np.ndarray]:
        """Agent i's networks by the reference's attribute names (weights1 ... bias3, target_weights1 ... target_bias3)."""
        out = {}
        for prefix, target in (("", False), ("target_", True)):
            v = self.weight_vector(i, target)
            o = 0
            for name, shape in zip(_WEIGHT_NAMES, _SHAPES):
                size = int(np.prod(shape))
                out[prefix + name] = v[o:o + size].reshape(shape)
                o += size
        return out

    def training_history(self, i: int) -> List[Dict]:
        """get_training_history's rows {loss, mean_q, epsilon, step} of the calls trained with history=True."""
        return [{"loss": float(r[0]), "mean_q": float(r[1]), "epsilon": float(r[2]), "step": int(r[3])}
                for block in self._history[i] for r in block]
