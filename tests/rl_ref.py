"""NumPy restatement of csrc/rl.cu: the states of b200bt_rl_states and the agents of b200bt_rl_train, operation for
operation (every float64 operation rounded on its own, every sum in index order from its first term), so the kernels are
compared with ==.  The rules and the reference's line numbers: include/b200bt.h (b200bt_rl_*).  Against the reference's own
TradingRLAgent (tests/golden/make_rl.py) the states, rewards, actions and counters are equal and the weights agree to the
last bits of the reference's BLAS summation order."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from oracle import mc_ref

FEATURES = 16
HID, OUT = 24, 3
PARAMS = 1083
STREAM_INIT, STREAM_ACT, STREAM_SAMPLE = 0, 1, 2
_2P26, _2M53 = 67108864.0, 1.0 / 9007199254740992.0

# analyzer column indices (enum b200bt_analyzer_column)
SMA_20, SMA_50, EMA_12, EMA_26, MACD, MACD_SIGNAL, RSI, BB_HIGH, BB_MID, BB_LOW, ATR = 0, 1, 3, 4, 5, 6, 10, 11, 12, 13, 15


def states(cols, close, volume, bar_minutes: int) -> np.ndarray:
    """[S][N][16] float64 from the analyzer columns [21][S][N] and close / volume [S][N] (fp32)."""
    col = lambda c: np.asarray(cols[c], dtype=np.float32).astype(np.float64)
    p = np.asarray(close, dtype=np.float32).astype(np.float64)
    v = np.asarray(volume, dtype=np.float32).astype(np.float64)
    S, N = p.shape
    f = np.empty((S, N, FEATURES))
    f[..., 0] = col(RSI) / 100.0
    f[..., 1] = (col(MACD) + 1.0) / 2.0
    f[..., 2] = (col(MACD_SIGNAL) + 1.0) / 2.0
    up, mid, lo = col(BB_HIGH), col(BB_MID), col(BB_LOW)
    rng = up - lo
    pos = p > 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        f[..., 3] = np.where(pos, np.where(rng > 0.0, (up - p) / rng, 0.5), 0.5)
        f[..., 4] = np.where(pos, np.where(rng > 0.0, (p - lo) / rng, 0.5), 0.5)
        f[..., 5] = np.where(pos, (p - mid) / p, 0.5)
        f[..., 6] = np.where(pos, col(EMA_12) / p, 1.0)
        f[..., 7] = np.where(pos, col(EMA_26) / p, 1.0)
        f[..., 8] = np.where(pos, col(ATR) / p, 0.0)
    vol = v / 1000000.0
    f[..., 9] = np.where(1.0 < vol, 1.0, vol)
    for k, (minutes, add, div) in enumerate(((60, 10.0, 20.0), (1440, 30.0, 60.0))):
        h = minutes // bar_minutes
        pc = np.zeros((S, N))
        if h < N:
            pc[:, h:] = (100.0 * (p[:, h:] - p[:, :-h])) / p[:, :-h]
        f[..., 10 + k] = (pc + add) / div
    f[..., 12] = 0.5
    f[..., 13] = 0.0
    f[..., 14] = 0.0
    s20, s50 = col(SMA_20), col(SMA_50)
    f[..., 15] = np.where((p > s20) & (s20 > s50), 0.8, np.where((p < s20) & (s20 < s50), 0.2, 0.5))
    return f


def reward(a: int, s, ns) -> float:
    """_calculate_reward (strategy_evolution_service.py:849-899); a = 0 BUY, 1 HOLD, 2 SELL."""
    pc = (float(ns[10]) - 0.5) * 2.0
    if a == 0:
        r = pc
        if s[0] < 0.3:
            r += 0.2
        if s[12] > 0.6:
            r += 0.1
        if s[4] < 0.2:
            r += 0.2
    elif a == 2:
        r = -pc
        if s[0] > 0.7:
            r += 0.2
        if s[12] < 0.4:
            r += 0.1
        if s[3] > 0.8:
            r += 0.2
    else:
        r = 0.05 if abs(pc) < 0.01 else 0.05 if 0.4 <= s[0] <= 0.6 else -0.05
    return float(r)


class Stream:
    """GaRng(seed, gid >> 32, gid, stream): counter = (gid low, gid high, stream, block), words x[3], x[2], x[1], x[0]."""

    def __init__(self, seed: int, gid: int, stream: int):
        self.key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
        self.ctr = (gid & 0xFFFFFFFF, (gid >> 32) & 0xFFFFFFFF, stream)
        self.words = 0
        self._x: List[int] = []

    def block(self, b: int) -> List[int]:
        x = mc_ref.philox4x32_10(np.uint32(self.ctr[0]), np.uint32(self.ctr[1]), np.uint32(self.ctr[2]), np.uint32(b),
                                 *self.key)
        return [int(w) for w in x]

    def next(self) -> int:
        if self.words % 4 == 0:
            self._x = self.block(self.words // 4)
        w = self._x[3 - self.words % 4]
        self.words += 1
        return w

    def uniform(self) -> float:
        hi = float(self.next() >> 5)
        lo = float(self.next() >> 6)
        return (hi * _2P26 + lo) * _2M53

    def below(self, n: int) -> int:
        return (self.next() * n) >> 32


def split(w):
    """Canonical parameter vector -> (W1, b1, W2, b2, W3, b3) views."""
    o = np.cumsum([0, FEATURES * HID, HID, HID * HID, HID, HID * OUT, OUT])
    shapes = ((FEATURES, HID), (HID,), (HID, HID), (HID,), (HID, OUT), (OUT,))
    return [w[o[i]:o[i + 1]].reshape(shapes[i]) for i in range(6)]


def init_weights(seed: int, gid: int) -> np.ndarray:
    """The INIT stream's randn * 0.1: normal pair p is Box-Muller of block p; the kernel's libm differs by a few ulps."""
    st = Stream(seed, gid, STREAM_INIT)
    n = FEATURES * HID + HID * HID + HID * OUT
    x = np.array([st.block(p) for p in range(n // 2)], dtype=np.float64)
    u1 = ((np.floor(x[:, 3] / 32) * _2P26 + np.floor(x[:, 2] / 64)) * _2M53)
    u2 = ((np.floor(x[:, 1] / 32) * _2P26 + np.floor(x[:, 0] / 64)) * _2M53)
    r = np.sqrt(-2.0 * np.log(1.0 - u1))
    ang = 6.283185307179586 * u2
    z = np.stack([r * np.cos(ang), r * np.sin(ang)], axis=1).reshape(-1) * 0.1
    w = np.zeros(PARAMS)
    W1, b1, W2, b2, W3, b3 = split(w)
    W1[:] = z[:FEATURES * HID].reshape(FEATURES, HID)
    W2[:] = z[FEATURES * HID:FEATURES * HID + HID * HID].reshape(HID, HID)
    W3[:] = z[FEATURES * HID + HID * HID:].reshape(HID, OUT)
    return w


def decode(text: str, dtype=np.float64) -> np.ndarray:
    """A fixture array: base64 of its little-endian bytes."""
    import base64
    return np.frombuffer(base64.b64decode(text), dtype=np.dtype(dtype).newbyteorder("<")).astype(dtype)


def fixture_weights(seed: int) -> np.ndarray:
    """Initial weights of the reference fixture's cases (tests/golden/make_rl.py): a PCG64 standard normal draw x 0.1 for
    W1, W2, W3 in order (platform independent), biases 0."""
    z = np.random.default_rng(seed).standard_normal(FEATURES * HID + HID * HID + HID * OUT) * 0.1
    w = np.zeros(PARAMS)
    W1, _, W2, _, W3, _ = split(w)
    W1[:] = z[:FEATURES * HID].reshape(FEATURES, HID)
    W2[:] = z[FEATURES * HID:FEATURES * HID + HID * HID].reshape(HID, HID)
    W3[:] = z[FEATURES * HID + HID * HID:].reshape(HID, OUT)
    return w


def _dot(x, W):
    """x [..., n] . W [n, m] summed in index order from the first term."""
    acc = x[..., 0:1] * W[0]
    for i in range(1, W.shape[0]):
        acc = acc + x[..., i:i + 1] * W[i]
    return acc


def forward(w, s, keep=False):
    W1, b1, W2, b2, W3, b3 = split(w)
    h1 = np.maximum(0.0, _dot(s, W1) + b1)
    h2 = np.maximum(0.0, _dot(h1, W2) + b2)
    q = _dot(h2, W3) + b3
    return (q, h1, h2) if keep else q


def sgd_step(w, s, tg, alpha):
    W1, b1, W2, b2, W3, b3 = split(w)
    out, h1, h2 = forward(w, s, keep=True)
    d_out = out - tg
    d_h2 = _dot(d_out, W3.T)
    d_h2[h2 <= 0] = 0.0
    d_h1 = _dot(d_h2, W2.T)
    d_h1[h1 <= 0] = 0.0
    d_W3, d_W2, d_W1 = np.outer(h2, d_out), np.outer(h1, d_h2), np.outer(s, d_h1)
    W3 -= alpha * d_W3
    b3 -= alpha * d_out
    W2 -= alpha * d_W2
    b2 -= alpha * d_h2
    W1 -= alpha * d_W1
    b1 -= alpha * d_h1


def _max3(q) -> float:
    m = q[0]
    if q[1] > m:
        m = q[1]
    if q[2] > m:
        m = q[2]
    return float(m)


@dataclass
class Agent:
    """One b200bt_rl_agent and its persisted state."""
    seed: int
    symbol: int = 0
    batch_size: int = 64
    memory_size: int = 10000
    update_target_every: int = 100
    learning_rate: float = 0.001
    gamma: float = 0.95
    epsilon_start: float = 1.0
    epsilon_end: float = 0.01
    epsilon_decay: float = 0.995
    gid: int = 0
    weights: Optional[np.ndarray] = None                  # online; the INIT draw when None
    target: Optional[np.ndarray] = None
    memory: List[tuple] = field(default_factory=list)     # (point, action, done), oldest first
    n_transitions: int = 0
    replays: int = 0
    epsilon: float = 0.0
    mean_q: float = float("nan")
    act: Optional[Stream] = None
    sample: Optional[Stream] = None
    trace: Optional[list] = None                          # when a list: (kind, ...) records of every draw and replay

    def __post_init__(self):
        self.weights = init_weights(self.seed, self.gid) if self.weights is None else np.array(self.weights, np.float64)
        self.target = self.weights.copy()
        self.epsilon = self.epsilon_start
        self.act = Stream(self.seed, self.gid, STREAM_ACT)
        self.sample = Stream(self.seed, self.gid, STREAM_SAMPLE)


def replay(ag: Agent, X, with_loss: bool):
    fill = len(ag.memory)
    picks: List[int] = []
    while len(picks) < ag.batch_size:                     # random.sample: distinct, in draw order
        c = ag.sample.below(fill)
        if c not in picks:
            picks.append(c)
    batch = [ag.memory[j] for j in picks]
    t = np.array([b[0] for b in batch])
    nt = np.array([b[0] if b[2] else b[0] + 1 for b in batch])
    cq = forward(ag.weights, X[t])
    nq = forward(ag.target, X[nt])
    tg = cq.copy()
    for i, (ti, a, done) in enumerate(batch):
        r = reward(a, X[ti], X[nt[i]])
        tg[i, a] = r if done else r + ag.gamma * _max3(nq[i])
    for i in range(len(batch)):
        sgd_step(ag.weights, X[t[i]], tg[i], ag.learning_rate)
    loss = float("nan")
    if with_loss:
        d = forward(ag.weights, X[t]) - tg
        e = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
        acc = e[0]
        for v in e[1:]:
            acc += v
        loss = float(acc / (3 * len(batch)))
    ag.replays += 1
    if ag.replays % ag.update_target_every == 0:
        ag.target = ag.weights.copy()
    if ag.epsilon > ag.epsilon_end:
        ag.epsilon *= ag.epsilon_decay
    mq = _max3(cq[0])
    for i in range(1, len(batch)):
        mq += _max3(cq[i])
    ag.mean_q = mq / len(batch)
    if ag.trace is not None:
        ag.trace.append(("replay", picks))
    return [loss, ag.mean_q, ag.epsilon, float(ag.replays)]


def py_sum(xs) -> float:
    """sum(xs) from the int 0 as Python 3.12 adds floats (Neumaier's compensated sum), restated step by step."""
    f, c = 0.0, 0.0
    for i, x in enumerate(xs):
        if i == 0:
            f = 0.0 + x
            continue
        t = f + x
        c += (f - t) + x if abs(f) >= abs(x) else (x - t) + f
        f = t
    return f + c if c != 0.0 and np.isfinite(c) else f


def train(ag: Agent, X, call_ends, points: int, history: bool = False):
    """X: states of the agent's symbol [N][16].  Returns (avg_reward [n_calls], q [n_calls][3], history rows)."""
    avg, qs, rows = [], [], []
    for end in call_ends:
        lo = max(0, end - points + 1)
        rewards = []
        for t in range(lo, end + 1):
            u = ag.act.uniform()
            if u < ag.epsilon:
                a = ag.act.below(3)
            else:
                q = forward(ag.weights, X[t])
                a = 0
                if q[1] > q[a]:
                    a = 1
                if q[2] > q[a]:
                    a = 2
            done = t == end
            r = reward(a, X[t], X[t if done else t + 1])
            rewards.append(r)
            if ag.trace is not None:
                ag.trace.append(("act", t, u, a, r))
            ag.memory.append((t, a, done))
            if len(ag.memory) > ag.memory_size:
                ag.memory.pop(0)
            ag.n_transitions += 1
            if len(ag.memory) >= ag.batch_size:
                rows.append(replay(ag, X, history))
        avg.append(py_sum(rewards) / (end - lo + 1))
        qs.append(forward(ag.weights, X[end]))
    return np.array(avg), np.array(qs).reshape(-1, OUT), np.array(rows).reshape(-1, 4)
