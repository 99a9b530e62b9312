"""CPU-side checks of the reinforcement-learning entry points (csrc/rl.cu): struct layouts, workspace sizing and every
argument refusal, which happens before the device is touched (the dummy device pointers are never dereferenced)."""
import ctypes as C

import numpy as np
import pytest

_EINVAL, _ENODEVICE, _ELIMIT = 10001, 10002, 10003
DEV = 1 << 20


def _status(fn, *args):
    from ai_crypto_trader_b200 import _lib
    try:
        _lib.call(fn, *args)
    except _lib.B200btError as e:
        return e.status
    return 0


def _agents(n=2, **kw):
    from ai_crypto_trader_b200 import _lib
    arr = (_lib.RlAgent * n)()
    for a in arr:
        a.seed, a.symbol, a.batch_size, a.memory_size, a.update_target_every = 7, 0, 64, 10000, 100
        a.learning_rate, a.gamma, a.epsilon_start, a.epsilon_end, a.epsilon_decay = 0.001, 0.95, 1.0, 0.01, 0.995
        for k, v in kw.items():
            setattr(a, k, v)
    return arr


def _train(states=DEV, S=2, N=1000, agents=None, A=2, offset=0, memory_max=10000, ws=DEV, ws_bytes=None, ends=(19, 500),
           points=20, init=None, avg=DEV, q=DEV, hist=None, rows=0):
    from ai_crypto_trader_b200 import _lib
    agents = _agents(A) if agents is None else agents
    if ws_bytes is None:
        ws_bytes = int(_lib.load().b200bt_rl_workspace_bytes(A, memory_max)) if 1 <= memory_max <= _lib.RL_MAX_MEMORY else 1 << 40
    e = np.ascontiguousarray(ends, dtype=np.int64)
    return _status("b200bt_rl_train", states, S, N, agents, A, offset, memory_max, ws, ws_bytes,
                   e.ctypes.data_as(C.POINTER(C.c_int64)) if len(e) else None, len(e), points, init, avg, q, hist, rows, None)


def test_struct_layouts(native_lib):
    from ai_crypto_trader_b200 import _lib
    assert C.sizeof(_lib.RlAgent) == 64 and _lib.RlAgent.learning_rate.offset == 24
    assert np.dtype(_lib.RL_STATE_DTYPE).itemsize == 64
    assert _lib.RL_PARAMS == 16 * 24 + 24 + 24 * 24 + 24 + 24 * 3 + 3


def test_workspace_bytes(native_lib):
    from ai_crypto_trader_b200 import _lib
    f = _lib.load().b200bt_rl_workspace_bytes
    for A, M in ((1, 1), (3, 100), (1024, 10000)):
        assert f(A, M) == A * (64 + 2 * 8 * 1083 + 8 * M)
    assert f(1, 10000) == 64 + 17328 + 80000          # 80 KB of replay memory at the service's size
    assert f(0, 10) == 0 and f(1, 0) == 0 and f(1, _lib.RL_MAX_MEMORY + 1) == 0


def test_rl_refusals(native_lib):
    import torch
    if not torch.cuda.is_available():                                        # every check passed
        assert _train() == _ENODEVICE
        assert _train(hist=DEV, rows=40) == _ENODEVICE and _train(ends=(0, 999), points=1) == _ENODEVICE
        assert _train(agents=_agents(2, batch_size=128, memory_size=128), memory_max=128) == _ENODEVICE
    for kw in ({"states": None}, {"ws": None}, {"avg": None}, {"q": None}, {"ends": ()}):
        assert _train(**kw) == _EINVAL, kw
    assert _train(S=0) == _EINVAL and _train(N=0) == _EINVAL and _train(A=0, agents=_agents(1)) == _EINVAL
    assert _train(offset=-1) == _EINVAL
    assert _train(points=0) == _EINVAL                                        # points_per_call < 1
    assert _train(ends=(19, 1000)) == _EINVAL and _train(ends=(-1,)) == _EINVAL   # a call end >= N, < 0
    assert _train(agents=_agents(2, symbol=2)) == _EINVAL                   # symbol out of range
    assert _train(agents=_agents(2, symbol=-1)) == _EINVAL
    assert _train(agents=_agents(2, batch_size=64, memory_size=63)) == _EINVAL   # batch > memory
    assert _train(agents=_agents(2, batch_size=0, memory_size=10)) == _EINVAL
    assert _train(agents=_agents(2, batch_size=129, memory_size=200)) == _EINVAL
    assert _train(agents=_agents(2, memory_size=10001)) == _EINVAL         # above the workspace's memory_max
    assert _train(agents=_agents(2, update_target_every=0)) == _EINVAL
    assert _train(memory_max=0) == _EINVAL
    assert _train(ws_bytes=int(_ws(2, 10000)) - 1) == _EINVAL     # undersized agent state
    assert _train(hist=DEV, rows=39) == _EINVAL                              # 20 + 20 points need 40 rows
    assert _train(N=1 << 40) == _ELIMIT


def _ws(A, M):
    from ai_crypto_trader_b200 import _lib
    return _lib.load().b200bt_rl_workspace_bytes(A, M)


def test_rl_states_refusals(native_lib):
    import torch
    f = lambda cols=DEV, close=DEV, vol=DEV, ld=100, S=2, N=100, bm=60, out=DEV: _status(
        "b200bt_rl_states", cols, close, vol, ld, S, N, bm, out, None)
    if not torch.cuda.is_available():
        assert f() == _ENODEVICE and f(bm=1) == _ENODEVICE and f(bm=15) == _ENODEVICE
    for kw in ({"cols": None}, {"close": None}, {"vol": None}, {"out": None}, {"S": 0}, {"N": 0}, {"ld": 99},
               {"bm": 0}, {"bm": 7}, {"bm": 120}, {"bm": 1440}):
        assert f(**kw) == _EINVAL, kw


@pytest.mark.parametrize("q, action", [((0.1, 0.2, 0.3), "SELL"), ((0.3, 0.3, 0.1), "BUY"), ((-0.5, -0.1, -0.2), "HOLD")])
def test_adjust_params_from_q_values(q, action):
    from ai_crypto_trader_b200.rl import adjust_params_from_q_values
    from ai_crypto_trader_b200.synth import param_ranges
    r = param_ranges(False)
    p = {"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30, "take_profit": 5, "stop_loss": 2,
         "social_sentiment_threshold": 60}
    out = adjust_params_from_q_values(p, q, r)
    changed = {k for k in p if out[k] != p[k]} - {"stop_loss"}
    assert changed == {"BUY": {"rsi_oversold", "social_sentiment_threshold"}, "SELL": {"rsi_overbought", "take_profit"},
                       "HOLD": {"rsi_period"}}[action]
    assert out["stop_loss"] == max(2 * (1 - max(q) * 0.2), r["stop_loss"][0])
    assert p["rsi_period"] == 14                                             # the input is not changed
