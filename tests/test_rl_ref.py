"""The restatement of the reinforcement-learning kernels (tests/rl_ref.py) against the reference's own TradingRLAgent and
StrategyEvolutionService helpers (tests/golden/rl_reference.json, written by tests/golden/make_rl.py): states, rewards,
actions, step counts, epsilon, target-copy steps, average rewards and adjusted parameters exactly; weights, Q-values and
the history's loss / mean_q within the fixture's tolerance.  The reference sums its dot products and means in BLAS and
pairwise order, the restatement (and the kernel) in index order; after a few hundred replays that leaves ~1e-12 relative."""
import json
from pathlib import Path

import numpy as np
import pytest

import rl_ref

FIXTURE = json.loads((Path(__file__).resolve().parent / "golden" / "rl_reference.json").read_text())
CASES = FIXTURE["cases"]
COLS = {"sma_20": 0, "sma_50": 1, "ema_12": 3, "ema_26": 4, "macd": 5, "macd_signal": 6, "rsi": 10, "bb_high": 11,
        "bb_mid": 12, "bb_low": 13, "atr": 15}


def case_states(case):
    N = len(rl_ref.decode(case["close"], np.float32))
    cols = np.zeros((21, 1, N), dtype=np.float32)
    for name, v in case["cols"].items():
        cols[COLS[name], 0] = rl_ref.decode(v, np.float32)
    close = rl_ref.decode(case["close"], np.float32)[None]
    vol = rl_ref.decode(case["volume"], np.float32)[None]
    return rl_ref.states(cols, close, vol, case["bar_minutes"])[0]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_states_equal_reference(case):
    got = case_states(case)
    want = rl_ref.decode(case["states"]).reshape(got.shape)
    assert np.array_equal(got, want)


def test_fixture_reaches_every_state_branch():
    allx = np.concatenate([case_states(c) for c in CASES])
    assert set(np.unique(allx[:, 15])) == {0.2, 0.5, 0.8}                    # every trend
    assert np.any(allx[:, 3] == 0.5) and np.any(allx[:, 4] == 0.5)           # a zero Bollinger range
    c4 = case_states(CASES[3])                                               # 30-minute clock
    assert np.all(c4[:2, 10] == 0.5) and np.all(c4[:48, 11] == 0.5) and c4[2, 10] != 0.5 and c4[48, 11] != 0.5


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_training_equals_reference(case):
    from ai_crypto_trader_b200.rl import adjust_params_from_q_values
    from ai_crypto_trader_b200.synth import param_ranges
    X = rl_ref.decode(case["states"]).reshape(-1, 16)
    ag = rl_ref.Agent(seed=case["seed"], weights=rl_ref.fixture_weights(case["seed"]), trace=[], **case["agent"])
    avg, q, hist = rl_ref.train(ag, X, case["call_ends"], case["points"], history=True)
    acts = [r for r in ag.trace if r[0] == "act"]
    assert "".join(str(r[3]) for r in acts) == case["actions"]
    assert np.array_equal([r[4] for r in acts], rl_ref.decode(case["rewards"]))
    assert ag.replays == case["step_counter"] and ag.epsilon == case["epsilon"]
    period = case["agent"]["update_target_every"]
    assert [k for k in range(1, ag.replays + 1) if k % period == 0] == case["target_copies"]
    tol = FIXTURE["tolerance"]
    ranges = param_ranges(case["leverage"])
    params = {"rsi_period": 14, "rsi_overbought": 70, "rsi_oversold": 30, "take_profit": 5, "stop_loss": 2,
              "social_sentiment_threshold": 60}
    eps = [row[2] for row in hist]
    for k, call in enumerate(case["calls"]):
        assert avg[k] == call["avg_reward"]
        np.testing.assert_allclose(q[k], call["q_values"], rtol=tol, atol=tol)
        new = adjust_params_from_q_values(params, call["q_values"], ranges)
        assert new == call["new_params"] and all(type(new[n]) is type(call["new_params"][n]) for n in new)
        params = new
    # epsilon after each call: the history's epsilon at the call's last replay (1.0 before the first)
    done = 0
    pts = [min(e + 1, case["points"]) for e in case["call_ends"]]
    first = case["agent"]["batch_size"]
    seen = 0
    for k, n in enumerate(pts):
        seen += n
        reps = max(0, seen - first + 1)
        want = 1.0 if reps == 0 else eps[reps - 1]
        assert case["calls"][k]["epsilon"] == want, k
        done = reps
    assert done == len(hist)
    ref_hist = rl_ref.decode(case["history_loss_mean_q"]).reshape(-1, 2)
    np.testing.assert_allclose(hist[:, :2], ref_hist, rtol=tol, atol=tol)
    if "final_weights" in case:
        np.testing.assert_allclose(ag.weights, rl_ref.decode(case["final_weights"]), rtol=tol, atol=tol)
