"""b200bt_rl_states and b200bt_rl_train on the H100 against the restatement (tests/rl_ref.py, itself pinned to the
reference's TradingRLAgent by tests/golden/rl_reference.json), compared with ==: states; weights, target, counters,
Q-values, avg_reward and history of a mixed population (batch sizes 1 / 16 / 64 / 128, memory wraparound, target
boundaries, the epsilon floor); one launch against several; determinism; an agent alone against the same agent in a
population of 1 000 and under an agent offset; the device weight initialisation; the fixture's cases; and the service's
optimize_with_reinforcement_learning on a configs[1]-sized market."""
import json
from pathlib import Path

import numpy as np
import pytest

import rl_ref

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "rl_reference.json"


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def make_market(torch, S, N, bar_minutes=60, seed=3):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    ohlcv = synth.synth_ohlcv(S, N, seed_base=1000 + seed)
    ohlcv[:, 0, 200:260] = ohlcv[:, 0, 200:201]          # a flat run: zero Bollinger range, zero price changes
    return MarketData(ohlcv, bar_minutes=bar_minutes)


def analyzer_cols(market):
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.indicators import TechnicalAnalyzer
    ta = TechnicalAnalyzer(market)
    return np.stack([ta.data[name].cpu().numpy() for name in _lib.ANALYZER_COLUMNS])


@pytest.fixture(scope="module")
def hourly(torch):
    from ai_crypto_trader_b200.rl import rl_states
    m = make_market(torch, 3, 3000)
    return m, rl_states(m)


@pytest.mark.parametrize("bar_minutes", [60, 15, 1])
def test_states_equal_restatement(torch, bar_minutes):
    from ai_crypto_trader_b200.rl import rl_states
    m = make_market(torch, 3, 3000, bar_minutes)
    got = rl_states(m).cpu().numpy()
    want = rl_ref.states(analyzer_cols(m), m.close.cpu().numpy(), m.volume.cpu().numpy(), bar_minutes)
    assert np.array_equal(got, want)
    assert np.any(got[0, 200 + 21:260, 3] == 0.5)                          # zero range inside the flat run
    assert set(np.unique(got[..., 15])) == {0.2, 0.5, 0.8}
    h = 60 // bar_minutes
    assert np.all(got[:, :h, 10] == 0.5) and np.all(got[:, :1440 // bar_minutes, 11] == 0.5)


MIXED = [
    dict(seed=11, symbol=0),                                                 # the service's agent
    dict(seed=12, symbol=1, batch_size=1, memory_size=1, update_target_every=7),
    dict(seed=13, symbol=2, batch_size=16, memory_size=40, update_target_every=5, epsilon_decay=0.9, epsilon_end=0.2),
    dict(seed=14, symbol=0, batch_size=128, memory_size=130, update_target_every=3, learning_rate=0.01, gamma=0.5),
    dict(seed=15, symbol=1, batch_size=16, memory_size=10000, epsilon_start=0.3, epsilon_end=0.05, epsilon_decay=0.98),
    dict(seed=2 ** 64 - 1, symbol=2, batch_size=32, memory_size=33, update_target_every=1, learning_rate=0.05),
]
ENDS = [19, 60, 61, 400, 401, 402, 1500, 10, 2999, 2000, 777, 300]


def ref_agents(agents, offset=0, weights=None):
    from ai_crypto_trader_b200.rl import SERVICE_AGENT
    out = []
    for i, a in enumerate(agents):
        kw = dict(SERVICE_AGENT, **a)
        kw["seed"] = int(kw["seed"])
        w = None if weights is None else weights[i]
        out.append(rl_ref.Agent(gid=offset + i, weights=w, **kw))
    return out


def init_for(agents, offset=0):
    return np.stack([rl_ref.init_weights(int(a["seed"]), offset + i) for i, a in enumerate(agents)])


def check_equal(pop, refs, X, results):
    for i, ag in enumerate(refs):
        avg, q, hist = results[i]
        assert np.array_equal(pop.weight_vector(i), ag.weights), i
        assert np.array_equal(pop.weight_vector(i, target=True), ag.target), i
        assert pop.replays[i] == ag.replays and pop.epsilon[i] == ag.epsilon, i
        assert np.array_equal(pop.mean_q[i], ag.mean_q, equal_nan=True), i
        assert np.array_equal(pop.avg_reward[i], avg), i
        assert np.array_equal(pop.q_values[i], q), i
        if hist is not None:
            got = np.array([[r["loss"], r["mean_q"], r["epsilon"], r["step"]] for r in pop.training_history(i)]).reshape(-1, 4)
            assert np.array_equal(got, hist), i


def test_mixed_population_equals_restatement(torch, hourly):
    from ai_crypto_trader_b200.rl import RLPopulation
    _, states = hourly
    X = states.cpu().numpy()
    w0 = init_for(MIXED)
    pop = RLPopulation(states, MIXED, init_weights=w0).train(ENDS, 20, history=True)
    refs = ref_agents(MIXED, weights=w0)
    results = [rl_ref.train(ag, X[ag.symbol], ENDS, 20, history=True) for ag in refs]
    check_equal(pop, refs, X, results)
    n = sum(min(e + 1, 20) for e in ENDS)
    assert pop.replays[1] == n and pop.replays[0] == n - 63                  # memory 1 / batch 1, service batch 64
    assert 0.2 * 0.9 < pop.epsilon[2] <= 0.2                                 # the floor: decay stops at epsilon_end
    assert refs[3].memory_size < refs[3].n_transitions                     # wraparound


def test_split_launches_equal_one(torch, hourly):
    from ai_crypto_trader_b200.rl import RLPopulation
    _, states = hourly
    w0 = init_for(MIXED)
    one = RLPopulation(states, MIXED, init_weights=w0).train(ENDS, 20, history=True)
    split = RLPopulation(states, MIXED, init_weights=w0)
    q, avg = [], []
    for part in (ENDS[:1], ENDS[1:5], ENDS[5:]):
        split.train(part, 20, history=True)
        q.append(split.q_values)
        avg.append(split.avg_reward)
    assert np.array_equal(np.concatenate(q, axis=1), one.q_values)
    assert np.array_equal(np.concatenate(avg, axis=1), one.avg_reward)
    for i in range(len(MIXED)):
        assert np.array_equal(split.weight_vector(i), one.weight_vector(i))
        assert np.array_equal(split.weight_vector(i, True), one.weight_vector(i, True))
        assert split.training_history(i) == one.training_history(i)
    assert np.array_equal(split.epsilon, one.epsilon) and np.array_equal(split.replays, one.replays)
    # without a history the loss pass is skipped; nothing else changes
    quiet = RLPopulation(states, MIXED, init_weights=w0).train(ENDS, 20)
    assert np.array_equal(quiet.q_values, one.q_values) and np.array_equal(quiet.mean_q, one.mean_q)


def test_determinism_and_agent_independence(torch, hourly):
    from ai_crypto_trader_b200.rl import RLPopulation
    _, states = hourly
    rng = np.random.default_rng(5)
    agents = [dict(seed=int(s), symbol=int(rng.integers(0, 3)), batch_size=int(rng.choice([1, 16, 64])))
              for s in rng.integers(0, 2 ** 63, 1000)]
    ends = [100, 900, 901, 2500, 40]
    a = RLPopulation(states, agents).train(ends)
    b = RLPopulation(states, agents).train(ends)
    assert np.array_equal(a.q_values, b.q_values) and np.array_equal(a.epsilon, b.epsilon)
    for k in (0, 1, 517, 999):
        alone = RLPopulation(states, [agents[k]], agent_offset=k).train(ends)
        assert np.array_equal(alone.q_values[0], a.q_values[k])
        assert np.array_equal(alone.avg_reward[0], a.avg_reward[k])
        assert np.array_equal(alone.weight_vector(0), a.weight_vector(k))
        assert np.array_equal(alone.weight_vector(0, True), a.weight_vector(k, True))
    shard = RLPopulation(states, agents[500:], agent_offset=500).train(ends)
    assert np.array_equal(shard.q_values, a.q_values[500:])
    other = RLPopulation(states, [agents[517]]).train(ends)                  # another global index: another stream
    assert not np.array_equal(other.weight_vector(0), a.weight_vector(517))


def test_device_init_within_ulps(torch, hourly):
    from ai_crypto_trader_b200.rl import RLPopulation
    _, states = hourly
    agents = [dict(seed=s, symbol=0) for s in (0, 1, 2 ** 40 + 3)]
    pop = RLPopulation(states, agents, agent_offset=77).train([19])          # 20 points: no replay at batch 64
    assert np.all(pop.replays == 0)
    for i, a in enumerate(agents):
        got, want = pop.weight_vector(i), rl_ref.init_weights(a["seed"], 77 + i)
        np.testing.assert_array_max_ulp(got, want, maxulp=4)
        assert np.array_equal(got, pop.weight_vector(i, True))
        w = pop.weights(i)
        assert w["weights1"].shape == (16, 24) and np.all(w["bias1"] == 0) and np.all(w["bias3"] == 0)
        assert 0.08 < np.std(got[got != 0]) < 0.12


def test_fixture_cases(torch):
    """The reference fixture's cases from their injected weights: states, actions, rewards, counters exact; weights,
    history and Q-values within the fixture's tolerance of the reference (its BLAS order), and == the restatement."""
    from ai_crypto_trader_b200.rl import RLPopulation
    fx = json.loads(GOLDEN.read_text())
    for case in fx["cases"]:
        X = rl_ref.decode(case["states"]).reshape(-1, 16)
        states = torch.tensor(X[None], device="cuda")
        agent = dict(case["agent"], seed=case["seed"], symbol=0)
        w0 = rl_ref.fixture_weights(case["seed"])
        pop = RLPopulation(states, [agent], init_weights=w0[None]).train(case["call_ends"], case["points"], history=True)
        ref = ref_agents([agent], weights=[w0])[0]
        avg, q, hist = rl_ref.train(ref, X, case["call_ends"], case["points"], history=True)
        check_equal(pop, [ref], X, [(avg, q, hist)])
        tol = fx["tolerance"]
        assert pop.replays[0] == case["step_counter"] and pop.epsilon[0] == case["epsilon"]
        assert np.array_equal(pop.avg_reward[0], [c["avg_reward"] for c in case["calls"]])
        np.testing.assert_allclose(pop.q_values[0], [c["q_values"] for c in case["calls"]], rtol=tol, atol=tol)
        if "final_weights" in case:
            np.testing.assert_allclose(pop.weight_vector(0), rl_ref.decode(case["final_weights"]), rtol=tol, atol=tol)


def test_service_on_configs1_market(torch):
    """optimize_with_reinforcement_learning on BASELINE configs[1]'s shape (10 symbols x 1M 1-minute bars): the record,
    the persistent agent's counters and the adjusted parameters from its Q-values."""
    import asyncio
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.evolution import StrategyEvolutionService
    from ai_crypto_trader_b200.rl import adjust_params_from_q_values
    from ai_crypto_trader_b200.sweep import MarketData
    m = MarketData(synth.synth_ohlcv(10, 1_000_000))
    svc = StrategyEvolutionService(m, config={}, random_seed=9)
    params = dict(synth.random_population(1, seed=4)[0])
    out = None
    for k, end in enumerate(range(500_000, 500_080, 20)):
        out = asyncio.run(svc.optimize_with_reinforcement_learning(params, end, symbol=3))
        assert out is not None
        rec = svc.evolution_records[-1]
        assert rec["algorithm"] == "reinforcement_learning" and rec["old_params"] == params
        assert rec["new_params"] == out == adjust_params_from_q_values(params, rec["q_values"], svc.param_ranges)
        assert svc.rl_agents[3].replays[0] == max(0, 20 * (k + 1) - 63)
    eps = 1.0
    for _ in range(17):
        eps *= 0.995
    assert svc.rl_agents[3].epsilon[0] == eps and rec["epsilon"] == eps
    assert list(rec["q_values"]) == ["BUY", "HOLD", "SELL"] and np.isfinite(rec["avg_reward"])
    # a bad end bar: logged, None (the reference's convention)
    assert asyncio.run(svc.optimize_with_reinforcement_learning(params, 1_000_000, symbol=3)) is None
    res = svc.optimize_rl_population(params, [100_000 + 20 * i for i in range(10)],
                                     [dict(seed=s, symbol=s % 10) for s in range(64)])
    assert len(res) == 64 and all(np.isfinite(r["avg_reward"]) for r in res)
    assert np.all(svc.last_rl_population.replays == 200 - 63)
