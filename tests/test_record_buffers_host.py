"""The synthetic event buffers of tests/record_buffers.py on the CPU: the invariant checker accepts what the C oracle
(oracle/sim_oracle.c) emits and refuses malformed lanes, the host pricer gives the oracle's record pnl bit for bit, and
every buffer tests/test_gpu_record_limits.py builds keeps the invariants and lands on the seams it names."""
import numpy as np
import pytest

import record_buffers as rb
import test_gpu_record_limits as limits
from oracle import sim_oracle

DENSE = dict(rsi_period=5, rsi_oversold=99, rsi_overbought=101, take_profit=0.0001, stop_loss=0.0001)


@pytest.mark.parametrize("bar_minutes, gap", [(1, None), (7, None), (1440, None), (1, (1201, 2 * 1440 + 17))])
def test_oracle_lanes_keep_the_invariants_and_the_pricer_is_exact(bar_minutes, gap):
    from ai_crypto_trader_b200 import synth
    S, N = 3, 3000
    close = synth.synth_ohlcv(S, N)[3]
    rng = np.random.default_rng(bar_minutes)
    pop = synth.random_population(12, seed=bar_minutes) + [dict(DENSE), dict(DENSE, max_position_size=13)]
    cfg = sim_oracle.config_of(limits.MINUTE0, bar_minutes)
    if gap is not None:
        cfg.gap_bar, cfg.gap_minutes = gap
    rsi = np.stack([rng.uniform(0.0, 100.0, N).astype(np.float32)[None] for _ in range(S)])      # one row per symbol
    stats, evs, pns = sim_oracle.population(close, rsi, lambda p: 0, pop, cfg, event_cap=N + 2)
    for i, p in enumerate(pop):
        for s in range(S):
            ev, pn = evs[i][s], pns[i][s]
            assert len(ev) == int(stats["n_records"][i, s])
            rb.check_lane(ev, N)
            got = rb.price_lane(ev, close[s], sim_oracle.params_of(p).position_size)
            assert np.array_equal(got.view(np.uint64), np.asarray(pn, dtype=np.float64).view(np.uint64)), (s, p)
    assert int(stats["n_records"].sum()) > 10_000                    # the dense lanes trade on most bars


@pytest.mark.parametrize("name", list(limits.CASES))
def test_every_gpu_case_keeps_the_invariants_and_lands_on_its_seams(name):
    case = limits.CASES[name]()
    events, stats = rb.pack(case.lanes, case.event_cap, case.n_records)
    rb.check_buffer(events, stats[..., 0], case.N)
    assert np.all(np.isnan(stats[..., 1:]))                   # the readers take n_records only
    assert case.seams and all(case.seams.values()), {k: v for k, v in case.seams.items() if not v}
    assert case.close.min() > 0 and np.all(np.isfinite(case.close))
    assert case.labels.shape == (case.S, case.N) and 1 <= case.R <= limits.CL_MAX


def _lane(*records):
    return np.array(records, dtype=np.uint32)


E, X, SELL = 0, rb.EXIT, rb.SELL
MALFORMED = [
    ("odd count", _lane(1 | E, 2 | X | SELL, 3 | E), "odd"),
    ("exit at an entry index", _lane(1 | X, 2 | X | SELL), "exit at an entry"),
    ("entry at an exit index", _lane(1 | E, 2 | E), "entry at an exit"),
    ("exit on its entry's side", _lane(1 | E, 2 | X), "same side"),
    ("bar not below N", _lane(1 | E, 100 | X | SELL), "not below"),
    ("bars going back", _lane(5 | E, 4 | X | SELL), "go back"),
    ("two records on a bar before the last", _lane(5 | E, 5 | X | SELL), "share bar"),
    ("the last bar's pair not last", _lane(99 | E, 99 | X | SELL, 99 | SELL, 99 | X), "share bar"),
    ("an exit and the next entry on one bar", _lane(1 | E, 2 | X | SELL, 2 | E, 3 | X | SELL), "share bar"),
]


@pytest.mark.parametrize("name, words, match", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_the_checker_refuses_malformed_lanes(name, words, match):
    with pytest.raises(ValueError, match=match):
        rb.check_lane(words, 100)


def test_the_checker_accepts_the_last_bar_pair_and_refuses_a_read_past_n_records():
    rb.check_lane(_lane(1 | E, 2 | X | SELL, 99 | SELL, 99 | X), 100)
    lanes = [[_lane(1 | E, 2 | X | SELL), _lane()]]
    events, stats = rb.pack(lanes, 4)
    rb.check_buffer(events, stats[..., 0], 100)
    events[0, 0, 3] = 3 | E                                   # a slot past n_records that is not POISON
    with pytest.raises(ValueError, match="POISON"):
        rb.check_buffer(events, stats[..., 0], 100)
    lost, stats = rb.pack([[_lane(1 | E, 2 | X | SELL, 3 | SELL, 4 | X)]], 3, n_records=[[4]])
    rb.check_buffer(lost, stats[..., 0], 100)                 # a lost lane: only its stored prefix is checked
    lost[0, 0, 2] = 3 | X
    with pytest.raises(ValueError):
        rb.check_buffer(lost, stats[..., 0], 100)


def test_a_read_past_n_records_would_change_the_results():
    """POISON is priced like any exit: a reader that took it would change pnl, counts and the day rows."""
    close = np.linspace(100.0, 120.0, 50).astype(np.float32)
    words = _lane(3 | E, 7 | X | SELL)
    read = rb.price_lane(np.append(words, [2 | E, rb.POISON]), close, 1000.0)
    assert read[-1] != 0.0 and np.isfinite(read[-1])
    assert rb.PAD_PRICE > 10 * close.max()                    # padding read as a close would move a pnl visibly
