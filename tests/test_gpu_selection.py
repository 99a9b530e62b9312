"""The strategy selection replay on the GPU (csrc/selection.cu, ai_crypto_trader_b200/strategy_selection.py) against the
CPU oracle tests/selection_ref.py: every candidate's score at every check, the per-check rows, the switch list and the
stitched run, on seeded markets and at the replay's limits."""
import numpy as np
import pytest

import selection_ref
from gpu_fixtures import torch_cuda  # noqa: F401
from oracle import sim_oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-9


def _goals():
    from ai_crypto_trader_b200.sweep import DEFAULT_GOALS      # the service's sweep scores with config.json's goals
    return DEFAULT_GOALS


def _service(torch, S, N, bar_minutes, K, interval, expiry, seed=5, candidates=None, minute0_offset=7 * 60 + 13,
             thresholds=(0.15, 0.7)):
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.strategy_selection import StrategySelectionService
    from ai_crypto_trader_b200.sweep import MarketData
    ohlcv = synth.synth_ohlcv(S, N, seed_base=100 + seed)
    m = MarketData(ohlcv, minute0=synth.EPOCH_2024_MINUTES + minute0_offset, bar_minutes=bar_minutes)
    cands = candidates if candidates is not None else synth.random_population(K, seed=seed)
    svc = StrategySelectionService(m, cands)
    svc.check_interval, svc.cache_expiry = interval, expiry
    svc.min_improvement_threshold, svc.min_confidence_threshold = thresholds
    return svc, ohlcv[3].astype(np.float32)


def _oracle(svc, close, start_bar=0, labels=None):
    from ai_crypto_trader_b200.strategy_selection import check_bars, n_checks
    m, sw = svc.market, svc.sweep
    bank = sw.bank.cpu().numpy()
    cfg = sim_oracle.config_of(m.minute0, m.bar_minutes, _goals())
    records = selection_ref.candidate_records(close, bank, sw.period_row, svc.candidates, cfg)
    lab = svc.market_regime_service.labels()[0].cpu().numpy() if labels is None else labels
    every = check_bars(svc.check_interval, m.bar_minutes)
    host = selection_ref.host_service({"cache_expiry": svc.cache_expiry,
                                       "min_improvement_threshold": svc.min_improvement_threshold,
                                       "min_confidence_threshold": svc.min_confidence_threshold})
    out = selection_ref.replay(host, records, svc.candidates, lab, m.minute0, m.bar_minutes, start_bar, every,
                               n_checks(m.N, start_bar, every))
    return out, bank, records, host


def _near_tie(scores):
    """Per check: the oracle's top two scores lie within the tolerance, so either may be the computed maximum."""
    if scores.shape[1] < 2:
        return np.zeros(len(scores), dtype=bool)
    top = np.sort(scores, axis=1)
    return top[:, -1] - top[:, -2] <= RTOL * np.maximum(1.0, np.abs(top[:, -1]))


def _check(svc, close, start_bar=0, labels=None):
    """Replay against the oracle -> (replay dict, oracle scores [C][K]).
    Scores, factors and regimes to 1e-9.  The best of every check whose oracle top two are apart is the oracle's; at a
    near tie the chosen one's oracle score is within tolerance of the maximum.  The switch list and the active columns are
    exactly the reference's switch methods run on the GPU's own (best, score) rows, and they are the oracle's own wherever
    no check has a near tie.  The stitched run is the oracle's on the GPU's schedule, every segment scored from its slice."""
    from ai_crypto_trader_b200.regime import REGIMES
    from ai_crypto_trader_b200.strategy_selection import FACTORS, switch_schedule
    res = svc.replay(start_bar=start_bar, scores=True)
    assert res is not None
    (scores, factors, regimes, best, switches, active, active_score), bank, records, host = \
        _oracle(svc, close, start_bar, labels)
    np.testing.assert_allclose(res["scores"], scores, rtol=RTOL, atol=1e-12)
    rows = res["checks"]
    C = len(scores)
    assert len(rows) == C
    assert [REGIMES[int(r)] for r in rows["regime"]] == regimes
    from ai_crypto_trader_b200.strategy_selection import check_bars
    assert np.array_equal(rows["bar"], start_bar + np.arange(C) * check_bars(svc.check_interval, svc.market.bar_minutes))
    got_best = rows["best"].astype(np.int64)
    # the device's tie rule on its own scores: the first maximum, exactly
    assert np.array_equal(got_best, np.argmax(res["scores"], axis=1))
    tie = _near_tie(scores)
    assert np.array_equal(got_best[~tie], best[~tie])
    idx = np.arange(C)
    assert np.all(scores[idx, got_best] >= scores[idx, best] - RTOL * np.maximum(1.0, np.abs(scores[idx, best])))
    np.testing.assert_allclose(rows["score"], scores[idx, got_best], rtol=RTOL, atol=1e-12)
    for f, name in enumerate(FACTORS):
        np.testing.assert_allclose(rows[name], factors[idx, got_best, f], rtol=RTOL, atol=1e-12, err_msg=name)
    # the switch rule on the GPU's rows: exact
    sw, act, act_score = selection_ref.switch_run(host, got_best, rows["score"])
    assert [s["check"] for s in res["switches"]] == sw
    assert np.array_equal(rows["active"].astype(np.int64), act)
    assert np.array_equal(rows["active_score"], act_score)
    if not tie.any():
        assert sw == switches and np.array_equal(act, active) and np.array_equal(act_score, active_score)
    for s in res["switches"]:
        assert s["previous_strategy_id"] == s["new_strategy_id"]       # the reference's quirk
        assert s["bar"] == int(rows["bar"][s["check"]])
    m, sw_ = svc.market, svc.sweep
    assert res["schedule"] == switch_schedule([int(rows["bar"][c]) for c in sw], [int(got_best[c]) for c in sw], m.N)
    if res["schedule"]:
        want = selection_ref.schedule_stats(close, bank, sw_.period_row, svc.candidates, res["schedule"], m.minute0,
                                            m.bar_minutes, _goals())
        sim_oracle.assert_lanes(res["stitched"], want, "stitched")
    else:
        assert res["stitched"] is None
    for k in range(len(svc.candidates)):
        want = selection_ref.schedule_stats(close, bank, sw_.period_row, svc.candidates, [(start_bar, m.N, k)], m.minute0,
                                            m.bar_minutes, _goals())
        sim_oracle.assert_lanes({f: v[k] for f, v in res["candidates"].items()}, want, f"candidate {k}")
    return res, scores


@pytest.mark.parametrize("S, N, bar_minutes, K, interval, expiry", [
    (1, 3000, 1, 8, 60, 60),              # a check every bar, a refresh at every check
    (3, 12000, 1, 16, 300, 3600),
    (10, 4000, 5, 12, 300, 3600),
    (3, 6000, 5, 8, 300, 300),
    (1, 20000, 1, 64, 300, 3600),
], ids=["S1-1m-every-bar", "S3-1m-300s", "S10-5m-300s", "S3-5m-expiry-300", "S1-1m-K64"])
def test_replay_matches_the_oracle(torch_cuda, S, N, bar_minutes, K, interval, expiry):
    svc, close = _service(torch_cuda, S, N, bar_minutes, K, interval, expiry)
    res, scores = _check(svc, close)
    assert np.isclose(res["active_share"].sum(), (res["checks"]["active"] >= 0).mean())


@pytest.mark.parametrize("S, N, bar_minutes, K, interval, expiry, thresholds", [
    (3, 12000, 1, 16, 300, 3600, (0.0, 0.3)),
    (3, 12000, 1, 16, 300, 3600, (0.02, 0.5)),
    (1, 3000, 1, 8, 60, 60, (0.0, 0.3)),
], ids=["S3-1m-no-improvement", "S3-1m-low-thresholds", "S1-1m-every-bar-no-improvement"])
def test_many_switches_and_the_stitched_run(torch_cuda, S, N, bar_minutes, K, interval, expiry, thresholds):
    """Lower switch thresholds: several switches, so the ballot loop of the switch scan and a stitched run of several
    segments are held to the oracle."""
    svc, close = _service(torch_cuda, S, N, bar_minutes, K, interval, expiry, thresholds=thresholds)
    res, _ = _check(svc, close)
    assert len(res["switches"]) >= 3 and len(res["schedule"]) >= 2
    assert len({s["new_strategy_id"] for s in res["switches"]}) >= 2


def test_single_candidate_and_duplicates(torch_cuda):
    from ai_crypto_trader_b200 import synth
    base = synth.random_population(3, seed=9)
    svc, close = _service(torch_cuda, 2, 3000, 1, 0, 300, 3600, candidates=[base[0]])
    _check(svc, close)
    dup = [base[1], base[0], base[1], base[0]]
    svc, close = _service(torch_cuda, 2, 3000, 1, 0, 300, 3600, candidates=dup)
    res, scores = _check(svc, close)
    assert np.array_equal(scores[:, 0], scores[:, 2]) and np.array_equal(scores[:, 1], scores[:, 3])
    assert set(res["checks"]["best"].astype(int)) <= {0, 1}       # exact ties go to the lowest index
    # many copies over many CTAs: every tie still goes to the lowest index, on every run
    many = [base[i % 3] for i in range(96)]
    svc, close = _service(torch_cuda, 2, 3000, 1, 0, 300, 3600, candidates=many)
    first = svc.replay(scores=True)
    assert set(first["checks"]["best"].astype(int)) <= {0, 1, 2}
    assert np.array_equal(first["checks"]["best"], np.argmax(first["scores"], axis=1))
    for _ in range(2):
        again = svc.replay(scores=True)
        assert np.array_equal(again["checks"], first["checks"]) and again["switches"] == first["switches"]


def test_candidates_without_records_and_edge_checks(torch_cuda):
    from ai_crypto_trader_b200 import synth
    pop = synth.random_population(4, seed=13)
    idle = dict(pop[0], rsi_oversold=0, rsi_overbought=100)      # never enters
    cands = [idle, pop[1], dict(idle), pop[2]]
    svc, close = _service(torch_cuda, 3, 4000, 1, 0, 300, 3600, candidates=cands, minute0_offset=23 * 60 + 40)
    res, scores = _check(svc, close)
    assert res["candidates"]["n_records"][0].sum() == 0
    # first check at bar 0 and at N - 1
    for start in (0, svc.market.N - 1):
        _check(svc, close, start_bar=start)
    sel = svc.replay(start_bar=svc.market.N - 1)
    assert len(sel["checks"]) == 1


def test_all_unknown_labels(torch_cuda):
    svc, close = _service(torch_cuda, 2, 4000, 1, 10, 300, 3600, seed=21)
    N = svc.market.N
    svc.market_regime_service._labels = torch_cuda.full((2, N), 4, dtype=torch_cuda.uint8, device="cuda")
    res, _ = _check(svc, close, labels=np.full(N, 4, dtype=np.uint8))
    assert set(res["checks"]["regime"].astype(int)) == {4}


def test_resweep_and_candidate_batches_merge_into_the_same_rows(torch_cuda):
    svc, close = _service(torch_cuda, 3, 6000, 1, 12, 300, 3600, seed=31)
    ref = svc.replay(scores=True)
    svc._event_cap = 2                               # a learnt cap far too small: the slices are swept again
    again = svc.replay(scores=True)
    assert svc.sweep.book_resweeps > 0
    assert np.array_equal(again["checks"], ref["checks"]) and np.array_equal(again["scores"], ref["scores"])
    svc.sweep.max_event_bytes = 3 * 4 * int(svc.sweep.lane_stats()["n_records"].max() + 2) * 2   # two rows per slice
    svc._event_cap = 0
    batched = svc.replay(scores=True)
    assert svc.last_batches > 1
    assert np.array_equal(batched["checks"], ref["checks"]) and np.array_equal(batched["scores"], ref["scores"])
    _check(svc, close)


def test_lost_records_are_never_selected(torch_cuda):
    """A candidate whose lane holds more records than the event buffer is invalid: NaN scores, never the best."""
    import ctypes as C
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.strategy_selection import gene_table
    torch = torch_cuda
    svc, close = _service(torch, 2, 3000, 1, 6, 300, 3600, seed=41)
    ref = svc.replay(scores=True)
    m, sw = svc.market, svc.sweep
    packed, _, _ = sw._unique(svc.candidates)
    sw._evaluate_unique(packed, svc.candidates, None, 0)
    n = sw.lane_stats()["n_records"]
    busy = int(np.argmax(n.max(axis=1)))
    cap = int(n.max()) - 1
    sw._evaluate_unique(packed, svc.candidates, None, cap)
    K, Cn = len(svc.candidates), len(ref["checks"])
    dev = "cuda"
    rows = torch.empty((Cn, len(_lib.SEL_ROW)), dtype=torch.float64, device=dev)
    scores = torch.empty((Cn, K), dtype=torch.float64, device=dev)
    locks = torch.empty(Cn, dtype=torch.int32, device=dev)
    idx = torch.arange(K, dtype=torch.int32, device=dev)
    genes = torch.from_numpy(gene_table(svc.candidates)).to(dev)
    labels = svc.market_regime_service.labels()[:1].contiguous()
    indiv = torch.from_numpy(packed.view(np.uint8)).to(dev)
    _lib.call("b200bt_selection_replay", m.close.data_ptr(), _lib.ld(m.close), m.S, m.N, indiv.data_ptr(), K,
              C.byref(sw.cfg), sw._stats.data_ptr(), sw._events.data_ptr(), cap, labels.data_ptr(), 0, idx.data_ptr(),
              idx.data_ptr(), genes.data_ptr(), K, K, svc.params_array(0, 5), Cn, 0, rows.data_ptr(), scores.data_ptr(),
              locks.data_ptr(), _lib.current_stream())
    got = scores.cpu().numpy()
    assert np.isnan(got[:, busy]).all()
    others = [k for k in range(K) if n[k].max() <= cap]
    np.testing.assert_array_equal(got[:, others], ref["scores"][:, others])
    assert not np.any(rows.cpu().numpy()[:, _lib.SEL_ROW.index("best")] == busy)
