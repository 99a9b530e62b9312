"""CPU oracle of the strategy selection replay (b200bt_selection_replay / b200bt_selection_switch, strategy_selection.py).

Each candidate's records come from the C oracle (oracle/sim_oracle.lane per symbol), merged in book order as
book_ref.merged merges them.  Every (check, candidate) snapshot is built literally: the prefix of records with bar <= t_c
as trade dicts, StrategyPerformanceMetrics.calculate_metrics / calculate_advanced_metrics, the supplied params,
regime_performance and hourly_performance; the scores are the service's scalar methods and _calculate_regime_score on
those dicts; then the first maximum is selected and the switch methods run in check order.  The stitched run and each
candidate's own run are scored the way test_gpu_walk_forward scores a schedule: the oracle lane on each segment's slice,
then book_ref.book over the concatenation."""
from __future__ import annotations

import numpy as np

import book_ref
from oracle import sim_oracle


def drive(coro):
    """The value of a coroutine that never suspends (the service's async methods here await nothing real)."""
    try:
        coro.send(None)
    except StopIteration as e:
        return e.value
    raise RuntimeError("coroutine suspended")


def host_service(settings=None):
    """A StrategySelectionService with its reference settings and no market (the scalar methods only)."""
    from ai_crypto_trader_b200 import strategy_selection as ss
    svc = object.__new__(ss.StrategySelectionService)
    svc.selection_weights = ss.selection_weights_from_env()
    svc.min_improvement_threshold, svc.min_confidence_threshold = 0.15, 0.7
    svc.time_windows = {k: dict(v) for k, v in ss.TIME_WINDOWS.items()}
    svc.risk_profiles = {k: dict(v) for k, v in ss.RISK_PROFILES.items()}
    svc.current_risk_profile = "moderate"
    svc.cache_expiry = ss.CACHE_EXPIRY
    svc.active_strategy_id, svc.strategy_history, svc.strategy_selection = None, [], {}
    svc.strategy_metrics, svc.worker_parameters, svc.current_hour = {}, {}, 0
    for k, v in (settings or {}).items():
        setattr(svc, k, v)
    return svc


def _trade(minute0, bar_minutes, bar, sym, pnl):
    from ai_crypto_trader_b200.population import iso_minute
    return {"timestamp": iso_minute(minute0 + bar * bar_minutes), "symbol": str(sym), "pnl": pnl}


def snapshot(records, params, labels, minute0, bar_minutes):
    """The strategy_performance dict of a non-empty prefix [(bar, symbol, word, pnl)]."""
    from ai_crypto_trader_b200.regime import SCORED_REGIMES
    from ai_crypto_trader_b200.strategy_evaluation import StrategyPerformanceMetrics as M
    trades = [_trade(minute0, bar_minutes, b, s, p) for b, s, _, p in records]
    perf = M.calculate_advanced_metrics(M.calculate_metrics(trades))
    perf["params"] = params
    rp = {}
    for r, name in enumerate(SCORED_REGIMES):
        sub = [t for t, (b, _, _, _) in zip(trades, records) if labels[b] == r]
        if not sub:
            continue
        pn = [t["pnl"] for t in sub]
        loss = sum(p for p in pn if p < 0)
        cm = M.calculate_metrics(sub)
        rp[name] = {"trade_count": len(sub), "win_rate": sum(p > 0 for p in pn) / len(sub),
                    "profit_factor": sum(pn) / abs(loss) if loss != 0 else 1,
                    "sharpe_ratio": cm["sharpe_ratio"], "max_drawdown": cm["max_drawdown"]}
    perf["regime_performance"] = rp
    hourly = {}
    for b, _, _, p in records:
        h = str(((minute0 + b * bar_minutes) // 60) % 24)
        e = hourly.setdefault(h, [0, 0])
        e[0] += 1
        e[1] += p > 0
    perf["hourly_performance"] = {h: {"win_rate": w / n, "trade_count": n} for h, (n, w) in hourly.items()}
    return perf


def candidate_records(close, bank, period_row, candidates, cfg):
    """Per candidate: its records [(bar, symbol, word, pnl)] in book order."""
    N = close.shape[1]
    _, events, pnl = sim_oracle.population(close, bank, period_row, candidates, cfg, event_cap=N + 1)
    return [book_ref.merged(events[i], pnl[i]) for i in range(len(candidates))]


def replay(svc, records, candidates, labels, minute0, bar_minutes, start_bar, every, n_checks):
    """(scores [C][K], factors [C][K][6], regime names [C], best [C], switch checks, active [C], active score [C])."""
    from ai_crypto_trader_b200.regime import MarketRegimeService, REGIMES
    K = len(candidates)
    minute_of = lambda t: minute0 + t * bar_minutes
    strategies = [{"worker_id": k} for k in range(K)]
    svc.worker_parameters = {k: p for k, p in enumerate(candidates)}
    check_bars = [start_bar + c * every for c in range(n_checks)]
    plans = [set(refresh_checks(check_bars, rec[0][0] if rec else None, minute_of, svc.cache_expiry)) for rec in records]
    bar_arr = [np.array([r[0] for r in rec], dtype=np.int64) for rec in records]
    cache = [None] * K            # the cached snapshot of each candidate
    memo = [(-1, None)] * K
    scores = np.zeros((n_checks, K))
    factors = np.zeros((n_checks, K, 6))
    regimes, best = [], []
    for c, t in enumerate(check_bars):
        now = minute_of(t)
        for k in range(K):
            if c in plans[k]:
                n = int(np.searchsorted(bar_arr[k], t, side="right"))
                if n != memo[k][0]:          # the same prefix gives the same snapshot
                    memo[k] = (n, snapshot(records[k][:n], candidates[k], labels, minute0, bar_minutes))
                cache[k] = memo[k][1]
        svc.strategy_metrics = {k: (cache[k] if cache[k] else {}) for k in range(K)}
        svc.current_hour = (now // 60) % 24
        lab = int(labels[t])
        regime = REGIMES[lab] if lab < 4 else "unknown"
        regimes.append(regime)
        rs = {k: MarketRegimeService._calculate_regime_score(None, svc.strategy_metrics[k], regime) for k in range(K)}
        parts = [rs, drive(svc.calculate_historical_performance_scores(strategies)),
                 drive(svc.calculate_risk_scores(strategies)), drive(svc.calculate_social_sentiment_scores(strategies)),
                 drive(svc.calculate_volatility_scores(strategies)), drive(svc.calculate_feature_importance_scores(strategies))]
        w = svc.selection_weights
        combined = {}
        for k in range(K):
            combined[k] = (parts[0].get(k, 0.0) * w["market_regime"] + parts[1].get(k, 0.0) * w["historical_performance"] +
                           parts[2].get(k, 0.0) * w["risk_profile"] + parts[3].get(k, 0.0) * w["social_sentiment"] +
                           parts[4].get(k, 0.0) * w["market_volatility"] + parts[5].get(k, 0.0) * w["feature_importance"])
            factors[c, k] = [parts[f][k] for f in range(6)]
        final = drive(svc.apply_time_based_adjustments(combined))
        scores[c] = [final[k] for k in range(K)]
        best.append(max(final.items(), key=lambda x: x[1])[0])
    switches, active, active_score = switch_run(svc, best, scores[np.arange(n_checks), best])
    return scores, factors, regimes, np.array(best), switches, active, active_score


def refresh_checks(check_bars, first_record_bar, minute_of, expiry_s):
    """The checks at which one candidate fetches a snapshot (get_strategy_metrics :171-258): the first check whose prefix
    holds a record (an empty fetch is not cached), then every check at least expiry_s seconds after the last fetch.
    check_bars: the checks' bars; first_record_bar: the bar of the candidate's first record (None: it has none);
    minute_of: bar -> minute."""
    out, tau = [], None
    for c, t in enumerate(check_bars):
        if tau is None:
            if first_record_bar is not None and t >= first_record_bar:
                out.append(c)
                tau = minute_of(t)
        elif (minute_of(t) - tau) * 60 >= expiry_s:
            out.append(c)
            tau = minute_of(t)
    return out


def switch_run(svc, best, score):
    """The service's should_switch_strategy / switch_strategy over checks in order, on per-check (best, score) rows (best
    < 0: no valid candidate, no selection) -> (switch checks, active [C] (-1: none), active score [C])."""
    svc.active_strategy_id, svc.strategy_selection, svc.strategy_history = None, {}, []
    switches, active, active_score = [], [], []
    for c, (b, x) in enumerate(zip(best, score)):
        if b >= 0:
            new = {"worker_id": int(b), "selection_score": float(x), "selection_confidence": float(x)}
            if drive(svc.should_switch_strategy(svc.active_strategy_id, new)):
                drive(svc.switch_strategy(new))
                switches.append(c)
        a = svc.active_strategy_id
        active.append(-1 if a is None else a)
        active_score.append(svc.strategy_selection[a]["selection_score"] if a is not None else 0.0)
    return switches, np.array(active, dtype=np.int64), np.array(active_score)


def schedule_stats(close, bank, period_row, candidates, sched, minute0, bar_minutes, goals):
    """Book stats per symbol of schedule [(start, end, candidate)]: the oracle lane on each segment's slice."""
    out = []
    for s in range(close.shape[0]):
        words, pnls = [], []
        for a, b, k in sched:
            p = candidates[k]
            cfg = sim_oracle.config_of(minute0 + a * bar_minutes, bar_minutes, goals)
            row = period_row[int(p.get("rsi_period", 14))]
            _, ev, pn = sim_oracle.lane(close[s, a:b], bank[s, row, a:b], p, cfg, event_cap=b - a + 1)
            words.append(ev.astype(np.uint32) + np.uint32(a))
            pnls.append(pn)
        w = np.concatenate(words) if words else np.zeros(0, np.uint32)
        pn = np.concatenate(pnls) if pnls else np.zeros(0)
        out.append(book_ref.book([w], [pn], sim_oracle.config_of(minute0, bar_minutes, goals)))
    return out
