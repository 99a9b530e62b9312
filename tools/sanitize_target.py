#!/usr/bin/env python
"""Small workload for compute-sanitizer (memcheck / racecheck / initcheck): every kernel family once, at sizes a
40-100x slowdown still finishes.  The sweep legs force the speculative paths (no warm-up -> repair passes on the main
and on the side stream, a pool that overflows -> fused fallback) because that is where the bump allocator, the
linked event pool and the overlapped repair stream live.  Results are checked against the C oracle, so a sanitizer
run that "passes" also computed the right thing.

    compute-sanitizer --tool memcheck  python tools/sanitize_target.py
    compute-sanitizer --tool racecheck python tools/sanitize_target.py
"""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np
import torch

from ai_crypto_trader_b200 import indicators as ind, synth
from ai_crypto_trader_b200.monte_carlo import PathEngine, risk_statistics
from ai_crypto_trader_b200.sweep import MarketData, PopulationSweep
from oracle import indicators_ref, sim_oracle

legs = sys.argv[1:] or ["sweep", "mc", "joint", "indicators", "pareto", "regime", "dca", "grid_service", "rl"]
torch.cuda.set_device(0)

if "sweep" in legs:
    S, N, POP = 2, 40_000, 70
    ohlcv = synth.synth_ohlcv(S, N, first_symbol=1)
    market = MarketData(ohlcv)
    population = synth.random_population(POP, seed=11)
    population[0].update(rsi_oversold=35, rsi_overbought=65, rsi_period=5, take_profit=1, stop_loss=1)
    population[1].update(rsi_oversold=34, rsi_overbought=66, rsi_period=6, take_profit=10, stop_loss=5)
    cfg = sim_oracle.config_of(market.minute0, 1)
    banks = [indicators_ref.rsi_bank(ohlcv[3, s], list(range(5, 31))) for s in range(S)]
    want = np.array([[int(sim_oracle.lane(ohlcv[3, s], banks[s][p["rsi_period"] - 5], p, cfg)[0]["trade_hash"])
                      for s in range(S)] for p in population], dtype=np.uint64)
    for mode, opts in (("tiled", dict(warm=0, chunks=12, max_repair_rounds=64)),      # repaired chunk by chunk, side stream
                       ("tiled", dict(warm=1024, chunks=6)),                          # speculation mostly right
                       ("tiled", dict(warm=512, chunks=6, pool_blocks=8)),            # pool overflow -> fused fallback
                       ("tiled", dict(warm=1024, chunks=6, order_by="identity")),     # unpacked warps (> 2 RSI rows) -> flagged, fused fallback
                       ("chunked", dict(target_events=300, warm=0, max_chunks=16, max_repair_rounds=64)),
                       ("fused", {})):
        sw = PopulationSweep(market, event_cap=256, mode=mode, chunk_options=opts)
        sw.chunk_min_bars = 0
        for _ in range(2):                       # second sweep: zone map
            sw.evaluate(population)
        got = sw.lane_stats()["trade_hash"]
        assert np.array_equal(got, want), (mode, opts, int((got != want).sum()))
        print("sweep", mode, opts, "ok; invalid lanes", getattr(sw, "last_invalid_lanes", 0), flush=True)

if "mc" in legs:
    eng = PathEngine()
    f, d, paths = eng.gbm(100.0, 0.08, 0.35, 1 / 252, 5000, 64, 2024, store_paths=True)
    f2, d2, _ = eng.gbm(100.0, 0.08, 0.35, 1 / 252, 5000, 64, 2024)
    assert torch.equal(f, f2) and torch.equal(d, d2)
    ret = np.random.default_rng(3).normal(5e-4, 0.02, 60).astype(np.float32)
    eng.bootstrap(ret, True, 100.0, 3000, 45, 77, block_len=5)
    st = risk_statistics(eng, f, d, 100.0, 0.95)
    print("mc ok", st["var"], flush=True)

if "joint" in legs:
    # joint portfolio paths: every asset bucket (4 / 8 / 16 / 32), the bootstrap table staged in shared memory
    eng = PathEngine()
    for S in (3, 8, 13, 32):
        rng = np.random.default_rng(S)
        A = rng.normal(size=(S, S + 2)); c = A @ A.T; c /= np.sqrt(np.outer(np.diag(c), np.diag(c)))
        L = np.linalg.cholesky(c).astype(np.float32)
        s0, qty = rng.uniform(1, 100, S), rng.uniform(0.1, 10, S)
        f, d, af = eng.portfolio_gbm(s0, qty, rng.uniform(-0.1, 0.2, S), rng.uniform(0.2, 0.8, S), 1 / 252, L, 1000, 37,
                                     2024, path_offset=5, asset_finals=True)
        table = rng.normal(0, 0.02, (12288 // S, S)).astype(np.float32)
        fb, db, _ = eng.portfolio_bootstrap(table, False, s0, qty, 1000, 37, 7, block_len=3, asset_finals=True)
        assert bool(torch.isfinite(f).all() and torch.isfinite(fb).all() and (d >= 0).all() and (db >= 0).all())
    print("joint ok", float(f.mean()), float(fb.mean()), flush=True)

if "indicators" in legs:
    m = MarketData(synth.synth_ohlcv(2, 9000))
    ta = ind.TechnicalAnalyzer(m)
    ind.multi_timeframe_indicators(m, 0)
    print("indicators ok", ta.get_all_indicators(0)["rsi"], flush=True)
if "pareto" in legs:
    # multi-objective ranking: the cooperative peel (grid barriers, rotating counters, appended member slots) and the
    # dominance tile in opted-in dynamic shared memory, on heavy ties and duplicate rows; checked against the host form
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import pareto_ref
    from ai_crypto_trader_b200.pareto import pareto_rank
    obj, mx = pareto_ref.make_input("ties", 4101, 3)
    got = [t.cpu().numpy() for t in pareto_rank(torch.from_numpy(obj).cuda(), mx, with_key=True)]
    want = pareto_ref.pareto_numpy(obj, mx)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    print("pareto ok:", int(got[0].max()) + 1, "fronts of 4101 points, bit-identical to pareto_numpy", flush=True)
if "regime" in legs:
    # market regimes: the labelling pass (block-wide head search, one warp per window) and the class pass (per-class
    # shared-memory staging, R WarpAccs per warp), on a market with a NaN head and labels >= R; checked against the oracle
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import regime_ref
    from ai_crypto_trader_b200 import regime
    S, N, POP = 2, 6_000, 12
    ohlcv = synth.synth_ohlcv(S, N, first_symbol=2)
    market = MarketData(ohlcv)
    labels, _ = regime.regime_labels(market, 15)
    rows = regime.trend_rows(market).cpu().numpy()
    for s in range(S):
        assert np.array_equal(labels[s].cpu().numpy(), regime_ref.symbol_labels(*rows[:, s], market.minute0, 1, 15)[0])
    sweep = PopulationSweep(market, rsi_periods=range(5, 31))
    population = synth.random_population(POP, seed=2)
    mixed = torch.from_numpy(np.random.default_rng(0).integers(0, 7, (S, N)).astype(np.uint8)).cuda()
    _, views = sweep.class_stats(population, mixed, 5)
    cfg = sim_oracle.config_of(market.minute0, 1)
    lab = mixed.cpu().numpy()
    for s in range(S):
        bank = sweep.bank[s].cpu().numpy()
        for i, p in enumerate(population):
            _, ev, pn = sim_oracle.lane(ohlcv[3, s], bank[sweep.period_row[p["rsi_period"]]], p, cfg, event_cap=N + 2)
            want = regime_ref.class_stats(ev, pn, lab[s], 5, cfg)
            for r in range(5):
                assert views[r]["n_records"][i, s] == want[r]["n_records"]
                assert int(views[r]["trade_hash"][i, s]) == int(want[r]["trade_hash"])
    print("regime ok: labels equal the restatement,", S * POP, "lanes x 5 classes match the oracle", flush=True)
if "dca" in legs:
    # DCA: the drop series, the pyramid search, the rebalance and day-end barriers (S = 3) and the grouped CTA (S = 33)
    import random as _random
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import dca_ref
    from ai_crypto_trader_b200.dca import DCASweep, dca_param_ranges, decode_individual
    rng = _random.Random(5)
    pop = [{k: (rng.randint(lo, hi) if isinstance(lo, int) else rng.uniform(lo, hi))
            for k, (lo, hi) in dca_param_ranges().items()} for _ in range(12)]
    for S, N, reb in ((3, 12 * 1440, 1), (33, 3 * 288, 0)):
        ohlcv = synth.synth_ohlcv(S, N)
        ohlcv[1] = np.maximum(ohlcv[1], ohlcv[3])
        m = MarketData(ohlcv, bar_minutes=1 if S == 3 else 5)
        p = [dict(x, periodic_rebalancing=reb, rebalance_interval_days=1) for x in pop]
        sw = DCASweep(m, start_bar=N // 8, usdc_balance=900.0)
        st = sw.dca_stats(p)
        if reb:
            sw.day_pnl(p)
        for i in range(0, len(p), 5):
            want = dca_ref.simulate(m.close.cpu().numpy().astype(np.float64), sw.dip.cpu().numpy(), m.minute0,
                                    m.bar_minutes, sw.start_bar, decode_individual(p[i], {}, m.symbols, m.bar_minutes),
                                    usdc_balance=900.0)
            for s in range(S):
                assert st["purchase_hash"][i, s] == want["stats"][s]["purchase_hash"], (S, i, s)
        print("dca ok: S =", S, flush=True)
if "grid_service" in legs:
    # the coupled grid service: adjust-tick barriers, lane state kept in the stats records, symbol rounds (S = 17), day rows
    import random as _random
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import grid_service_ref
    from ai_crypto_trader_b200.grid import GridSweep, decode_individual
    rng = _random.Random(6)
    pop = [{"num_grids": rng.randint(3, 30), "grid_type": 0, "auto_boundaries": 0, "lower_boundary_pct": rng.uniform(0.5, 3),
            "upper_boundary_pct": rng.uniform(0.5, 3), "rebalance_frequency": rng.randint(60, 3600),
            "auto_adjust_period": rng.randint(300, 7200), "adapt_to_market_regime": 0} for _ in range(6)]
    for S in (3, 17):
        m = MarketData(synth.synth_ohlcv(S, 2 * 1440))
        sw = GridSweep(m, quantity=0.01, start_bar=100, service=True)
        st = sw.grid_stats(pop)
        sw.day_profit(pop)
        for i in range(0, len(pop), 3):
            d = decode_individual(pop[i], sw.defaults, 1)
            _, bounds = sw.decode([pop[i]])
            want = grid_service_ref.simulate_service(
                m.close.cpu().numpy().astype(np.float64)[:, 100:], [tuple(bounds[0, s]) for s in range(S)],
                d["num_grids"], 0, list(sw.quantity), d["lower_pct"], d["upper_pct"], d["rebalance_ticks"],
                d["adjust_ticks"])
            for s in range(S):
                assert st["total_trades"][i, s] == want["lanes"][s]["total_trades"], (S, i, s)
        print("grid_service ok: S =", S, flush=True)

torch.cuda.synchronize()
print("sanitize target done")
if "rl" in legs:
    # RL agents: the state table, replay-memory wraparound, batch 1 and 128, the target copy, the loss pass, two launches
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import rl_ref
    from ai_crypto_trader_b200.rl import SERVICE_AGENT, RLPopulation, rl_states
    m = MarketData(synth.synth_ohlcv(2, 400), bar_minutes=60)
    states = rl_states(m)
    agents = [dict(seed=1, symbol=0, batch_size=1, memory_size=1, update_target_every=2),
              dict(seed=2, symbol=1, batch_size=128, memory_size=130, update_target_every=3)]
    w0 = np.stack([rl_ref.init_weights(a["seed"], i) for i, a in enumerate(agents)])
    pop = RLPopulation(states, agents, init_weights=w0)
    ends = [150, 151, 300, 399, 20, 250, 260, 270]
    pop.train(ends[:3], history=True)
    pop.train(ends[3:], history=True)
    X = states.cpu().numpy()
    for i, a in enumerate(agents):
        ag = rl_ref.Agent(gid=i, weights=w0[i], **dict(SERVICE_AGENT, **a))
        rl_ref.train(ag, X[a["symbol"]], ends, 20, history=True)
        assert np.array_equal(pop.weight_vector(i), ag.weights) and pop.replays[i] == ag.replays, i
    print("rl ok:", int(pop.replays.sum()), "replays equal the restatement", flush=True)
