"""Strategy selection replay timing on the configs[1] market (10 symbols x 1 000 000 one-minute bars): 300 s checks
(200 000 checks), 3 600 s cache expiry.

Rows (one JSON line each, with the card beside every number):
  replay_call     wall time of StrategySelectionService.replay(): labels, sweeps with event buffers, the replay and switch
                  kernels, the read-back and the stitched and per-candidate scoring, after one untimed call
  replay_kernel   CUDA-event time of one b200bt_selection_replay launch over the whole population's records
  switch_scan     CUDA-event time of b200bt_selection_switch over the rows
  book_metrics    CUDA-event time of b200bt_book_metrics on the same records, for scale
Shapes: the configs[1] population (1024 candidates) and the 64 fittest of generation 3 of the reference GA.

    python tools/selection_bench.py [--reps 5] [--bars 1000000]
"""
import argparse
import ctypes as C
import json
import statistics

import harness
import numpy as np
import torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--shapes", nargs="+", default=["configs1", "top64"])
    args = ap.parse_args()

    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.strategy_selection import StrategySelectionService, gene_table
    from ai_crypto_trader_b200.sweep import PopulationSweep
    torch.cuda.set_device(0)
    card = harness.card()
    market, population = harness.configs1(bars=args.bars)
    shapes = {}
    if "configs1" in args.shapes:
        shapes["configs1"] = population
    if "top64" in args.shapes:
        sweep = PopulationSweep(market)
        evolved = harness.generation3(sweep.fitness_function, population)
        fit = sweep.evaluate(evolved)
        order = np.argsort(-np.where(np.isnan(fit), -np.inf, fit), kind="stable")[:64]
        shapes["top64"] = [evolved[i] for i in order]
        del sweep

    for name, cands in shapes.items():
        svc = StrategySelectionService(market, cands)
        K = len(cands)

        def emit(row):
            print(json.dumps(dict(row, shape=name, candidates=K, symbols=market.S, bars=market.N, **card)), flush=True)

        with harness.sampled_clocks() as clk:
            ms, res = harness.wall_ms(lambda: svc.replay(), reps=args.reps, warmup=1)
        Cn = len(res["checks"])
        emit({"row": "replay_call", "ms_median": statistics.median(ms), "ms": ms, "checks": Cn,
              "switches": len(res["switches"]), "batches": svc.last_batches, "sm_clock": clk.sm_clock})
        if svc.last_batches != 1:
            emit({"row": "replay_kernel", "ms_median": "not measured: the records took more than one batch"})
            continue
        sw, m = svc.sweep, market
        dev = m.device
        packed, _, expand = sw._unique(svc.candidates)
        U = len(packed)
        cap = int(sw._events.shape[2])
        row_of = np.arange(K) if expand is None else np.asarray(expand)
        indiv = torch.from_numpy(packed.view(np.uint8)).to(dev)
        idx = torch.arange(K, dtype=torch.int32, device=dev)
        rows_of = torch.from_numpy(row_of.astype(np.int32)).to(dev)
        genes = torch.from_numpy(gene_table(svc.candidates)).to(dev)
        labels = svc.market_regime_service.labels()[:1].contiguous()
        params = svc.params_array(0, 5)
        rows = torch.empty((Cn, len(_lib.SEL_ROW)), dtype=torch.float64, device=dev)
        locks = torch.empty(Cn, dtype=torch.int32, device=dev)
        sws = torch.empty(Cn, dtype=torch.int32, device=dev)
        nsw = torch.empty(1, dtype=torch.int32, device=dev)
        book = torch.empty((U, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=dev)

        def replay():
            _lib.call("b200bt_selection_replay", m.close.data_ptr(), _lib.ld(m.close), m.S, m.N, indiv.data_ptr(), U,
                      C.byref(sw.cfg), sw._stats.data_ptr(), sw._events.data_ptr(), cap, labels.data_ptr(), 0,
                      rows_of.data_ptr(), idx.data_ptr(), genes.data_ptr(), K, K, params, Cn, 0, rows.data_ptr(), None,
                      locks.data_ptr(), _lib.current_stream())

        def switch():
            _lib.call("b200bt_selection_switch", rows.data_ptr(), Cn, params, sws.data_ptr(), nsw.data_ptr(),
                      _lib.current_stream())

        def book_metrics():
            _lib.call("b200bt_book_metrics", m.close.data_ptr(), _lib.ld(m.close), m.S, m.N, indiv.data_ptr(), U,
                      C.byref(sw.cfg), sw._stats.data_ptr(), sw._events.data_ptr(), cap, book.data_ptr(), None,
                      _lib.current_stream())

        ms = harness.event_ms(replay, args.reps)
        same = np.array_equal(rows.cpu().numpy()[:, :10], res["checks"].view(np.float64).reshape(Cn, -1)[:, :10],
                              equal_nan=True)
        n_records = int(sw._stats[:, :, 0].sum().item())
        emit({"row": "replay_kernel", "ms_median": statistics.median(ms), "ms": ms, "checks": Cn, "records": n_records,
              "rows_match_replay_call": same, "resources": harness.kernel_resources(["selection_kernel"])})
        ms = harness.event_ms(switch, args.reps)
        emit({"row": "switch_scan", "ms_median": statistics.median(ms), "ms": ms, "checks": Cn})
        ms = harness.event_ms(book_metrics, args.reps)
        emit({"row": "book_metrics", "ms_median": statistics.median(ms), "ms": ms, "records": n_records})


if __name__ == "__main__":
    main()
