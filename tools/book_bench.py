#!/usr/bin/env python
"""Cost of the book pass (b200bt_book_metrics) on the configs[1] workload, beside the sweep that feeds it.

    python tools/book_bench.py [--reps 5] [--check 3]

The configs[1] synthetic market of bench.py (10 symbols x 1M 1-minute bars) and two populations of 1024: the random one
(seed 42) and generation 3 of GeneticAlgorithm(seed 42) started from it (its lanes write several times more records).  For
each population, in alternating rounds, CUDA events time
  * the sweep without event buffers (PopulationSweep.evaluate_device, the plan `evaluate` uses);
  * the same sweep writing every lane's event words (event_cap = the busiest lane);
  * b200bt_book_metrics on those buffers.
records/s = the population's trade records / time.  `--check` books of each population (the busiest ones and a random
sample) are compared with the record-by-record oracle (tests/book_ref.py on the C oracle's lanes).  Prints one JSON line
with the card's name, power limit, the SM clock sampled while timing and the book kernel's registers / local memory.
Needs an H100; no fallback.
"""
import argparse
import ctypes as C
import json
import sys

import numpy as np
import torch

import harness


def _check(sweep, population, idx, close, bank):
    """Largest relative deviation of the GPU books `idx` (of the last book evaluation) from the oracle's."""
    from oracle import sim_oracle
    sys.path.insert(0, str(harness.ROOT / "tests"))
    import book_ref
    got = sweep.book_stats()
    cfg = sim_oracle.config_of(sweep.market.minute0, sweep.market.bar_minutes)
    _, evs, pns = sim_oracle.population(close, bank, sweep.period_row, [population[i] for i in idx], cfg,
                                        event_cap=close.shape[1] + 2)
    worst, exact = 0.0, True
    for i, ev, pn in zip(idx, evs, pns):
        want = book_ref.book(ev, pn, cfg)
        for f in sim_oracle.EXACT_FIELDS:
            exact &= bool(got[f][i] == want[f])
        for f in ("net_profit", "max_drawdown", "sharpe_ratio", "sortino_ratio", "score"):
            a, b = float(got[f][i]), float(want[f])
            if not (a == b or (np.isnan(a) and np.isnan(b))):
                worst = max(worst, abs(a - b) / max(abs(b), 1e-300))
    return {"books": len(idx), "exact_fields_equal": exact, "max_rel_dev": worst}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--check", type=int, default=3)
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--pop", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("book_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.sweep import PopulationSweep, decode_population
    torch.cuda.set_device(0)
    market, random_pop = harness.configs1(a.symbols, a.bars, a.pop)
    close = market.close.cpu().numpy()
    evolved = harness.generation3(PopulationSweep(market).fitness_function, random_pop)
    resources = harness.kernel_resources(["book_kernel"])
    out = {"workload": f"configs[1]: population {a.pop} x {a.symbols} symbols x {a.bars} 1-minute bars",
           **harness.card(), "book_kernel": resources and resources.get("book_kernel"), "populations": {}}
    rng = np.random.default_rng(7)
    for label, population in (("random", random_pop), ("generation_3", list(evolved))):
        sweep = PopulationSweep(market, aggregation="book")
        sweep.evaluate(population)                        # plans, buffers, zone map, learnt cap
        sweep.evaluate(population)
        packed = decode_population(population, sweep.period_row)
        pop = len(population)
        indiv = torch.from_numpy(packed.view(np.uint8)).to(market.device)
        plan = sweep.plan(population)
        lanes = sweep.lane_stats()
        records = float(lanes["n_records"].sum())
        cap = max(2, int(lanes["n_records"].max()))
        fit = torch.empty(pop, dtype=torch.float64, device=market.device)
        book = torch.empty((pop, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=market.device)
        st = _lib.current_stream()

        # the sweep without events runs on its own instance: one instance would reallocate (and zero) its event buffer
        # every time the event cap changes between the timed legs
        plain = PopulationSweep(market)
        plain.evaluate(population)
        plain_plan = plain.plan(population)
        plain_fit = torch.empty(pop, dtype=torch.float64, device=market.device)

        def sweep_plain():
            plain.evaluate_device(indiv, None, pop, plain_fit, plan=plain_plan, event_cap=0)

        def sweep_events():
            sweep.evaluate_device(indiv, None, pop, fit, plan=plan, event_cap=cap)

        def book_pass():
            _lib.call("b200bt_book_metrics", market.close.data_ptr(), _lib.ld(market.close), market.S, market.N,
                      indiv.data_ptr(), pop, C.byref(sweep.cfg), sweep._stats.data_ptr(), sweep._events.data_ptr(), cap,
                      book.data_ptr(), fit.data_ptr(), st)

        legs = {"sweep_no_events": sweep_plain, "sweep_with_events": sweep_events, "book_metrics": book_pass}
        sweep_plain(); sweep_events(); book_pass(); torch.cuda.synchronize()
        times = {k: [] for k in legs}
        with harness.sampled_clocks() as clocks:
            for _ in range(a.reps):
                for k, fn in legs.items():
                    if k == "book_metrics":
                        sweep_events()                    # the book reads the buffers this sweep wrote
                    times[k] += harness.event_ms(fn, 1, warmup=0)
        res = {k: {"ms_median": float(np.median(v)), "ms_runs": v, "records_per_s": records / (float(np.median(v)) * 1e-3)}
               for k, v in times.items()}
        # the timed book equals the one evaluate() returned
        mine = book.cpu().numpy()
        ref = sweep._book if sweep._inverse is None else None
        same = None if ref is None else bool(np.array_equal(mine[:, 0], ref[:, 0]) and
                                             np.array_equal(mine[:, -1].view(np.uint64), ref[:, -1].view(np.uint64)))
        busiest = list(np.argsort(-sweep.book_stats()["n_records"])[:max(1, a.check // 2)])
        sample = busiest + list(rng.choice(pop, size=max(0, a.check - len(busiest)), replace=False))
        check = _check(sweep, population, sample, close, sweep.bank.cpu().numpy()) if a.check else None
        out["populations"][label] = {"records": records, "busiest_lane": cap, "event_buffer_bytes": pop * market.S * cap * 4,
                                     "legs": res, "sm_clock": clocks.sm_clock, "timed_book_equals_evaluate": same,
                                     "oracle_check": check}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
