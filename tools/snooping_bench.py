#!/usr/bin/env python
"""Cost of the data-snooping tests (csrc/overfitting.cu b200bt_spa_moments / b200bt_spa_bootstrap, overfitting.spa) on
the configs[1] workload.

    python tools/snooping_bench.py [--reps 5] [--boot 10000]

* the book rows (PopulationSweep.daily_pnl, one row per calendar day) of the two populations of tools/book_bench.py on
  the configs[1] synthetic market (10 symbols x 1M 1-minute bars, 695 days): the random one (seed 42) and generation 3
  of GeneticAlgorithm(seed 42) started from it -- N = 1024 trials each;
* N = 10 000 trials of as many days (normal rows), the size of a large search.
At B = --boot resamples and a mean block length of 10 days: b200bt_spa_moments and one n_stats = 4 launch of
b200bt_spa_bootstrap (the Reality Check and the three SPA rows) timed with CUDA events, and the whole spa() call (its
StepM launches and copies included) on the host clock with a device synchronise.  Prints one JSON line with the card's
name, power limit, the SM clock sampled while timing and the kernels' registers.  Needs an H100; no fallback.
"""
import argparse
import json

import numpy as np
import torch

import harness


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--boot", type=int, default=10_000)
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--pop", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("snooping_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.overfitting import spa, spa_q32, spa_shifts
    from ai_crypto_trader_b200.sweep import PopulationSweep
    torch.cuda.set_device(0)
    market, random_pop = harness.configs1(a.symbols, a.bars, a.pop)
    evolved = harness.generation3(PopulationSweep(market).fitness_function, random_pop)
    matrices = {}
    for label, population in (("random", random_pop), ("generation_3", list(evolved))):
        book, _, _ = PopulationSweep(market).daily_pnl(population)
        matrices[f"{label}, N={book.shape[0]}"] = book
    D = int(book.shape[1])
    matrices["normal rows, N=10000"] = torch.from_numpy(np.random.default_rng(3).normal(0.0, 1.0, (10_000, D))).cuda()
    q32 = spa_q32(10.0)
    out = {"workload": f"configs[1]: book rows of {a.symbols} symbols x {a.bars} 1-minute bars, {D} days; B = {a.boot}, "
                       f"block_len = 10", **harness.card(),
           "kernels": harness.kernel_resources(["spa_moments_kernel", "spa_bootstrap_kernelILb1", "spa_bootstrap_kernelILb0"]),
           "spa": {}}
    st = _lib.current_stream()
    with harness.sampled_clocks() as clocks:
        for label, x in matrices.items():
            N, T = int(x.shape[0]), int(x.shape[1])
            mean = torch.empty(N, dtype=torch.float64, device="cuda")
            omega2 = torch.empty(N, dtype=torch.float64, device="cuda")

            def moments():
                _lib.call("b200bt_spa_moments", x.data_ptr(), _lib.ld(x), N, T, q32 / 2.0 ** 32, mean.data_ptr(),
                          omega2.data_ptr(), st)

            t_mom = harness.event_ms(moments, a.reps)
            m, w2 = mean.cpu().numpy(), omega2.cpu().numpy()
            w = np.where(w2 > 0, np.sqrt(np.where(w2 > 0, w2, 1.0)), np.nan)
            shift, scale = (torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in spa_shifts(m, w, T))
            res = torch.empty((4, a.boot), dtype=torch.float64, device="cuda")

            def bootstrap():
                _lib.call("b200bt_spa_bootstrap", x.data_ptr(), _lib.ld(x), N, T, q32, a.boot, 0, 0, 4, shift.data_ptr(),
                          scale.data_ptr(), res.data_ptr(), st)

            t_boot = harness.event_ms(bootstrap, a.reps)
            t_call, r = harness.wall_ms(lambda: spa(x, n_boot=a.boot, block_len=10.0), a.reps, warmup=1)
            adds = float(N) * T * a.boot
            med = float(np.median(t_boot))
            out["spa"][label] = {
                "trials": N, "days": T, "eligible": int(np.isfinite(w).sum()),
                "spa_moments_ms": {"median": float(np.median(t_mom)), "runs": t_mom},
                "bootstrap_n_stats_4_ms": {"median": med, "runs": t_boot},
                "bootstrap_gathered_adds_per_s": adds / (med * 1e-3),
                "spa_call_ms": {"median": float(np.median(t_call)), "runs": t_call},
                "stepm_steps": len(r["stepm"]["critical_values"]), "stepm_rejected": int(r["stepm"]["rejected"].sum()),
                "pvalues": {"reality_check": r["reality_check"]["pvalue"], **{k: v for k, v in r["spa"].items() if
                                                                               k.startswith("pvalue")}}}
    out["sm_clock"] = clocks.sm_clock
    print(json.dumps(out))


if __name__ == "__main__":
    main()
