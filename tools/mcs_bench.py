#!/usr/bin/env python
"""Cost of the Model Confidence Set (csrc/overfitting.cu b200bt_boot_means / b200bt_mcs_* / b200bt_autocov,
overfitting.mcs) on the configs[1] workload.

    python tools/mcs_bench.py [--reps 3] [--boot 10000] [--compare-lib OTHER.so]

* the book rows of the random population and of its GA generation 3 on the configs[1] market (as
  tools/snooping_bench.py builds them; N = 1024 trials of 695 days each);
* N = 10 000 normal rows of as many days (T_R only by default: T_max reads the [B][N] means about N / 2 times).
At B = --boot resamples and a mean block length of 10 days, each entry point is timed with CUDA events and the whole
mcs() call on the host clock with a device synchronise.  With --compare-lib, b200bt_spa_bootstrap (n_stats = 4) of this
build and of the other library are timed alternately on the same rows.  Prints one JSON line with the card's name,
power limit, the SM clock sampled while timing and the kernels' registers.  Needs an H100; no fallback.
"""
import argparse
import ctypes as C
import json

import numpy as np
import torch

import harness

KERNELS = ["boot_means_kernelILb1", "boot_means_kernelILb0", "spa_bootstrap_kernelILb1", "autocov_kernel",
           "mcs_pairwise_kernel", "mcs_range_stats_kernel", "mcs_range_order_kernel", "mcs_rank_rho_kernel",
           "mcs_range_boot_kernel", "mcs_range_count_kernel", "mcs_max_init_kernel", "mcs_max_rows_kernel",
           "mcs_max_var_kernel", "mcs_max_step_kernel"]


def med(runs):
    return {"median": float(np.median(runs)), "runs": runs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--boot", type=int, default=10_000)
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--pop", type=int, default=1024)
    ap.add_argument("--max-n-tmax", type=int, default=2048, help="largest N whose T_max is timed")
    ap.add_argument("--compare-lib", default=None, help="another libb200bt.so whose spa_bootstrap is timed alternately")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mcs_bench needs a CUDA device (H100); there is no CPU path")
    from ai_crypto_trader_b200 import _lib
    from ai_crypto_trader_b200.overfitting import mcs, optimal_block_length, spa_q32
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
    B = a.boot
    BIG = 1 << 40
    out = {"workload": f"configs[1]: book rows of {a.symbols} symbols x {a.bars} 1-minute bars, {D} days; B = {B}, "
                       "block_len = 10", **harness.card(), "kernels": harness.kernel_resources(KERNELS), "mcs": {}}
    st = _lib.current_stream()
    f64 = lambda *s: torch.empty(s, dtype=torch.float64, device="cuda")
    with harness.sampled_clocks() as clocks:
        for label, x in matrices.items():
            N, T = int(x.shape[0]), int(x.shape[1])
            mean, z = f64(N), f64(B, N)
            acov = f64(N, 1)
            _lib.call("b200bt_autocov", x.data_ptr(), _lib.ld(x), N, T, 0, acov.data_ptr(), mean.data_ptr(), st)
            r = {"trials": N, "days": T}
            r["boot_means_ms"] = med(harness.event_ms(lambda: _lib.call(
                "b200bt_boot_means", x.data_ptr(), _lib.ld(x), N, T, q32, B, 0, 0, mean.data_ptr(), z.data_ptr(), N, BIG,
                st), a.reps))
            w, t = torch.zeros((N, N), dtype=torch.float64, device="cuda"), f64(N, N)
            r["pairwise_ms"] = med(harness.event_ms(lambda: _lib.call(
                "b200bt_mcs_pairwise", z.data_ptr(), N, N, B, w.zero_().data_ptr(), BIG, st), a.reps))
            r["range_stats_ms"] = med(harness.event_ms(lambda: _lib.call(
                "b200bt_mcs_range_stats", mean.data_ptr(), N, B, w.data_ptr(), t.data_ptr(), BIG, st), 1, warmup=0))
            order, stat = torch.empty(N, dtype=torch.int32, device="cuda"), f64(N)
            rho_rank = f64(N, N)
            r["range_order_ms"] = med(harness.event_ms(lambda: _lib.call(
                "b200bt_mcs_range_order", t.data_ptr(), w.data_ptr(), N, order.data_ptr(), stat.data_ptr(),
                rho_rank.data_ptr(), BIG, st), a.reps))
            del w, t
            rmax = f64(B, N)
            count = torch.zeros(N, dtype=torch.int64, device="cuda")
            r["range_boot_ms"] = med(harness.event_ms(lambda: _lib.call(
                "b200bt_mcs_range_boot", z.data_ptr(), N, N, B, order.data_ptr(), rho_rank.data_ptr(), stat.data_ptr(),
                rmax.data_ptr(), count.data_ptr(), BIG, st), a.reps))
            del rmax, rho_rank
            K = min(int(np.ceil(np.sqrt(T))) + 10, T - 1)
            acov = f64(N, K + 1)
            r["autocov_ms"] = med(harness.event_ms(lambda: _lib.call(
                "b200bt_autocov", x.data_ptr(), _lib.ld(x), N, T, K, acov.data_ptr(), None, st), a.reps))
            r["block_len_auto"] = optimal_block_length(x)["block_len"]
            t_call, res = harness.wall_ms(lambda: mcs(x, statistic="R", n_boot=B, block_len=10.0), a.reps, warmup=1)
            r["mcs_R_call_ms"] = med(t_call)
            r["mcs_R_set_size"] = int(res["included"].sum())
            if N <= a.max_n_tmax:
                ws_bytes = int(_lib.load().b200bt_mcs_max_workspace_bytes(N, B))
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
                r["mcs_max_entry_ms"] = med(harness.event_ms(lambda: _lib.call(
                    "b200bt_mcs_max", z.data_ptr(), N, N, B, mean.data_ptr(), ws.data_ptr(), ws_bytes, order.data_ptr(),
                    stat.data_ptr(), count.zero_().data_ptr(), BIG, st), 1, warmup=0))
                # where the step loop's time goes: the device time of each kernel (torch.profiler, a run of its own)
                # against the entry's event time, and the same loop at B = 1, where every launch does almost no work
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    _lib.call("b200bt_mcs_max", z.data_ptr(), N, N, B, mean.data_ptr(), ws.data_ptr(), ws_bytes,
                              order.data_ptr(), stat.data_ptr(), count.zero_().data_ptr(), BIG, st)
                    torch.cuda.synchronize()
                dev_us = lambda e: getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                r["mcs_max_kernel_ms"] = {e.key.split("(")[0][-40:]: dev_us(e) / 1e3 for e in prof.key_averages()
                                          if "mcs_max" in e.key}
                ws1 = torch.empty(int(_lib.load().b200bt_mcs_max_workspace_bytes(N, 1)), dtype=torch.uint8,
                                  device="cuda")
                r["mcs_max_entry_B1_ms"] = med(harness.event_ms(lambda: _lib.call(
                    "b200bt_mcs_max", z.data_ptr(), N, N, 1, mean.data_ptr(), ws1.data_ptr(), ws1.numel(),
                    order.data_ptr(), stat.data_ptr(), count.zero_().data_ptr(), BIG, st), a.reps))
                t_call, res = harness.wall_ms(lambda: mcs(x, statistic="max", n_boot=B, block_len=10.0), 1)
                r["mcs_max_call_ms"] = med(t_call)
                r["mcs_max_set_size"] = int(res["included"].sum())
            if a.compare_lib:
                other = C.CDLL(a.compare_lib)
                other.b200bt_spa_bootstrap.restype = C.c_int
                other.b200bt_spa_bootstrap.argtypes = _lib.load().b200bt_spa_bootstrap.argtypes
                sh = torch.zeros((4, N), dtype=torch.float64, device="cuda")
                sc = torch.ones((4, N), dtype=torch.float64, device="cuda")
                o1, o2 = f64(4, B), f64(4, B)
                args = lambda o: (x.data_ptr(), _lib.ld(x), N, T, q32, B, 0, 0, 4, sh.data_ptr(), sc.data_ptr(),
                                  o.data_ptr(), st)
                new, old = [], []
                for _ in range(2 * a.reps):
                    new += harness.event_ms(lambda: _lib.call("b200bt_spa_bootstrap", *args(o1)), 1, warmup=1)
                    old += harness.event_ms(lambda: other.b200bt_spa_bootstrap(*args(o2)), 1, warmup=1)
                r["spa_bootstrap_shared_gather_ms"] = med(new)
                r["spa_bootstrap_parent_ms"] = med(old)
                r["spa_bootstrap_outputs_identical"] = bool(torch.equal(o1, o2))
            del z
            torch.cuda.empty_cache()
            out["mcs"][label] = r
            print(json.dumps({label: r}), flush=True)
    out["sm_clock"] = clocks.sm_clock
    print(json.dumps(out))


if __name__ == "__main__":
    main()
