#!/usr/bin/env python
"""Monte-Carlo throughput (BASELINE configs[2]): 1M GBM paths x 10k steps, VaR + max drawdown.

    python tools/mc_bench.py [--paths 1000000] [--steps 10000] [--store-steps 1000]

Prints one JSON object: risk-only path-steps/s (compute-bound: Philox + Box-Muller per step),
path-store mode GB/s against the measured HBM peak (4 B per path-step written), the statistics
stage time, and the reference's NumPy GBM timed on the host on a bounded sample.
"""
import argparse, json, sys, time
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import numpy as np
import torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10_000)
    ap.add_argument("--store-steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from ai_crypto_trader_b200.monte_carlo import PathEngine, risk_statistics
    import os
    world, rank = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    mu, sigma = 0.08, 0.35            # annualised drift / volatility; horizon = steps/252 years at dt = 1/252
    if world > 1:
        # BASELINE configs[2] on several GPUs (torchrun): paths sharded by rank, one gather of finals + drawdowns, the
        # statistics on every rank; STRONG scaling (the 1M paths are fixed), device time = max over ranks
        import torch.distributed as dist
        from ai_crypto_trader_b200.dist import gather_paths, shard_bounds
        dist.init_process_group("nccl")
        eng = PathEngine()
        lo, hi, _ = shard_bounds(a.paths, world, rank)
        def job():
            f, d, _ = eng.gbm(100.0, mu, sigma, 1 / 252, hi - lo, a.steps, 2024, path_offset=lo)
            f, d = gather_paths(f, d, a.paths)
            return risk_statistics(eng, f, d, 100.0, 0.95)
        job(); dist.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps): st = job()
        e1.record(); dist.barrier(); torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / a.reps], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(json.dumps({"workload": f"GBM {a.paths} paths x {a.steps} steps, risk statistics, {world} GPUs (paths sharded, strong scaling)",
                              "n_gpus": world, "ms": float(t.item()), "path_steps_per_s": a.paths * a.steps / (float(t.item()) * 1e-3),
                              "var_pct": abs(st["var"]), "mdd_mean": st["mdd_mean"]}))
        dist.destroy_process_group()
        return
    eng = PathEngine()
    def timed(fn, reps):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): out = fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps, out
    ms, (f, d, _) = timed(lambda: eng.gbm(100.0, mu, sigma, 1 / 252, a.paths, a.steps, 2024), a.reps)
    ms_store, _ = timed(lambda: eng.gbm(100.0, mu, sigma, 1 / 252, a.paths, a.store_steps, 2024, store_paths=True), 3)
    t0 = time.perf_counter(); st = risk_statistics(eng, f, d, 100.0, 0.95); torch.cuda.synchronize(); ms_stats = (time.perf_counter() - t0) * 1e3
    peak = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 3350.0     # H100 SXM data sheet
    # reference generator (NumPy, monte_carlo_service.py:266-273) on a bounded sample
    n_ref, days_ref = 100_000, 101
    t0 = time.perf_counter()
    paths = np.zeros((days_ref, n_ref)); paths[0] = 100.0
    for t in range(1, days_ref):
        Z = np.random.standard_normal(n_ref)
        paths[t] = paths[t - 1] * np.exp((mu - 0.5 * sigma ** 2) / 252 + sigma * np.sqrt(1 / 252) * Z)
    ref_s = time.perf_counter() - t0
    store_bytes = a.paths * (a.store_steps + 1) * 4
    print(json.dumps({
        "workload": f"GBM {a.paths} paths x {a.steps} steps, risk-only",
        "risk_only": {"ms": ms, "path_steps_per_s": a.paths * a.steps / (ms * 1e-3), "bound": "fp32/fp64 ALU (Philox4x32-10 + Box-Muller + fp64 log-price)"},
        "path_store": {"steps": a.store_steps, "ms": ms_store, "GBps": store_bytes / (ms_store * 1e-3) / 1e9, "hbm_peak_GBps": peak,
                       "frac": store_bytes / (ms_store * 1e-3) / 1e9 / peak},
        "statistics_ms": ms_stats, "var_pct": abs(st["var"]), "mdd_mean": st["mdd_mean"],
        "cpu_reference_numpy": {"path_steps_per_s": n_ref * (days_ref - 1) / ref_s, "sample": f"{n_ref} paths x {days_ref - 1} steps, 1 core"},
    }))


if __name__ == "__main__":
    main()
