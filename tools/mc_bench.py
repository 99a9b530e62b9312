#!/usr/bin/env python
"""Monte-Carlo throughput (BASELINE configs[2]): 1M GBM paths x 10k steps, VaR + max drawdown.

    python tools/mc_bench.py [--paths 1000000] [--steps 10000] [--store-steps 1000]
    python tools/mc_bench.py --assets [1 4 16 32]

Prints one JSON object: risk-only path-steps/s (compute-bound: Philox + Box-Muller per step),
path-store mode GB/s against the measured HBM peak (4 B per path-step written), the statistics
stage time, and the reference's NumPy GBM timed on the host on a bounded sample.
With --assets: the joint (portfolio) GBM for each asset count S, in path-asset-steps/s, next to the
single-asset kernel on the same paths and steps, with the card's name and power limit.
"""
import argparse, json, time
import numpy as np
import torch

import harness


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10_000)
    ap.add_argument("--store-steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--assets", type=int, nargs="*", default=None,
                    help="time the joint GBM for these asset counts (no value: 1 4 16 32)")
    a = ap.parse_args()
    if a.assets is not None:
        return joint(a, a.assets or [1, 4, 16, 32])
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
        job(); dist.barrier()
        ms = harness.event_ms(job, a.reps, warmup=0)
        st = job()
        dist.barrier()
        t = torch.tensor([float(np.mean(ms))], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(json.dumps({"workload": f"GBM {a.paths} paths x {a.steps} steps, risk statistics, {world} GPUs (paths sharded, strong scaling)",
                              **harness.card(), "n_gpus": world, "ms": float(t.item()), "path_steps_per_s": a.paths * a.steps / (float(t.item()) * 1e-3),
                              "var_pct": abs(st["var"]), "mdd_mean": st["mdd_mean"]}))
        dist.destroy_process_group()
        return
    eng = PathEngine()
    risk_only = lambda: eng.gbm(100.0, mu, sigma, 1 / 252, a.paths, a.steps, 2024)
    ms = float(np.mean(harness.event_ms(risk_only, a.reps)))
    f, d, _ = risk_only()
    ms_store = float(np.mean(harness.event_ms(
        lambda: eng.gbm(100.0, mu, sigma, 1 / 252, a.paths, a.store_steps, 2024, store_paths=True), 3)))
    t0 = time.perf_counter(); st = risk_statistics(eng, f, d, 100.0, 0.95); torch.cuda.synchronize(); ms_stats = (time.perf_counter() - t0) * 1e3
    peak = json.loads((harness.ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (harness.ROOT / "MEASURED_PEAKS.json").exists() else 3350.0     # H100 SXM data sheet
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
        "workload": f"GBM {a.paths} paths x {a.steps} steps, risk-only", **harness.card(),
        "risk_only": {"ms": ms, "path_steps_per_s": a.paths * a.steps / (ms * 1e-3), "bound": "fp32/fp64 ALU (Philox4x32-10 + Box-Muller + fp64 log-price)"},
        "path_store": {"steps": a.store_steps, "ms": ms_store, "GBps": store_bytes / (ms_store * 1e-3) / 1e9, "hbm_peak_GBps": peak,
                       "frac": store_bytes / (ms_store * 1e-3) / 1e9 / peak},
        "statistics_ms": ms_stats, "var_pct": abs(st["var"]), "mdd_mean": st["mdd_mean"],
        "cpu_reference_numpy": {"path_steps_per_s": n_ref * (days_ref - 1) / ref_s, "sample": f"{n_ref} paths x {days_ref - 1} steps, 1 core"},
    }))


def joint(a, assets):
    from ai_crypto_trader_b200.monte_carlo import PathEngine
    torch.cuda.set_device(0)
    eng = PathEngine()
    reps = max(1, min(a.reps, 3))

    timed = lambda fn: float(np.mean(harness.event_ms(fn, reps)))

    ms1 = timed(lambda: eng.gbm(100.0, 0.08, 0.35, 1 / 252, a.paths, a.steps, 2024))
    rows = []
    for S in assets:
        rng = np.random.default_rng(S)
        A = rng.normal(size=(S, S + 2)); c = A @ A.T; c /= np.sqrt(np.outer(np.diag(c), np.diag(c)))
        L = np.linalg.cholesky(c).astype(np.float32)
        s0, qty = rng.uniform(1, 100, S), rng.uniform(0.1, 10, S)
        mu, sigma = rng.uniform(-0.1, 0.2, S), rng.uniform(0.2, 0.8, S)
        ms = timed(lambda: eng.portfolio_gbm(s0, qty, mu, sigma, 1 / 252, L, a.paths, a.steps, 2024))
        rows.append({"assets": S, "ms": ms, "path_asset_steps_per_s": a.paths * a.steps * S / (ms * 1e-3),
                     "vs_single_asset_per_asset_step": (ms1 / ms) * S})
    print(json.dumps({
        "workload": f"joint GBM {a.paths} paths x {a.steps} steps, portfolio value + drawdown every step",
        **harness.card(), "reps": reps,
        "single_asset": {"ms": ms1, "path_steps_per_s": a.paths * a.steps / (ms1 * 1e-3)},
        "joint": rows,
    }))


if __name__ == "__main__":
    main()
