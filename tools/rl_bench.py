"""Time the reinforcement-learning agents at BASELINE configs[1]'s market (10 symbols x 1M 1-minute bars, resampled to
60 minutes): populations of 1 024 and 8 192 agents with the service's hyperparameters and random seeds, hourly calls of
20 points (the first --calls calls; --full: all of them).

    python tools/rl_bench.py [--agents 1024 8192] [--calls 2000] [--full] [--reps 1]

Prints one JSON line per workload with the card, its power limit and max SM clock: the state build (analyzer + states,
CUDA events), and per population the training time with and without the history (one launch of all calls from a fresh
population; the median of --reps), replays per second, the achieved FP64 rate from the algorithmic operation count below,
its share of the H100 SXM data sheet's 34 TFLOP/s non-tensor FP64, and the reference agent's CPU time per replay (the
unmodified TradingRLAgent on its NumPy path, measured here on the host when the reference tree is present).
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
FP64_PEAK = 34e12          # H100 SXM data sheet, FP64 (non-tensor), FLOP/s


def replay_fma_pairs(batch: int, history: bool) -> int:
    """float64 multiply-add pairs of one replay: current_q + next_q (2 forward passes per sample), per sample one SGD step
    (forward, d_hidden2, d_hidden1, and the 1 083 updates, each a product of two plus alpha times it: 2 pairs), and the
    loss pass (one more forward per sample) when the history is kept."""
    fwd = 16 * 24 + 24 * 24 + 24 * 3                                  # 1 032
    sgd = fwd + 24 * 3 + 24 * 24 + 2 * (16 * 24 + 24 * 24 + 24 * 3) + 51
    return batch * (2 * fwd + sgd + (fwd if history else 0))


def reference_cpu_replay_ms(n=200):
    """The reference TradingRLAgent's replay() at batch 64 on one host core (NumPy path), ms per replay."""
    try:
        from oracle import ref_runner
        if not ref_runner.available():
            return None
        ref_runner._prepare()
        import importlib
        import logging
        import random
        import numpy as np
        rl = importlib.import_module("services.reinforcement_learning")
        logging.getLogger("reinforcement_learning").setLevel(logging.ERROR)
        feats = [f"f{i}" for i in range(16)]
        agent = rl.TradingRLAgent(feats, random_seed=1)
        rng = random.Random(2)
        for _ in range(1000):
            s = {f: rng.random() for f in feats}
            agent.remember(s, "HOLD", rng.random() - 0.5, {f: rng.random() for f in feats}, False)
        agent.replay()
        t0 = time.perf_counter()
        for _ in range(n):
            agent.replay()
        return (time.perf_counter() - t0) * 1e3 / n
    except Exception as e:                     # noqa: BLE001 -- the reference tree is optional here
        print(json.dumps({"reference_cpu": f"not measured: {e}"}), flush=True)
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--agents", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--symbols", type=int, default=10)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--full", action="store_true")
    ap.add_argument("--reps", type=int, default=1)
    a = ap.parse_args()
    import numpy as np
    import torch
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.indicators import resample
    from ai_crypto_trader_b200.rl import RLPopulation, rl_states
    from ai_crypto_trader_b200.sweep import MarketData
    torch.cuda.set_device(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    gpu = q[0] if q else "unknown"
    market = MarketData(synth.synth_ohlcv(a.symbols, a.bars))
    hourly = resample(market, 60)
    rl_states(hourly)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    states = rl_states(hourly)
    t1.record()
    torch.cuda.synchronize()
    print(json.dumps({"workload": "rl_states", "gpu": gpu, "symbols": a.symbols, "hourly_bars": hourly.N,
                      "ms": round(t0.elapsed_time(t1), 3)}), flush=True)
    ends = np.arange(19, hourly.N, dtype=np.int64)
    if not a.full:
        ends = ends[:a.calls]
    ref_ms = reference_cpu_replay_ms()
    rng = np.random.default_rng(7)
    for A in a.agents:
        agents = [dict(seed=int(s), symbol=i % a.symbols) for i, s in enumerate(rng.integers(0, 2 ** 63, A))]
        for history in (False, True):
            times, pop = [], None
            for _ in range(a.reps):
                pop = RLPopulation(states, agents)
                torch.cuda.synchronize()
                s0 = time.perf_counter()
                pop.train(ends, 20, history=history)              # ends in a device -> host copy: synchronised
                times.append(time.perf_counter() - s0)
            sec = sorted(times)[len(times) // 2]
            replays = int(pop.replays.sum())
            flops = 2 * replay_fma_pairs(64, history) * replays
            print(json.dumps({"workload": "rl_train" + ("+history" if history else ""), "gpu": gpu, "agents": A,
                              "calls": len(ends), "replays": replays, "s": round(sec, 3),
                              "replays_per_s": round(replays / sec), "fma_pairs_per_replay": replay_fma_pairs(64, history),
                              "fp64_tflops": round(flops / sec / 1e12, 3),
                              "share_of_fp64_peak": round(flops / sec / FP64_PEAK, 4),
                              "reference_cpu_ms_per_replay": None if ref_ms is None else round(ref_ms, 3)}), flush=True)


if __name__ == "__main__":
    main()
