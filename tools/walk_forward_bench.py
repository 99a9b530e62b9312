"""Walk-forward timing on the configs[1] market (10 symbols x 1 000 000 one-minute bars, ~694 days): rolling 30-day
in-sample / 7-day out-of-sample windows, GA generations at a given population.

Rows (one JSON line each, with the card beside every number):
  lockstep_generation   wall time of one generation of the lockstep GA over all windows (WalkForward.evolve: decode,
                        b200bt_sweep_segments, fitness reduce, one fitness read-back, W operator calls), averaged over a
                        run that follows one untimed run
  segments_kernel       CUDA-event time of one generation's b200bt_sweep_segments call alone, and its lane-bars/s
  per_window_loop       the same generation's lanes as W calls of b200bt_sweep on the windows' slices, timed alternately with
                        the segments call in the same run
  final_scoring         wall time of the scoring call (stitched out-of-sample schedule + every window's two lanes) and its
                        kernel time

    python tools/walk_forward_bench.py [--pop 20 1024] [--generations 10] [--reps 5]
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
    ap.add_argument("--pop", type=int, nargs="+", default=[20, 1024])
    ap.add_argument("--generations", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bars", type=int, default=1_000_000)
    args = ap.parse_args()

    from ai_crypto_trader_b200 import _lib, synth
    from ai_crypto_trader_b200.sweep import PopulationSweep
    from ai_crypto_trader_b200.walk_forward import (WalkForward, ga_schedules, plan_windows, scoring_schedules,
                                                    window_seed)
    torch.cuda.set_device(0)
    card = harness.card()
    market, _ = harness.configs1(bars=args.bars)
    sweep = PopulationSweep(market, mode="fused")
    windows = plan_windows(market.minute0, market.bar_minutes, market.N, 30, 7)
    ranges = [(a, b) for a, b, _, _ in windows]
    W, S = len(windows), market.S
    current = {"rsi_period": 14, "rsi_oversold": 30, "rsi_overbought": 70, "take_profit": 3, "stop_loss": 2}

    def emit(row):
        print(json.dumps(dict(row, windows=W, symbols=S, bars=market.N, **card)), flush=True)

    for pop in args.pop:
        wf = WalkForward(sweep, synth.param_ranges(), population_size=pop, generations=args.generations, random_seed=42)
        seeds = [window_seed(42, w) for w in range(W)]
        with harness.sampled_clocks() as clk:      # one untimed run first: first-call set-up is not in the time
            ms, (winners, _, _, params) = harness.wall_ms(lambda: wf.evolve(ranges, seeds, current), reps=1, warmup=1)
        emit({"row": "lockstep_generation", "pop": pop, "generations": args.generations,
              "ms_per_generation": ms[0] / (args.generations + 1), "ms_total": ms[0], "sm_clock": clk.sm_clock})

        # one generation's lanes (the final population), as one segments call and as a per-window loop of b200bt_sweep
        indiv = torch.empty(W * pop * C.sizeof(_lib.Individual), dtype=torch.uint8, device=market.device)
        wf.decode(params, indiv)
        segments, seg_begin = wf._tables(ga_schedules(ranges, pop))
        stats = torch.empty((W * pop, S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=market.device)
        run_segments = lambda: wf.sweep_segments(indiv, W * pop, segments, seg_begin, stats)
        cfgs = [_lib.SweepConfig(initial_capital=sweep.cfg.initial_capital, minute0=market.minute0 + a * market.bar_minutes,
                                 bar_minutes=market.bar_minutes, primary=sweep.cfg.primary,
                                 secondary_mask=sweep.cfg.secondary_mask, variant=0) for a, _ in ranges]
        rec = C.sizeof(_lib.Individual)

        def run_loop():
            st = _lib.current_stream()
            for w, (a, b) in enumerate(ranges):
                _lib.call("b200bt_sweep", market.close.data_ptr() + 4 * a, _lib.ld(market.close),
                          sweep.bank.data_ptr() + 4 * a, _lib.ld(sweep.bank), sweep.bank.shape[1], S, b - a,
                          indiv.data_ptr() + w * pop * rec, None, pop, C.byref(cfgs[w]),
                          stats.data_ptr() + w * pop * S * _lib.LANE_STATS_WORDS * 8, None, 0, st)

        seg_ms, loop_ms = [], []
        with harness.sampled_clocks() as clk:
            for _ in range(args.reps):
                seg_ms += harness.event_ms(run_segments, 1, warmup=0)
                loop_ms += harness.event_ms(run_loop, 1, warmup=0)
        lane_bars = pop * S * sum(b - a for a, b in ranges)
        seg_med, loop_med = statistics.median(seg_ms), statistics.median(loop_ms)
        emit({"row": "segments_kernel", "pop": pop, "ms_median": seg_med, "ms": seg_ms, "lane_bars": lane_bars,
              "lane_bars_per_s": lane_bars / (seg_med * 1e-3), "sm_clock": clk.sm_clock})
        emit({"row": "per_window_loop", "pop": pop, "ms_median": loop_med, "ms": loop_ms,
              "lane_bars_per_s": lane_bars / (loop_med * 1e-3), "segments_speedup": loop_med / seg_med,
              "sm_clock": clk.sm_clock})

        # the final scoring call: wall time of WalkForward.score (decode, tables, launch, read-back) and its kernel alone
        sched = scoring_schedules(windows)
        from ai_crypto_trader_b200.sweep import decode_population
        packed = decode_population(winners, sweep.period_row)
        sind = torch.from_numpy(packed.view(np.uint8).copy()).to(market.device)
        sseg, sbeg = wf._tables(sched)
        sst = torch.empty((len(sched), S, _lib.LANE_STATS_WORDS), dtype=torch.float64, device=market.device)
        with harness.sampled_clocks() as clk:
            score_ms, _ = harness.wall_ms(lambda: wf.score(sched, winners), reps=args.reps, warmup=1)
            kern_ms = harness.event_ms(lambda: wf.sweep_segments(sind, W, sseg, sbeg, sst), args.reps)
        emit({"row": "final_scoring", "pop": pop, "ms_wall_median": statistics.median(score_ms),
              "ms_kernel_median": statistics.median(kern_ms), "schedules": len(sched), "sm_clock": clk.sm_clock})


if __name__ == "__main__":
    main()
