#!/usr/bin/env python
"""CPU model of the thread-per-lane scan's event passes (lane_scan_kernel, csrc/sweep_chunked.cu) on the bench workload:
configs[1], the seed-42 random population of 1024 individuals packed into warps as the tiled plan packs them
(decode_population, costs_from_packed, pack_warps), 1M bars of one synthetic symbol, the zone-map gating of the kernel.

Every packed warp's 32 machines are stepped through the series with the kernel's arithmetic (fp32 thresholds and
screening band, the float64 exit decision inside the band).  Whole-lane trajectories: the time chunks, their warm-up and
the repair of wrong chunk starts are not modelled (they change which bars are scanned twice, not how a group is scanned).
Per 32-bar block a warp is skipped when none of its machines can fire in it (coarse zone test); inside a scanned block a
machine tests each 4-bar group against the group's range (fine test) and screens the group's bars against its CURRENT
thresholds.  A (machine, bar) that passes the screen is a candidate; the kernel runs its event body for it.  Counted per
warp and in total:

    blocks scanned           (warp, 32-bar block) pairs not skipped
    fine groups              (warp, group) pairs in which at least one machine passes the fine test
    passes, per-bar form     (warp, group, bar) with at least one candidate: one body pass per bar of the group that
                             any machine of the warp screens in (the form that steps the four bars one after another)
    passes, per-lane form    per (warp, group) the most candidates of one machine: every machine takes its own next
                             candidate in each pass (the form with one event loop per group)
    lanes per pass           candidates / passes, in both forms
    near-band                candidates decided by the float64 expression (price inside the fp32 screening band), and
                             how many of them it rejects
    events                   per machine, checked against the C oracle's n_records (oracle/sim_oracle.c)

    python tools/lane_scan_model.py [--symbol 0] [--bars 1000000] [--per-warp]

Symbol 0, 1M bars (every lane's record count equals the C oracle's):
    blocks scanned             597 630 of 1 000 000 (59.8 %)
    fine groups (>=1 lane)   1 456 192 (18.2 % of warp-groups)
    candidates (lane, bar)  10 619 109
    passes, per-bar form     2 453 368   4.33 lanes per pass
    passes, per-lane form    2 003 313   5.30 lanes per pass (0.817 x)
    near-band fp64 decisions     2 529   (0.024 % of candidates), 1 289 rejected
Firing machines rarely share a group: the per-lane form saves 18 % of the body passes, not half.  Built and measured on an
H100 80GB HBM3 (700 W limit, SM at 1980 MHz), that form (one event loop per group, a re-screen of the group after every
event) made lane_scan_kernel slower, 6.28-6.41 ms -> 7.94-8.02 ms per configs[1] step (7.03-7.11 ms with the group loop
not unrolled): the loop control and the re-screen cost more per pass than the saved passes (DESIGN.md section 8).  The
scan keeps the per-bar form; what it gained came from code size instead (LS_UNROLL_SPARSE in csrc/sweep_chunked.cu).
"""
import argparse
import sys
import time
import warnings
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np

from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.sweep import EVENTS_PER_COST_BAR, costs_from_packed, decode_population, pack_warps
from oracle import indicators_ref, sim_oracle

POP, PERIODS = 1024, list(range(5, 31))      # bench.py's population, PopulationSweep's default RSI bank
SW_MARGIN = np.float64(np.float32(1e-6))    # relative width of the fp32 screening band (csrc/sweep_dev.cuh)
f32 = np.float32


def ranges(x: np.ndarray, width: int):
    """(min, max) of every `width` values of the last axis, NaNs ignored (all-NaN: NaN, every compare false)"""
    n = x.shape[-1]
    pad = -n % width
    y = np.concatenate([x, np.full(x.shape[:-1] + (pad,), np.nan, x.dtype)], axis=-1).reshape(x.shape[:-1] + (-1, width))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return np.nanmin(y, axis=-1), np.nanmax(y, axis=-1)


def model(symbol: int, n_bars: int):
    pop = synth.random_population(POP, seed=42)
    packed = decode_population(pop, {w: i for i, w in enumerate(PERIODS)})
    pred = EVENTS_PER_COST_BAR * costs_from_packed(packed, PERIODS) * n_bars
    slots = pack_warps(pop, pred, rows=packed["rsi_row"])
    W, L = len(slots) // 32, len(slots)
    valid = slots >= 0
    ind = np.where(valid, slots, 0)
    close = synth.synth_symbol(symbol, n_bars)["close"].astype(np.float32)
    bank = indicators_ref.rsi_bank(close, PERIODS)
    rows = packed["rsi_row"][ind].astype(np.int64)
    os_f, ob_f = packed["rsi_lo"][ind].astype(f32), packed["rsi_hi"][ind].astype(f32)
    tp, sl = packed["take_profit"][ind], packed["stop_loss"][ind]
    # init_scan_const (csrc/sweep_dev.cuh)
    hiL_c, hiL_d = f32((1 + tp) * (1 - SW_MARGIN)), f32((1 + tp) * (1 + SW_MARGIN))
    loL_c, loL_d = f32((1 - sl) * (1 + SW_MARGIN)), f32((1 - sl) * (1 - SW_MARGIN))
    loS_c, loS_d = f32((1 - tp) * (1 + SW_MARGIN)), f32((1 - tp) * (1 - SW_MARGIN))
    hiS_c, hiS_d = f32((1 + sl) * (1 - SW_MARGIN)), f32((1 + sl) * (1 + SW_MARGIN))

    bank_t = np.ascontiguousarray(bank.T)                       # [N][P]
    pz, rz = ranges(close[None], 32), ranges(bank, 32)          # coarse: per 32-bar block
    pf, rf = ranges(close[None], 4), ranges(bank, 4)            # fine: per 4-bar group

    pos = np.zeros(L, np.int8)
    e_px = np.zeros(L, f32)
    rlo, rhi = os_f.copy(), ob_f.copy()
    plo, phi = np.full(L, -np.inf, f32), np.full(L, np.inf, f32)
    events = np.zeros(L, np.int64)
    c_blocks, c_groups = np.zeros(W, np.int64), np.zeros(W, np.int64)
    c_bar_passes, c_lane_passes, c_cand = np.zeros(W, np.int64), np.zeros(W, np.int64), np.zeros(W, np.int64)
    near_n = near_rej = 0
    n_blocks = -(-n_bars // 32)
    for b in range(n_blocks):
        can = valid & ((rz[0][rows, b] < rlo) | (rz[1][rows, b] > rhi) | (pz[0][0, b] <= plo) | (pz[1][0, b] >= phi))
        wscan = can.reshape(W, 32).any(axis=1)
        if not wscan.any():
            continue
        c_blocks += wscan
        lane_in = np.repeat(wscan, 32) & valid
        for g in range(8 * b, min(8 * b + 8, -(-n_bars // 4))):
            fine = lane_in & ((rf[0][rows, g] < rlo) | (rf[1][rows, g] > rhi) | (pf[0][0, g] <= plo) | (pf[1][0, g] >= phi))
            if not fine.any():
                continue
            c_groups += fine.reshape(W, 32).any(axis=1)
            cnt = np.zeros(L, np.int64)
            for t in range(4 * g, min(4 * g + 4, n_bars)):
                p, r = close[t], bank_t[t][rows]
                rsi_hit = (r < rlo) | (r > rhi)
                cand = fine & (rsi_hit | (p <= plo) | (p >= phi))
                if not cand.any():
                    continue
                cnt += cand
                c_bar_passes += cand.reshape(W, 32).any(axis=1)
                flat, lng_open = pos == 0, pos > 0
                hd = e_px * np.where(lng_open, hiL_d, hiS_d)
                ld = e_px * np.where(lng_open, loL_d, loS_d)
                near = cand & ~flat & ~rsi_hit & ~((p >= hd) | (p <= ld))
                ev = cand.copy()
                if near.any():
                    ed, pd = e_px[near].astype(np.float64), np.float64(p)
                    q = np.where(lng_open[near], (pd - ed) / ed, (ed - pd) / ed)
                    ok = (q >= tp[near]) | (q <= -sl[near])
                    ev[near] = ok
                    near_n += int(near.sum())
                    near_rej += int((~ok).sum())
                if not ev.any():
                    continue
                lng = r < os_f
                entry, exit_ = ev & flat, ev & ~flat
                pos = np.where(entry, np.where(lng, 1, -1), np.where(exit_, 0, pos)).astype(np.int8)
                rlo = np.where(entry & lng, f32(-np.inf), np.where(ev, os_f, rlo)).astype(f32)
                rhi = np.where(entry & ~lng, f32(np.inf), np.where(ev, ob_f, rhi)).astype(f32)
                phi = np.where(entry, f32(p) * np.where(lng, hiL_c, hiS_c), np.where(exit_, f32(np.inf), phi)).astype(f32)
                plo = np.where(entry, f32(p) * np.where(lng, loL_c, loS_c), np.where(exit_, f32(-np.inf), plo)).astype(f32)
                e_px = np.where(entry, f32(p), e_px).astype(f32)
                events += ev
            c_lane_passes += cnt.reshape(W, 32).max(axis=1)
            c_cand += cnt.reshape(W, 32).sum(axis=1)
    n_records = events + (pos != 0)                             # the force-close at the last bar

    # the C oracle's record counts of the same machines
    cfg = sim_oracle.config_of(synth.EPOCH_2024_MINUTES, 1)
    want = np.zeros(L, np.int64)
    for rw in np.unique(rows[valid]):
        sel = np.nonzero(valid & (rows == rw))[0]
        out = sim_oracle.lanes(close, bank[rw], [pop[int(slots[k])] for k in sel], cfg)
        want[sel] = out["n_records"]
    return dict(W=W, slots=slots, n_blocks=n_blocks, n_groups=-(-n_bars // 4), blocks=c_blocks, groups=c_groups,
                bar_passes=c_bar_passes, lane_passes=c_lane_passes, cand=c_cand, near=near_n, near_rejected=near_rej,
                n_records=n_records, want=want, valid=valid)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--symbol", type=int, default=0)
    ap.add_argument("--bars", type=int, default=1_000_000)
    ap.add_argument("--per-warp", action="store_true")
    a = ap.parse_args()
    t0 = time.time()
    m = model(a.symbol, a.bars)
    v = m["valid"]
    match = np.array_equal(m["n_records"][v], m["want"][v])
    bp, lp, cd = m["bar_passes"], m["lane_passes"], m["cand"]
    print(f"# lane_scan model: population {POP} (seed 42) in {m['W']} packed warps, symbol {a.symbol}, {a.bars} bars "
          f"({time.time() - t0:.0f} s on the CPU)")
    if a.per_warp:
        print(f"{'warp':>4} {'blocks':>7} {'groups':>8} {'per-bar':>8} {'per-lane':>8} {'cand':>9} {'lanes/pass':>14}")
        for w in range(m["W"]):
            print(f"{w:4d} {m['blocks'][w]:7d} {m['groups'][w]:8d} {bp[w]:8d} {lp[w]:8d} {cd[w]:9d} "
                  f"{cd[w] / max(bp[w], 1):6.2f} {cd[w] / max(lp[w], 1):6.2f}")
    wb = m["W"] * m["n_blocks"]
    print(f"blocks scanned           {m['blocks'].sum():>11d} of {wb} ({m['blocks'].sum() / wb * 100:.1f} %)")
    print(f"fine groups (>=1 lane)   {m['groups'].sum():>11d} ({m['groups'].sum() / (m['W'] * m['n_groups']) * 100:.2f} % of warp-groups)")
    print(f"candidates (lane, bar)   {cd.sum():>11d}")
    print(f"passes, per-bar form     {bp.sum():>11d}   lanes per pass {cd.sum() / bp.sum():.2f}")
    print(f"passes, per-lane form    {lp.sum():>11d}   lanes per pass {cd.sum() / lp.sum():.2f}   "
          f"({lp.sum() / bp.sum():.3f} x the per-bar form)")
    print(f"near-band fp64 decisions {m['near']:>11d}   ({m['near'] / cd.sum() * 100:.4f} % of candidates), rejected {m['near_rejected']}")
    print(f"events (records)         {m['n_records'][v].sum():>11d}   C oracle {m['want'][v].sum()}: "
          f"{'every lane matches' if match else 'MISMATCH in %d lanes' % int((m['n_records'][v] != m['want'][v]).sum())}")
    return 0 if match else 1


if __name__ == "__main__":
    sys.exit(main())
