#!/usr/bin/env python
"""CPU model behind the sparse drawdown pass of the time-chunked sweeps (DESIGN.md section 3.1): how many time chunks of a
lane set a NEW EQUITY PEAK?

The equity and the running peak at the start of a chunk are needed for one metric, the max drawdown.  A chunk in which the
equity never exceeds the peak it inherits has max drawdown (P0 - E0 - min prefix) / P0, which chunk_prefix_kernel forms from
three per-chunk scalars; only the chunks that set a new peak take the record-by-record pass (chunk_peak_kernel).  This
script counts them on the bench workload (configs[1]: population 1024, symbol 0, 1M bars, K = 28 chunks) for the random
seed-42 population and for the generation-3 population of the GA run bench.py times (`evolved`: the GA is run on the C
oracle over all 10 symbols, ~40 s on 8 cores).  The GPU's count is PopulationSweep.last_peak_chunks
(tools/sweep_kernels.py prints it).

    python tools/peak_chunks_model.py [random|evolved]

Measured: random 4.9 % of the chunks (1.9 % of the records); generation 3: 0.44 % of the chunks (0.15 % of the records).
"""
import sys, time
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np
from ai_crypto_trader_b200 import synth
from ai_crypto_trader_b200.genetic_algorithm import GeneticAlgorithm
from oracle import indicators_ref, parallel

N, S, POP, K = 1_000_000, 10, 1024, 28
def fitness_batch(pop):
    st = parallel.population_stats(pop, list(range(S)), N, minute0=synth.EPOCH_2024_MINUTES, workers=None)
    sc = st["score"].astype(np.float64)
    return [float(x) for x in sc.mean(axis=1)]

def evolved_population():
    pop = synth.random_population(POP, seed=42)
    f = lambda ind: 0.0
    f.batch = fitness_batch
    ga = GeneticAlgorithm(synth.param_ranges(), f, population_size=POP, generations=3, random_seed=42)
    t0 = time.time(); ga.run(seeded_individuals=pop); print('GA 3 generations on the C oracle', time.time() - t0, 's', flush=True)
    return ga.population

def analyse(pop, tag):
    close = synth.synth_symbol(0, N)["close"].astype(np.float64)
    bank = indicators_ref.rsi_bank(close.astype(np.float32), list(range(5, 31))).astype(np.float64)
    g = lambda k: np.array([float(p[k]) for p in pop])
    os_, ob, tp, sl = g('rsi_oversold'), g('rsi_overbought'), g('take_profit') / 100, g('stop_loss') / 100
    row = np.array([int(p['rsi_period']) - 5 for p in pop]); L = len(pop)
    side = np.zeros(L, np.int8); entry = np.ones(L)
    eq = np.zeros(L); peak = np.zeros(L)
    bounds = [((N * c) // K) & ~511 for c in range(K)] + [N]
    newpeak = np.zeros((L, K), bool); nrec = np.zeros((L, K), np.int64)
    bankT = np.ascontiguousarray(bank.T); c = 0
    for t in range(N):
        while t >= bounds[c + 1]: c += 1
        r = bankT[t][row]; p = close[t]
        flat = side == 0
        lng = r < os_; sht = (r > ob) & ~lng
        gain = np.where(side > 0, p - entry, entry - p) / entry
        rev = np.where(side > 0, r > ob, r < os_)
        ex = (~flat) & ((gain >= tp) | (gain <= -sl) | rev)
        en = flat & (lng | sht)
        if ex.any() or en.any():
            pnl = np.where(ex, 500.0 * gain - 1.0, np.where(en, -0.5, 0.0))
            ev = ex | en
            eq = eq + pnl
            np_ = ev & (eq > peak)
            peak = np.where(np_, eq, peak)
            newpeak[:, c] |= np_
            nrec[:, c] += ev
            side = np.where(en, np.where(lng, 1, -1), np.where(ex, 0, side)).astype(np.int8)
            entry = np.where(en, p, entry)
    has = nrec > 0
    print(f"{tag}: records {nrec.sum()} (x10 symbols ~ {nrec.sum()*10:.3g}); chunks with records {has.mean()*100:.1f} %; "
          f"chunks (with records) that set a new equity peak: {(newpeak & has).sum() / has.sum() * 100:.2f} %; "
          f"records living in such chunks: {nrec[newpeak].sum() / nrec.sum() * 100:.2f} %; lanes that end above their start: {(eq > 0).mean()*100:.1f} %", flush=True)

if __name__ == '__main__':
    which = sys.argv[1] if len(sys.argv) > 1 else 'random'
    if which == 'random':
        analyse(synth.random_population(POP, seed=42), 'random population (seed 42)')
    else:
        pop = evolved_population()
        analyse(pop, 'generation-3 population')
