"""What every measurement script in tools/ shares: the timers, the record of the card a number was taken on, the SM clock
sampled during the timed region, the kernels' resource table, and the configs[1] workload with its generation-3
population (the one bench.py's `evolved_population_value` times).

A time means nothing without the card it was taken on: every tool prints `card()` beside its numbers.  Importing this
module puts the repository root on sys.path, so a tool run as `python tools/<name>.py` imports the package directly."""
import contextlib
import re
import shutil
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import torch  # noqa: E402


def event_ms(fn, reps, warmup=1):
    """Milliseconds of each of `reps` calls of fn(), in call order: CUDA events on the current stream around each call
    and a synchronise after it, following `warmup` untimed calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def wall_ms(fn, reps=1, warmup=0):
    """(milliseconds of each of `reps` calls of fn() on the host clock, the last call's result); every call ends in a
    device synchronise, so the time covers its device work too.  `warmup` untimed calls go first."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out, result = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        result = fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out, result


def card(index=None):
    """{"card", "power_limit", "sm_max_mhz"} of device `index` (default: the current one) as nvidia-smi prints them
    (a read-only query).  When the query fails the name comes from torch and the other fields are "unavailable"; it
    never raises, so a measurement is never lost to it."""
    try:
        index = torch.cuda.current_device() if index is None else index
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(index)], capture_output=True, text=True, timeout=30, check=True).stdout
        name, power, sm_max = (x.strip() for x in out.strip().splitlines()[0].split(","))
        return {"card": name, "power_limit": power, "sm_max_mhz": sm_max}
    except Exception:
        try:
            name = torch.cuda.get_device_name(index)
        except Exception:
            name = "unavailable"
        return {"card": name, "power_limit": "unavailable", "sm_max_mhz": "unavailable"}


@contextlib.contextmanager
def sampled_clocks(index=None):
    """Samples the SM clock and throttle reasons (bench.ClockSampler's nvidia-smi child) while the body runs.  Yields a
    handle whose `sm_clock` holds ClockSampler.stop's dict after the block; the child is terminated and reaped on
    every exit, an exception included."""
    from bench import ClockSampler
    sampler = ClockSampler(torch.cuda.current_device() if index is None else index)
    clocks = SimpleNamespace(sm_clock=None)
    t0 = time.time()
    try:
        sampler.start()
        time.sleep(0.3)                     # the sampler's first rows arrive before the timed region starts
        t0 = time.time()
        yield clocks
    finally:
        try:
            clocks.sm_clock = sampler.stop(t0, time.time())
        finally:
            if sampler.proc is not None:
                sampler.proc.terminate()
                sampler.proc.wait()


def kernel_resources(names):
    """{name: {"registers", "local_bytes", "shared_bytes"}} per thread of the first kernel of the library whose mangled
    name contains `name`, from `cuobjdump -res-usage`; None when cuobjdump is absent."""
    from ai_crypto_trader_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        text = subprocess.run([tool, "-res-usage", str(_lib.LIB_PATH)], capture_output=True, text=True,
                              timeout=120).stdout
    except OSError:
        return None
    out, fn = {}, None
    for line in text.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        reg = re.search(r"REG:(\d+)", line)
        if fn is None or reg is None:
            continue
        loc, sh = re.search(r"LOCAL:(\d+)", line), re.search(r"SHARED:(\d+)", line)
        for name in names:
            if name in fn and name not in out:
                out[name] = {"registers": int(reg.group(1)), "local_bytes": int(loc.group(1)) if loc else None,
                             "shared_bytes": int(sh.group(1)) if sh else None}
        fn = None
    return out


def configs1(symbols=10, bars=1_000_000, pop=1024):
    """(MarketData, population) of BASELINE configs[1]: the synthetic market of `symbols` x `bars` 1-minute bars and
    the random seed-42 population bench.py times."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.sweep import MarketData
    return MarketData(synth.synth_ohlcv(symbols, bars)), synth.random_population(pop, seed=42)


def generation3(fitness, population):
    """Generation 3 of the reference GA (seed 42) started from `population`: bench.py's `evolved_population_value`
    population, which writes several times more trade records than the random one."""
    from ai_crypto_trader_b200 import synth
    from ai_crypto_trader_b200.genetic_algorithm import GeneticAlgorithm
    ga = GeneticAlgorithm(synth.param_ranges(), fitness, population_size=len(population), generations=3, random_seed=42)
    ga.run(seeded_individuals=population)
    return ga.population
