"""The GA operators' restatement (tests/ga_ref.py) on its own, and the refusals of b200bt_ga_init /
b200bt_ga_next_generation: argument checks run before the device check, so these statuses hold with or without a GPU."""
import ctypes as C
import math

import numpy as np
import pytest

import ga_ref
from oracle import mc_ref
from abi_header import EINVAL, ELIMIT, ENODEVICE, status


# -- fma ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("a, b, c, fused, twice", [
    (0.1, 10.0, -1.0, 5.551115123125783e-17, 0.0),
    (1.0 + 2.0 ** -30, 1.0 - 2.0 ** -30, -1.0, -(2.0 ** -60), 0.0),       # (1 + e)(1 - e) - 1 = -e^2 exactly
    (1.5e308, 2.0, -1.5e308, 1.5e308, math.inf),                           # the product alone overflows
    (3.0, 0.5, 0.25, 1.75, 1.75),                                          # exact either way
    (0.0, 5.0, -0.0, 0.0, 0.0),
    (-0.0, 5.0, -0.0, -0.0, -0.0),
    (2.0, -3.0, 6.0, 0.0, 0.0),                                            # exact cancellation is +0
])
def test_fma_known_answers(a, b, c, fused, twice):
    got = ga_ref.fma(a, b, c)
    assert np.float64(got).view(np.uint64) == np.float64(fused).view(np.uint64), (got, fused)
    assert np.float64(a * b + c).view(np.uint64) == np.float64(twice).view(np.uint64)


def test_fma_is_correctly_rounded_on_random_operands():
    """Against an independent exact evaluation: the integer significands scaled to a common exponent."""
    rng = np.random.default_rng(3)
    a, b, c = rng.uniform(-4, 4, 2000), rng.uniform(-4, 4, 2000), rng.uniform(-4, 4, 2000)
    differs = 0
    for x, y, z in zip(a.tolist(), b.tolist(), c.tolist()):
        (mx, ex), (my, ey), (mz, ez) = (x.as_integer_ratio(), y.as_integer_ratio(), z.as_integer_ratio())
        num = mx * my * ez + mz * ex * ey
        den = ex * ey * ez
        want = num / den                                    # int / int true division is correctly rounded
        got = ga_ref.fma(x, y, z)
        assert got == want, (x, y, z)
        differs += got != x * y + z
    assert differs > 100                                    # the operands exercise the single rounding


# -- word stream -------------------------------------------------------------------------------------------------------

def _block(seed, generation, slot, stream, blk):
    return [int(w[0]) for w in mc_ref.philox4x32_10(np.array([slot], np.uint32), np.uint32(generation), np.uint32(stream),
                                                     np.array([blk], np.uint32), seed & 0xFFFFFFFF, seed >> 32)]


def test_word_stream_order_and_continuation():
    seed, generation, slot, stream = 0x0123456789ABCDEF, 0xFFFFFFFF, 77, ga_ref.MUTATION
    b0, b1, b2 = (_block(seed, generation, slot, stream, k) for k in range(3))
    w = ga_ref.Words(seed, generation, [slot], stream)
    got = [int(w.next()[0]) for _ in range(8)]
    assert got == b0[::-1] + b1[::-1]                     # x[3], x[2], x[1], x[0], then the next block
    # a uniform after an odd number of words takes its high word from one block and its low word from the next
    st = ga_ref.Stats()
    w = ga_ref.Words(seed, generation, [slot], stream, st)
    first = [int(w.next()[0]) for _ in range(3)]
    assert first == b0[:0:-1]
    u = float(w.uniform()[0])
    assert st.straddles == 1
    assert u == ((b0[0] >> 5) * 67108864.0 + (b1[3] >> 6)) / 9007199254740992.0
    u2 = float(w.uniform()[0])
    assert st.straddles == 1 and u2 == ((b1[2] >> 5) * 67108864.0 + (b1[1] >> 6)) / 9007199254740992.0
    assert int(w.next()[0]) == b1[0] and int(w.next()[0]) == b2[3]
    # below(n) = (word * n) >> 32
    w = ga_ref.Words(seed, generation, [slot], stream)
    assert int(w.below(1000)[0]) == (b0[3] * 1000) >> 32 and int(w.below(2 ** 32 - 1)[0]) == (b0[2] * (2 ** 32 - 1)) >> 32


def test_word_streams_move_only_in_active_lanes():
    seed = 99
    w = ga_ref.Words(seed, 5, [0, 1, 2], ga_ref.SELECT)
    mask = np.array([True, False, True])
    a = w.next(mask)
    assert a[1] == 0
    b = w.next()
    for lane, want in ((0, _block(seed, 5, 0, 0, 0)[2]), (1, _block(seed, 5, 1, 0, 0)[3]), (2, _block(seed, 5, 2, 0, 0)[2])):
        assert int(b[lane]) == want
    # keys and counters: the seed's high word is the second key word, the generation the second counter word
    assert _block(1 << 32, 0, 0, 0, 0) != _block(1, 0, 0, 0, 0)
    assert int(ga_ref.Words(1 << 32, 0, [0], 0).next()[0]) == _block(1 << 32, 0, 0, 0, 0)[3]


# -- invariants on large random inputs ---------------------------------------------------------------------------------

def _genes():
    from ai_crypto_trader_b200 import synth
    r = synth.param_ranges()
    lo = [float(v[0]) for v in r.values()] + [0.0, -2.0e9, 3.0, -7.5, -1.0, 2.5, -1e-3]
    hi = [float(v[1]) for v in r.values()] + [9.0, 1.999999999e9, 3.0, -0.5, 2.0, 2.5, 1e6]
    is_int = [isinstance(v[0], int) and isinstance(v[1], int) for v in r.values()] + [True, True, True, False, False,
                                                                                       False, False]
    return np.array(lo), np.array(hi), np.array(is_int)


@pytest.mark.parametrize("pop, elitism, tournament", [(6000, 0.1, 3), (3001, 0.29, 8), (50, 0.0, 1), (8, 0.9, 8)])
def test_restatement_invariants(pop, elitism, tournament):
    lo, hi, is_int = _genes()
    seed, generation = 0xDEADBEEF00000001, 12
    st = ga_ref.Stats()
    params = ga_ref.init(np.zeros((pop, len(lo))), 0, lo, hi, is_int, seed, st)
    assert (params >= lo).all() and (params <= hi).all()
    assert np.array_equal(params[:, is_int], np.round(params[:, is_int]))
    fitness = np.round(np.random.default_rng(pop).standard_normal(pop), 1)        # many ties
    fitness[::17] = -np.inf
    key, ranked = ga_ref.rank(fitness)
    n_elite = ga_ref.elite_count(elitism, pop)
    sel, out = ga_ref.next_generation(params, key, ranked, lo, hi, is_int, elitism, tournament, 0.8, 0.3, seed,
                                      generation, st)
    assert np.array_equal(sel[:n_elite], ranked[:n_elite])
    assert np.array_equal(out[:n_elite], params[ranked[:n_elite]])
    assert (out >= lo).all() and (out <= hi).all()
    assert np.array_equal(out[:, is_int], np.round(out[:, is_int]))
    picks, winners = ga_ref.tournaments(key, pop, n_elite, tournament, seed, generation)
    assert np.array_equal(winners, sel[n_elite:])
    assert all(len(set(row)) == tournament for row in picks.tolist())            # distinct contenders
    fits = key[picks]
    assert np.array_equal(winners, picks[np.arange(len(picks)), np.argmax(fits, axis=1)])   # first maximum wins
    assert st.mutated > 0 and st.straddles > 0


def test_restatement_is_deterministic_and_keyed():
    lo, hi, is_int = _genes()
    params = ga_ref.init(np.zeros((300, len(lo))), 0, lo, hi, is_int, 5)
    key, ranked = ga_ref.rank(np.arange(300.0))
    a = ga_ref.next_generation(params, key, ranked, lo, hi, is_int, 0.1, 3, 0.8, 0.2, 5, 1)
    b = ga_ref.next_generation(params, key, ranked, lo, hi, is_int, 0.1, 3, 0.8, 0.2, 5, 1)
    c = ga_ref.next_generation(params, key, ranked, lo, hi, is_int, 0.1, 3, 0.8, 0.2, 5, 2)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert not np.array_equal(a[1], c[1])


def test_rank_puts_nan_last_and_keeps_ties_in_index_order():
    key, ranked = ga_ref.rank([1.0, float("nan"), 3.0, 1.0, -math.inf, 3.0])
    assert ranked.tolist() == [2, 5, 0, 3, 1, 4]
    assert key[1] == -math.inf


# -- refusals ----------------------------------------------------------------------------------------------------------

_DEV = 1 << 20             # non-null, never dereferenced: every call below is refused before the device is touched


def _init(pop=8, genes=2, n_seeded=0, lo=(0.0, 1.0), hi=(1.0, 5.0), is_int=(0, 1)):
    G = max(genes, len(lo))
    return ("b200bt_ga_init", _DEV, pop, genes, n_seeded, (C.c_double * G)(*lo), (C.c_double * G)(*hi),
            (C.c_int * G)(*is_int), 1, None)


def _next(pop=8, genes=2, lo=(0.0, 1.0), hi=(1.0, 5.0), is_int=(0, 1), elitism=0.1, tournament=3, out=_DEV + 4096):
    G = max(genes, len(lo))
    return ("b200bt_ga_next_generation", _DEV, _DEV + 1024, _DEV + 2048, pop, genes, (C.c_double * G)(*lo),
            (C.c_double * G)(*hi), (C.c_int * G)(*is_int), elitism, tournament, 0.8, 0.2, 1, 1, _DEV + 3072, out, None)


def _wide(n, lo, hi, is_int):
    return dict(lo=(lo,) * n, hi=(hi,) * n, is_int=(is_int,) * n)


@pytest.mark.parametrize("entry", [_init, _next])
def test_ga_entry_points_validate_ranges(native_lib, entry):
    assert status(*entry(genes=0)) == EINVAL
    assert status(*entry(genes=65, **_wide(65, 0.0, 1.0, 0))) == EINVAL
    assert status(*entry(lo=(0.0, 2.0), hi=(1.0, 1.0))) == EINVAL                       # hi < lo
    assert status(*entry(lo=(0.0, 0.0), hi=(1.0, 4.0e9), is_int=(0, 1))) == ELIMIT        # integer span >= 4e9
    assert status(*entry(lo=(0.0, -2.0e9), hi=(1.0, 2.0e9), is_int=(0, 1))) == ELIMIT


def test_ga_init_validates_arguments(native_lib):
    assert status(*_init(n_seeded=9)) == EINVAL                  # more seeded rows than the population
    assert status(*_init(n_seeded=-1)) == EINVAL
    assert status(*_init(pop=0)) == EINVAL


@pytest.mark.parametrize("tournament", [0, 9, 5])
def test_ga_next_generation_validates_tournament(native_lib, tournament):
    assert status(*_next(pop=4, tournament=tournament)) == EINVAL


@pytest.mark.parametrize("elitism", [math.nan, math.inf, -math.inf])
def test_ga_next_generation_refuses_a_non_finite_elitism(native_lib, elitism):
    assert status(*_next(elitism=elitism)) == EINVAL


def test_ga_next_generation_refuses_aliased_or_null_buffers(native_lib):
    assert status(*_next(out=_DEV)) == EINVAL                    # params == params_out
    assert status(*_next(out=None)) == EINVAL


def test_ga_entry_points_refuse_without_device(native_lib):
    """Arguments that pass validation -- an elitism_pct far above 1 and a float gene wider than the integer limit among
    them -- reach the device check.  Only without a GPU: with one, these calls would launch on the dummy pointers."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    assert status(*_init()) == ENODEVICE
    assert status(*_init(n_seeded=8)) == ENODEVICE
    assert status(*_init(lo=(0.0, 0.0), hi=(1.0, 4.0e9), is_int=(0, 0))) == ENODEVICE
    assert status(*_next(lo=(0.0, 0.0), hi=(1.0, 4.0e9), is_int=(0, 0))) == ENODEVICE
    for elitism in (0.1, 0.0, -5.0, 1.0, 1e300):
        assert status(*_next(elitism=elitism)) == ENODEVICE
    assert status(*_next(pop=8, tournament=8)) == ENODEVICE
