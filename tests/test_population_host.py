"""CPU checks of the population plumbing the sweeps share: the dedup of decoded records against sorting the rows, on the
record widths of the RSI, grid and DCA sweeps, and the calendar of a series' days."""
import ctypes as C

import numpy as np
import pytest

from ai_crypto_trader_b200 import _lib, population
from ai_crypto_trader_b200.population import calendar_days, unique_rows

GRID = C.sizeof(_lib.GridIndividual)
DCA = C.sizeof(_lib.DcaIndividual)
WIDTHS = {"rsi": 40, "grid S=1": GRID + 16, "grid S=10": GRID + 16 * 10, "dca S=3": DCA + 80 * 3,
          "dca S=33": DCA + 80 * 33}


def sorted_keep_rank(rows):
    """The first-occurrence keep and rank of np.unique(axis=0), as the sweeps computed them before unique_rows."""
    _, first, inverse = np.unique(rows, axis=0, return_index=True, return_inverse=True)
    keep = np.sort(first)
    if len(keep) == len(rows):
        return keep, None
    rank = np.empty(len(first), dtype=np.int64)
    rank[np.argsort(first)] = np.arange(len(first))
    return keep, rank[inverse.reshape(-1)]


def populations(width, rng):
    """Random byte rows of one width: with duplicates, all distinct, one row, all alike, and twins differing in one byte."""
    distinct = rng.integers(0, 256, size=(300, width), dtype=np.uint8)
    yield "duplicates", distinct[rng.integers(0, 60, size=300)]
    yield "distinct", distinct
    yield "one row", distinct[:1]
    yield "all alike", np.repeat(distinct[:1], 7, axis=0)
    twins = np.repeat(distinct[:4], 3, axis=0)
    twins[1::3, -1] ^= 1
    yield "one byte apart", twins


@pytest.mark.parametrize("exact", [False, True], ids=["hashed", "every row collides"])
@pytest.mark.parametrize("name", list(WIDTHS))
def test_unique_rows_matches_sorting(name, exact, monkeypatch):
    if exact:
        monkeypatch.setattr(population, "_HASH_MULTIPLIERS", np.zeros(5, dtype=np.uint64))
    rng = np.random.default_rng(WIDTHS[name])
    for case, rows in populations(WIDTHS[name], rng):
        keep, expand = unique_rows(np.ascontiguousarray(rows))
        want_keep, want_expand = sorted_keep_rank(rows)
        assert np.array_equal(keep, want_keep), case
        if want_expand is None:
            assert expand is None, case
        else:
            assert np.array_equal(expand, want_expand), case
            assert np.array_equal(rows[keep][expand], rows), case


def test_unique_rows_compares_bytes():
    """Records with NaN fields are equal when their bytes are (identical bytes are identical kernel input)."""
    rows = np.array([[1.0, np.nan], [2.0, 3.0], [1.0, np.nan], [-0.0, 3.0], [0.0, 3.0]])
    keep, expand = unique_rows(rows)
    assert keep.tolist() == [0, 1, 3, 4] and expand.tolist() == [0, 1, 0, 2, 3]


def test_calendar_days_matches_the_sweeps_formulas():
    rng = np.random.default_rng(3)
    for _ in range(2000):
        minute0 = int(rng.integers(0, 60_000_000))
        bar_minutes = int(rng.choice([1, 3, 5, 15, 60, 240, 1440]))
        N = int(rng.integers(1, 5000))
        first = minute0 // 1440
        # the grid and DCA sweeps: no gap
        assert calendar_days(minute0, bar_minutes, N) == (first, (minute0 + (N - 1) * bar_minutes) // 1440 - first + 1)
        # the RSI sweep on a glued series: gap_minutes skipped before bar gap_bar
        gap_bar, gap_minutes = int(rng.integers(0, N + 2)), int(rng.integers(0, 50_000))
        last = N - 1
        gap = gap_minutes if (gap_bar > 0 and last >= gap_bar) else 0
        assert calendar_days(minute0, bar_minutes, N, gap_bar, gap_minutes) == \
            (first, (minute0 + last * bar_minutes + gap) // 1440 - first + 1)
