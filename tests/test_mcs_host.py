"""The Model Confidence Set and the automatic block length on the CPU: the exact restatement (the device's arithmetic,
tests/mcs_ref.py) against the literal one (Hansen, Lunde and Nason's algorithm as written), the known answers, and the
host block-length rule (overfitting.block_length_rule) against Politis and White's rule step by step."""
import math

import numpy as np
import pytest

import mcs_ref
from ai_crypto_trader_b200.overfitting import block_length_rule, distinct_rows, mcs_pvalues


def _separated(seed, N=7, T=80):
    rng = np.random.default_rng(seed)
    return rng.normal(0.0, 1.0, (N, T)) + rng.permutation(N)[:, None] * 0.35


@pytest.mark.parametrize("statistic", ["R", "max"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_literal_and_exact_agree_on_separated_cases(statistic, seed):
    x = _separated(seed)
    a = mcs_ref.mcs_exact(x, 0.1, statistic, 300, 5.0, seed)
    b = mcs_ref.mcs_literal(x, 0.1, statistic, 300, 5.0, seed)
    np.testing.assert_array_equal(a["elimination_order"], b["elimination_order"])
    np.testing.assert_array_equal(a["step_pvalues"], b["step_pvalues"])
    np.testing.assert_array_equal(a["p_values"], b["p_values"])
    np.testing.assert_array_equal(a["included"], b["included"])


@pytest.mark.parametrize("statistic", ["R", "max"])
def test_one_model_ahead_by_a_constant_is_the_set(statistic):
    rng = np.random.default_rng(4)
    x = rng.normal(0.0, 1.0, (6, 120))
    x[4] += 2.0
    r = mcs_ref.mcs_exact(x, 0.1, statistic, 300, 5.0, 1)
    assert list(np.flatnonzero(r["included"])) == [4] and r["elimination_order"][-1] == 4


@pytest.mark.parametrize("statistic", ["R", "max"])
def test_identical_rows_all_stay_at_p_one(statistic):
    rng = np.random.default_rng(5)
    for x in (np.zeros((4, 50)), np.tile(rng.normal(0.0, 1.0, 50), (5, 1)), np.tile(rng.normal(1.0, 0.01, 60), (7, 1))):
        for r in (mcs_ref.mcs_exact(x, 0.1, statistic, 200, 5.0, 1), mcs_ref.mcs_literal(x, 0.1, statistic, 200, 5.0, 1)):
            assert np.all(r["p_values"] == 1.0) and r["included"].all()
            np.testing.assert_array_equal(r["elimination_order"], np.arange(len(x)))


@pytest.mark.parametrize("statistic", ["R", "max"])
@pytest.mark.parametrize("seed", range(8))
def test_copies_of_the_best_row_stand_together_in_a_mixed_set(statistic, seed):
    """Copies of a large-mean best row beside worse rows: every copy is the last survivor, at p = 1.  Without treating
    copies as one model, T_max would compare rounding residues of the set's mean and could drop some of them."""
    rng = np.random.default_rng(seed)
    best = rng.normal(1.0, 0.01, 120)
    x = np.vstack([rng.normal(0.0, 0.01, (2, 120)), np.tile(best, (4, 1)), rng.normal(0.0, 0.01, (2, 120)),
                   np.tile(best, (3, 1))])
    copies = [2, 3, 4, 5, 8, 9, 10]
    for r in (mcs_ref.mcs_exact(x, 0.1, statistic, 200, 5.0, seed), mcs_ref.mcs_literal(x, 0.1, statistic, 200, 5.0, seed)):
        assert np.all(r["p_values"][copies] == 1.0) and r["included"][copies].all()
        assert sorted(r["elimination_order"][-7:]) == copies
        assert not r["included"][[0, 1, 6, 7]].any()


@pytest.mark.parametrize("statistic", ["R", "max"])
def test_literal_and_exact_agree_with_copies_in_the_set(statistic):
    x = _separated(3, N=6)
    x = np.vstack([x, x[2], np.zeros(x.shape[1]), np.zeros(x.shape[1]), x[5]])
    a = mcs_ref.mcs_exact(x, 0.1, statistic, 300, 5.0, 3)
    b = mcs_ref.mcs_literal(x, 0.1, statistic, 300, 5.0, 3)
    for k in ("elimination_order", "step_pvalues", "p_values", "included"):
        np.testing.assert_array_equal(a[k], b[k])
    assert a["n_models"] == 7 and a["p_values"][6] == a["p_values"][2] and a["p_values"][9] == a["p_values"][5]


def test_distinct_rows_groups_byte_identical_rows():
    import torch
    x = np.random.default_rng(0).normal(0.0, 1.0, (7, 5))
    x[4] = x[1]
    x[6] = x[1]
    x[5] = 0.0
    x[3] = -0.0                                              # other bytes: another model
    reps, model_of = distinct_rows(torch.from_numpy(x))
    np.testing.assert_array_equal(reps, [0, 1, 2, 3, 5])
    np.testing.assert_array_equal(model_of, [0, 1, 2, 3, 1, 4, 1])


@pytest.mark.parametrize("statistic", ["R", "max"])
def test_pvalues_do_not_decrease_along_the_order(statistic):
    x = np.random.default_rng(6).normal(0.0, 1.0, (9, 60)) + np.linspace(0, 0.4, 9)[:, None]
    x[2] = 0.0
    r = mcs_ref.mcs_exact(x, 0.1, statistic, 200, 3.0, 2)
    p = r["p_values"][r["elimination_order"]]
    assert np.all(np.diff(p) >= 0) and p[-1] == 1.0


def test_mcs_pvalues_rule():
    p, inc = mcs_pvalues(np.array([2, 0, 3, 1]), np.array([0.3, 0.05, 0.2]), 0.25)
    np.testing.assert_array_equal(p, [0.3, 1.0, 0.3, 0.3])
    np.testing.assert_array_equal(inc, [True, True, True, True])
    rng = np.random.default_rng(1)
    for _ in range(20):                                      # the package's rule against the reference's own
        order, step_p = rng.permutation(9), rng.integers(0, 5, 8) / 4.0
        np.testing.assert_array_equal(mcs_pvalues(order, step_p, 0.3)[0], mcs_ref.pvalues(order, step_p, 0.3)[0])


def _ar1(phi, N=40, T=600, seed=0):
    rng = np.random.default_rng(seed)
    e = rng.normal(0.0, 1.0, (N, T))
    x = e.copy()
    for t in range(1, T):
        x[:, t] = phi * x[:, t - 1] + e[:, t]
    return x


def _rule(x):
    T = x.shape[1]
    K = min(math.ceil(math.sqrt(T)) + 10, T - 1)
    return block_length_rule(mcs_ref.autocov_exact(x, K), T)


def test_block_length_grows_with_the_autocorrelation():
    b = [_rule(_ar1(phi))[1] for phi in (0.0, 0.3, 0.6, 0.9)]
    assert all(u < v for u, v in zip(b, b[1:])), b
    assert b[0] < 3.0


@pytest.mark.parametrize("T", [2, 30, 695, 3000])
def test_block_length_rule_equals_the_literal_rule(T):
    x = _ar1(0.5, N=6, T=T, seed=T)
    x[1] = 0.0                                               # no estimate
    per_row, b = _rule(x)
    want = np.array([mcs_ref.block_length_literal(r) for r in x])
    assert np.isnan(per_row[1]) and np.isnan(want[1])
    np.testing.assert_allclose(per_row, want, rtol=1e-9, equal_nan=True)
    assert b == pytest.approx(float(np.median(want[np.isfinite(want)])), rel=1e-9)
    assert block_length_rule(np.zeros((3, 4)), T)[1] == 1.0
