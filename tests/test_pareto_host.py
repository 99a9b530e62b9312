"""The host restatements of b200bt_pareto_rank's contract (tests/pareto_ref.py) against each other, their properties and
known answers; objectives_from_goals; the status codes of the new entry points.  No GPU needed."""
import math

import numpy as np
import pytest

import pareto_ref as pr
from abi_header import EINVAL, ELIMIT, ENODEVICE, status

# config.json evolution.optimization_goals of the reference
REFERENCE_GOALS = {"primary": "sharpe_ratio", "secondary": ["max_drawdown", "win_rate", "profit_factor"],
                   "constraints": {"min_trades_per_day": 20, "max_trades_per_day": 50, "min_holding_period": "1m",
                                   "max_holding_period": "15m"}}


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("kind", pr.KINDS)
@pytest.mark.parametrize("M", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [1, 2, 3, 31, 33, 200])
def test_numpy_form_is_the_exact_form_bit_for_bit(kind, M, n):
    obj, mx = pr.make_input(kind, n, M)
    want = pr.pareto_exact(obj, mx)
    got = pr.pareto_numpy(obj, mx)
    for name, a, b in zip(("front", "crowding", "order", "key"), got, want):
        assert _same(a, b), (name, kind, n, M)


@pytest.mark.parametrize("kind", pr.KINDS)
def test_numpy_form_is_the_exact_form_at_2047(kind):
    obj, mx = pr.make_input(kind, 2047, 3)
    for a, b in zip(pr.pareto_numpy(obj, mx), pr.pareto_exact(obj, mx)):
        assert _same(a, b), kind


@pytest.mark.parametrize("kind", pr.KINDS)
@pytest.mark.parametrize("M", [1, 2, 4])
def test_literal_deb_sort_gives_the_same_fronts(kind, M):
    obj, mx = pr.make_input(kind, 150, M, seed=7)
    front, crowd = pr.fast_nondominated_sort_literal(obj, mx)
    want = pr.pareto_exact(obj, mx)
    assert np.array_equal(front, want[0])
    if kind in ("uniform", "anti", "chain"):      # without ties the paper's sort picks the same boundary members
        assert np.array_equal(np.isinf(crowd), np.isinf(want[1]))


def _dominates(v, p, q):
    return bool(np.all(v[p] >= v[q]) and np.any(v[p] > v[q]))


@pytest.mark.parametrize("kind", pr.KINDS)
@pytest.mark.parametrize("M", [1, 2, 3])
def test_front_properties(kind, M):
    obj, mx = pr.make_input(kind, 120, M, seed=3)
    v = pr.values(obj, mx)
    front, crowd, order, key = pr.pareto_exact(obj, mx)
    n = len(front)
    for p in range(n):
        for q in range(n):
            if front[q] >= front[p]:
                assert not _dominates(v, q, p), (p, q)           # nothing in the same or a later front dominates p
    for p in range(n):
        if front[p] > 0:
            assert any(_dominates(v, q, p) for q in np.flatnonzero(front == front[p] - 1)), p
    for p in range(n):                                           # duplicates share a front
        for q in range(p + 1, n):
            if np.array_equal(v[p], v[q]):
                assert front[p] == front[q]
    assert not np.isnan(crowd).any()
    for f in np.unique(front):                                   # each objective's extremes of a front are +inf
        F = np.flatnonzero(front == f)
        for j in range(M):
            s = sorted(F, key=lambda p: (v[p, j], p))
            assert math.isinf(crowd[s[0]]) and math.isinf(crowd[s[-1]])
    assert sorted(order.tolist()) == list(range(n))
    assert np.array_equal(key[order], -np.arange(n, dtype=np.float64) + 0.0)
    ranks = [(front[p], -crowd[p], p) for p in order]
    assert ranks == sorted(ranks)


def test_nan_rows_come_last():
    obj = np.array([[1.0, 2.0], [np.nan, np.nan], [2.0, 1.0], [0.5, 0.5], [np.nan, np.nan]])
    front, _, order, _ = pr.pareto_exact(obj, [True, True])
    assert front.tolist() == [0, 2, 0, 1, 2]
    assert order[-2:].tolist() == [1, 4]


def test_one_objective_gives_one_front_per_distinct_value():
    x = np.array([3.0, 1.0, 3.0, 2.0, -np.inf, np.nan, 1.0])
    front, _, _, _ = pr.pareto_exact(x[:, None], [True])
    assert front.tolist() == [0, 2, 0, 1, 3, 3, 2]
    front, _, _, _ = pr.pareto_exact(x[:, None], [False])
    assert front.tolist() == [3, 1, 3, 2, 0, 4, 1]       # -(-inf) = +inf is the best; -(NaN) is NaN -> -inf the worst


def test_quarter_circle_is_one_front():
    t = np.linspace(0.0, np.pi / 2, 101)
    obj = np.stack([np.cos(t), np.sin(t)], axis=1)
    front, crowd, _, _ = pr.pareto_exact(obj, [True, True])
    assert (front == 0).all()
    assert math.isinf(crowd[0]) and math.isinf(crowd[-1]) and np.isfinite(crowd[1:-1]).all()


def test_integer_grid_fronts_are_anti_diagonals():
    K = 7
    a, b = np.meshgrid(np.arange(K), np.arange(K), indexing="ij")
    obj = np.stack([a.ravel(), b.ravel()], axis=1).astype(np.float64)
    front, _, _, _ = pr.pareto_exact(obj, [True, True])
    assert np.array_equal(front, (2 * (K - 1) - obj.sum(axis=1)).astype(np.int32))
    front, _, _, _ = pr.pareto_exact(obj, [False, False])
    assert np.array_equal(front, obj.sum(axis=1).astype(np.int32))


def test_objectives_from_goals():
    from ai_crypto_trader_b200.pareto import objectives_from_goals
    from ai_crypto_trader_b200.sweep import DEFAULT_GOALS
    want = [("sharpe_ratio", True), ("max_drawdown", False), ("win_rate", True), ("profit_factor", True)]
    assert objectives_from_goals(REFERENCE_GOALS) == want
    assert objectives_from_goals(DEFAULT_GOALS) == want
    assert objectives_from_goals(["sortino_ratio", "n_losses", ("max_drawdown", "max"), "downside_deviation"]) == [
        ("sortino_ratio", True), ("n_losses", False), ("max_drawdown", True), ("downside_deviation", False)]
    assert objectives_from_goals({"primary": "net_profit", "secondary": ["net_profit", "n_negative_days"]}) == [
        ("net_profit", True), ("n_negative_days", False)]
    for bad in ({"primary": "calmar_ratio"}, {"primary": "sharpe_ratio", "secondary": ["expectancy"]},
                ["trade_hash"], [("win_rate", "up")]):
        with pytest.raises(ValueError):
            objectives_from_goals(bad)


def _rank_args(n=4, M=2, ld=None, ws_bytes=None, maximize=None, null_out=False):
    import ctypes as C
    from ai_crypto_trader_b200 import _lib
    buf = (C.c_double * 64)()
    dev = C.addressof(buf)
    mx = (C.c_int * max(1, M))(*([1] * max(1, M) if maximize is None else maximize))
    need = int(_lib.load().b200bt_pareto_workspace_bytes(n, M))
    return ("b200bt_pareto_rank", dev, M if ld is None else ld, n, M, mx, (dev + 255) & ~255,
            need if ws_bytes is None else ws_bytes, None if null_out else dev, dev, dev, None, None)


def _matrix_args(pop=4, S=2, fields=(12,), ld=None):
    import ctypes as C
    buf = (C.c_double * 64)()
    dev = C.addressof(buf)
    M = len(fields)
    return ("b200bt_objective_matrix", dev, pop, S, (C.c_int * max(1, M))(*(fields or (0,))), M, dev,
            M if ld is None else ld, None)


def test_entry_points_refuse_without_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    assert status(*_rank_args()) == ENODEVICE
    assert status(*_matrix_args()) == ENODEVICE


def test_pareto_rank_validates_arguments(native_lib):
    lib = native_lib
    assert status(*_rank_args(n=0)) == EINVAL
    assert status(*_rank_args(n=65537)) == ELIMIT
    assert status(*_rank_args(M=0)) == EINVAL
    assert status(*_rank_args(M=9)) == ELIMIT
    assert status(*_rank_args(M=3, ld=2)) == EINVAL
    assert status(*_rank_args(ws_bytes=64)) == EINVAL
    assert status(*_rank_args(null_out=True)) == EINVAL
    for n, M in ((0, 2), (65537, 2), (10, 0), (10, 9)):
        assert lib.b200bt_pareto_workspace_bytes(n, M) == 0, (n, M)
    assert lib.b200bt_pareto_workspace_bytes(65536, 8) >= 65536 * 65536 // 8
    assert lib.b200bt_pareto_workspace_bytes(1, 1) > 0


def test_objective_matrix_validates_arguments(native_lib):
    assert status(*_matrix_args(pop=0)) == EINVAL
    assert status(*_matrix_args(S=0)) == EINVAL
    assert status(*_matrix_args(fields=())) == EINVAL
    assert status(*_matrix_args(fields=tuple(range(9)))) == ELIMIT
    assert status(*_matrix_args(fields=(12, 19))) == EINVAL       # trade_hash is not a field
    assert status(*_matrix_args(fields=(-1,))) == EINVAL
    assert status(*_matrix_args(fields=(0, 1), ld=1)) == EINVAL


def test_host_wrappers_refuse_host_tensors():
    import torch
    from ai_crypto_trader_b200.pareto import objective_matrix, pareto_rank
    with pytest.raises(TypeError):
        pareto_rank(torch.zeros((4, 2), dtype=torch.float64), [True, True])
    with pytest.raises(TypeError):
        objective_matrix(torch.zeros((4, 2, 20), dtype=torch.float64), [("score", True)])
