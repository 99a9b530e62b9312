"""Status codes of the model-confidence-set entry points (b200bt_boot_means, b200bt_autocov, b200bt_mcs_*): argument
checks, byte budgets included, come before the device check, so EINVAL and ELIMIT are exercised with or without a GPU;
ENODEVICE without one."""
import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status

BIG = 1 << 40


def _means(d=DEV, ld=None, N=4, T=40, q32=1 << 28, n_boot=100, out=DEV, ld_out=None, max_bytes=BIG):
    return ("b200bt_boot_means", d, T if ld is None else ld, N, T, q32, n_boot, 0, 0, None, out,
            N if ld_out is None else ld_out, max_bytes, None)


def _acov(d=DEV, ld=None, N=4, T=40, K=5, out=DEV):
    return ("b200bt_autocov", d, T if ld is None else ld, N, T, K, out, None, None)


def _pair(z=DEV, ld=None, N=4, B=100, s2=DEV, max_bytes=BIG):
    return ("b200bt_mcs_pairwise", z, N if ld is None else ld, N, B, s2, max_bytes, None)


def _stats(mean=DEV, N=4, B=100, w=DEV, t=DEV, max_bytes=BIG):
    return ("b200bt_mcs_range_stats", mean, N, B, w, t, max_bytes, None)


def _order(t=DEV, rho=DEV + 64, N=4, order=DEV, stat=DEV, rho_rank=DEV, max_bytes=BIG):
    return ("b200bt_mcs_range_order", t, rho, N, order, stat, rho_rank, max_bytes, None)


def _rboot(z=DEV, ld=None, N=4, B=100, order=DEV, rho_rank=DEV, stat=DEV, rmax=DEV, count=DEV, max_bytes=BIG):
    return ("b200bt_mcs_range_boot", z, N if ld is None else ld, N, B, order, rho_rank, stat, rmax, count, max_bytes,
            None)


def _max(z=DEV, ld=None, N=4, B=100, mean=DEV, ws=DEV, ws_bytes=1 << 20, order=DEV, stat=DEV, count=DEV,
         max_bytes=BIG):
    return ("b200bt_mcs_max", z, N if ld is None else ld, N, B, mean, ws, ws_bytes, order, stat, count, max_bytes, None)


ALL = (_means, _acov, _pair, _stats, _order, _rboot, _max)


def test_entry_points_refuse_without_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    for f in ALL:
        assert status(*f()) == ENODEVICE, f.__name__
    assert status(*_means(N=1, T=8192, q32=1 << 32)) == ENODEVICE and status(*_acov(T=2, K=1)) == ENODEVICE
    assert status(*_pair(N=16384, B=1)) == ENODEVICE and status(*_max(N=2, B=1)) == ENODEVICE


def test_null_pointers_are_refused(native_lib):
    nulls = {_means: ("d", "out"), _acov: ("d", "out"), _pair: ("z", "s2"), _stats: ("mean", "w", "t"),
             _order: ("t", "rho", "order", "stat", "rho_rank"),
             _rboot: ("z", "order", "rho_rank", "stat", "rmax", "count"),
             _max: ("z", "mean", "ws", "order", "stat", "count")}
    for f, names in nulls.items():
        for name in names:
            assert status(*f(**{name: None})) == EINVAL, (f.__name__, name)


def test_shapes_and_limits(native_lib):
    assert status(*_means(T=1)) == EINVAL and status(*_means(T=8193)) == ELIMIT
    assert status(*_means(N=0)) == EINVAL and status(*_means(N=16385)) == ELIMIT
    assert status(*_means(ld=39)) == EINVAL and status(*_means(ld_out=3)) == EINVAL
    assert status(*_means(q32=0)) == EINVAL and status(*_means(q32=(1 << 32) + 1)) == EINVAL
    assert status(*_means(n_boot=0)) == EINVAL
    assert status(*_acov(K=-1)) == EINVAL and status(*_acov(K=40)) == EINVAL and status(*_acov(T=8193, K=3)) == ELIMIT
    assert status(*_acov(ld=39)) == EINVAL and status(*_acov(N=0)) == EINVAL
    for f in (_pair, _stats, _order, _rboot, _max):
        assert status(*f(N=1)) == EINVAL, f.__name__
        assert status(*f(N=16385)) == ELIMIT, f.__name__
    for f in (_pair, _stats, _rboot, _max):
        assert status(*f(B=0)) == EINVAL, f.__name__
    for f in (_pair, _rboot, _max):
        assert status(*f(ld=3)) == EINVAL, f.__name__
    assert status(*_order(rho=DEV, rho_rank=DEV)) == EINVAL        # rho_rank may alias t, not rho
    assert status(*_max(ws_bytes=8)) == EINVAL
    assert status(*_max(ws=DEV + 8)) == EINVAL                     # not 16-byte aligned


def test_byte_budgets(native_lib):
    N, B = 4, 100
    assert status(*_means(max_bytes=B * N * 8 - 1)) == ELIMIT
    assert status(*_means(ld_out=N + 1, max_bytes=B * N * 8)) == ELIMIT
    assert status(*_pair(max_bytes=B * N * 8 + N * N * 8 - 1)) == ELIMIT
    assert status(*_stats(max_bytes=2 * N * N * 8 - 1)) == ELIMIT
    assert status(*_order(max_bytes=2 * N * N * 8 - 1)) == ELIMIT                 # rho_rank aliases t
    assert status(*_order(rho_rank=DEV + 128, max_bytes=3 * N * N * 8 - 1)) == ELIMIT
    assert status(*_rboot(max_bytes=2 * B * N * 8 + N * N * 8 - 1)) == ELIMIT
    assert status(*_max(max_bytes=B * N * 8 - 1)) == ELIMIT
    assert status(*_means(n_boot=1 << 60, max_bytes=(1 << 63) - 1)) == ELIMIT      # the product overflows int64


def test_max_workspace_bytes(native_lib):
    from ai_crypto_trader_b200 import _lib
    lib = _lib.load()
    assert lib.b200bt_mcs_max_workspace_bytes(1, 100) == 0 and lib.b200bt_mcs_max_workspace_bytes(16385, 100) == 0
    assert lib.b200bt_mcs_max_workspace_bytes(4, 0) == 0
    assert lib.b200bt_mcs_max_workspace_bytes(4, 100) >= 100 * 8 + 4 * 8 * 2 + 4 * 4 * 2
