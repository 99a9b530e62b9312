"""Status codes of the data-snooping entry points (b200bt_spa_moments, b200bt_spa_bootstrap): argument checks come before
the device check, so EINVAL and ELIMIT are exercised with or without a GPU; ENODEVICE without one."""
import pytest

from abi_header import DEV, EINVAL, ELIMIT, ENODEVICE, status


def _moments(d=DEV, ld=None, N=4, T=40, q=0.1, mean=DEV, omega2=DEV):
    return ("b200bt_spa_moments", d, T if ld is None else ld, N, T, q, mean, omega2, None)


def _boot(d=DEV, ld=None, N=4, T=40, q32=1 << 28, n_boot=100, n_stats=4, shift=DEV, scale=DEV, out=DEV):
    return ("b200bt_spa_bootstrap", d, T if ld is None else ld, N, T, q32, n_boot, 0, 0, n_stats, shift, scale, out, None)


def test_entry_points_refuse_without_device(native_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    assert status(*_moments()) == ENODEVICE
    assert status(*_boot()) == ENODEVICE
    assert status(*_moments(T=2, q=1.0)) == ENODEVICE and status(*_boot(T=8192, N=1, n_stats=8, q32=1 << 32)) == ENODEVICE


def test_spa_moments_validates_arguments(native_lib):
    for null in ("d", "mean", "omega2"):
        assert status(*_moments(**{null: None})) == EINVAL, null
    assert status(*_moments(T=1)) == EINVAL
    assert status(*_moments(T=8193)) == ELIMIT
    assert status(*_moments(N=0)) == EINVAL
    assert status(*_moments(ld=39)) == EINVAL                    # row stride below T
    for q in (0.0, -0.1, 1.0000001, float("nan")):
        assert status(*_moments(q=q)) == EINVAL, q


def test_spa_bootstrap_validates_arguments(native_lib):
    for null in ("d", "shift", "scale", "out"):
        assert status(*_boot(**{null: None})) == EINVAL, null
    assert status(*_boot(T=1)) == EINVAL
    assert status(*_boot(T=8193)) == ELIMIT
    assert status(*_boot(N=0)) == EINVAL
    assert status(*_boot(ld=39)) == EINVAL
    assert status(*_boot(n_stats=0)) == EINVAL
    assert status(*_boot(n_stats=9)) == ELIMIT
    assert status(*_boot(q32=0)) == EINVAL
    assert status(*_boot(q32=(1 << 32) + 1)) == EINVAL
    assert status(*_boot(n_boot=0)) == EINVAL
    assert status(*_boot(n_boot=1 << 62, n_stats=8)) == ELIMIT  # n_stats * n_boot doubles overflow
