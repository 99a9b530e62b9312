"""Host arithmetic of the Monte-Carlo statistics that needs no GPU: NumPy's linear-interpolation percentile rule
rebuilt from exact order statistics (ai_crypto_trader_b200.monte_carlo.percentile_points / _virtual_index / _lerp)."""
import numpy as np

from ai_crypto_trader_b200.monte_carlo import PERCENTILES, _lerp, _virtual_index, percentile_points


def test_percentile_rule_equals_numpy():
    rng = np.random.default_rng(12)
    qs = list(PERCENTILES) + [0.0, 100.0, 5.0, 0.1, 99.9, 33.333, 100 * (1 - 0.95)]
    for n in (1, 2, 3, 10, 101, 1000, 99_999):
        x = rng.standard_normal(n).astype(np.float32)
        srt = np.sort(x).astype(np.float64)
        x64 = x.astype(np.float64)
        for q in qs:
            lo, hi, g = _virtual_index(n, q)
            assert 0 <= lo <= hi <= n - 1 and 0.0 <= g < 1.0
            got = _lerp(srt[lo], srt[hi], g)
            assert got == np.percentile(x64, q), (n, q)
        # every percentile from ONE select over the union of the ranks, as the device select is called
        calls = []

        def select(ranks):
            calls.append(list(ranks))
            assert list(ranks) == sorted(set(ranks))
            return srt[ranks]

        points = percentile_points(select, n, qs)
        assert len(calls) == 1 and len(points) == len(qs)
        pct = lambda v: (v / 1.2345 - 1) * 100
        for q, (x_lo, x_hi, g) in zip(qs, points):
            assert _lerp(x_lo, x_hi, g) == np.percentile(x64, q), (n, q)
            # the VaR form: the percentage change of each order statistic, then the interpolation
            assert _lerp(pct(x_lo), pct(x_hi), g) == np.percentile(pct(x64), q), (n, q)
