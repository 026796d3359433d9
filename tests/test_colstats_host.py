"""MultivariateStatisticalSummary.from_sums: the host derivation of Statistics.colStats from the sums agd_col_stats returns
(no GPU needed)."""
import math

import numpy as np
import pytest


def _sums(X):
    """The AGD_COLSTAT_* block of a dense matrix, as the device defines it (mu = fl(sum / n))."""
    X = np.asarray(X, dtype=np.float64)
    n = X.shape[0]
    s = np.array([math.fsum(c) for c in X.T])
    mu = s / n
    dev = np.array([math.fsum(c) for c in (X - mu).T])
    dev2 = np.array([math.fsum(c) for c in ((X - mu) ** 2).T])
    return n, np.stack([s, (X * X).sum(0), np.abs(X).sum(0), (X != 0).sum(0).astype(np.float64), dev, dev2,
                        np.fmax.reduce(X, axis=0), np.fmin.reduce(X, axis=0)])


def test_from_sums_against_numpy(agd):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((57, 6)) * [1, 10, 0.1, 1, 5, 2] + [0, 3, -2, 0, 1e3, 7]
    X[::4, 3] = 0.0
    n, sums = _sums(X)
    s = agd.MultivariateStatisticalSummary.from_sums(n, sums)
    assert s.count == 57 and isinstance(s.count, int)
    np.testing.assert_allclose(s.mean, X.mean(0), rtol=1e-14)
    np.testing.assert_allclose(s.variance, X.var(0, ddof=1), rtol=1e-12)
    np.testing.assert_array_equal(s.numNonzeros, (X != 0).sum(0))
    np.testing.assert_array_equal(s.max, X.max(0))
    np.testing.assert_array_equal(s.min, X.min(0))
    np.testing.assert_allclose(s.normL1, np.abs(X).sum(0), rtol=1e-14)
    np.testing.assert_allclose(s.normL2, np.linalg.norm(X, axis=0), rtol=1e-14)


def test_corrected_variance_survives_a_large_mean(agd):
    """mean 1e6, unit spread: sum x^2 - (sum x)^2 / n cancels to garbage; the corrected two-pass formula does not."""
    rng = np.random.default_rng(4)
    X = 1e6 + rng.standard_normal((1000, 1))
    n, sums = _sums(X)
    s = agd.MultivariateStatisticalSummary.from_sums(n, sums)
    exact = math.fsum((X[:, 0] - math.fsum(X[:, 0]) / n) ** 2) / (n - 1)
    assert abs(s.variance[0] - exact) <= 1e-12 * exact
    naive = (sums[1, 0] - sums[0, 0] ** 2 / n) / (n - 1)
    assert abs(naive - exact) > 1e-6 * exact          # the formula the device sums avoid


def test_one_row_has_zero_variance(agd):
    n, sums = _sums([[3.5, -1.0, 0.0]])
    s = agd.MultivariateStatisticalSummary.from_sums(n, sums)
    assert s.count == 1
    np.testing.assert_array_equal(s.variance, [0.0, 0.0, 0.0])
    np.testing.assert_array_equal(s.mean, [3.5, -1.0, 0.0])
    np.testing.assert_array_equal(s.numNonzeros, [1, 1, 0])


def test_all_nan_column_reports_nan_extrema(agd):
    nan = float("nan")
    X = np.array([[nan, 1.0], [nan, -2.0], [nan, nan]])
    n, sums = _sums(X)
    s = agd.MultivariateStatisticalSummary.from_sums(n, sums)
    assert math.isnan(s.max[0]) and math.isnan(s.min[0])          # MLlib would report its Double.MinValue / MaxValue
    assert s.max[1] == 1.0 and s.min[1] == -2.0                   # NaN ignored by max / min ...
    assert math.isnan(s.mean[1]) and s.numNonzeros[1] == 3        # ... but not by the sums; a NaN is nonzero


def test_empty_raises(agd):
    with pytest.raises(ValueError, match="Nothing has been added"):
        agd.MultivariateStatisticalSummary.from_sums(0.0, np.zeros((agd._native.COLSTAT_N, 3)))


def test_summary_is_frozen_and_shape_checked(agd):
    n, sums = _sums([[1.0, 2.0], [3.0, 4.0]])
    s = agd.MultivariateStatisticalSummary.from_sums(n, sums)
    with pytest.raises(Exception):
        s.n = 3.0
    with pytest.raises(ValueError):
        s.sum[0] = 1.0
    s.max[0] = 99.0                                               # a property returns a copy
    assert s.max[0] == 3.0
    with pytest.raises(ValueError, match="x d"):
        agd.MultivariateStatisticalSummary.from_sums(2.0, np.zeros((3, 2)))
    assert agd._native.COLSTAT_N == 8 and "agd_col_stats" in agd.exported_symbols()
