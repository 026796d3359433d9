"""The host derivations of RowMatrix / Statistics.corr from the augmented cross-product matrix agd_gramian returns (no GPU
needed): covariance with the two-pass correction, Pearson correlation with MLlib's zero-variance rule, principal components
and their sign convention, the StandardScaler / appendBias mapping, and the errors."""
import numpy as np
import pytest


def _aug(Z):
    """[Z^T Z, Z^T 1; 1^T Z, n] of the rows Z."""
    A = np.concatenate([np.asarray(Z, dtype=np.float64), np.ones((Z.shape[0], 1))], axis=1)
    return A.T @ A


def _centered_aug(X):
    mu = X.sum(0) / X.shape[0]
    return _aug(X - mu)


@pytest.fixture(scope="module")
def L(agd):
    return agd.linalg


def test_covariance_with_correction(L):
    rng = np.random.default_rng(1)
    X = rng.standard_normal((83, 7)) @ rng.standard_normal((7, 7)) + rng.uniform(-5, 5, 7)
    ref = np.cov(X, rowvar=False, ddof=1)
    for aug in (_aug(X), _centered_aug(X)):
        cov = L.covariance_from_augmented(aug)
        np.testing.assert_allclose(cov, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
        assert np.array_equal(cov, cov.T)
    # the correction term: centering about a shifted mu gives the same covariance
    cov = L.covariance_from_augmented(_aug(X - (X.mean(0) + 0.25)))
    np.testing.assert_allclose(cov, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())


def test_centered_form_survives_a_large_mean(L):
    rng = np.random.default_rng(2)
    X = 1e6 + rng.standard_normal((2000, 3))
    ref = np.cov(X - X.mean(0), rowvar=False, ddof=1)
    np.testing.assert_allclose(L.covariance_from_augmented(_centered_aug(X)), ref, rtol=1e-12)
    # MLlib's uncentered form loses most digits here (the reason the device centres dense shards)
    assert np.abs(L.covariance_from_augmented(_aug(X)) - ref).max() > 1e-6


def test_corr_zero_variance_rule(L):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((50, 5))
    X[:, 1] = 3.0                       # constant column
    X[:, 3] = 2.0 + 1e-7 * (np.arange(50) % 2)   # variance ~2.5e-15 <= 1e-12: treated as constant
    cov = np.cov(X, rowvar=False, ddof=1)
    r = L.correlation_from_covariance(cov)
    assert np.all(np.diag(r) == 1.0)
    for j in (1, 3):
        off = np.delete(r[j], j)
        assert np.all(np.isnan(off)) and np.all(np.isnan(np.delete(r[:, j], j)))
    keep = [0, 2, 4]
    np.testing.assert_allclose(r[np.ix_(keep, keep)], np.corrcoef(X[:, keep], rowvar=False), rtol=1e-13, atol=1e-15)
    assert np.array_equal(r, r.T, equal_nan=True)
    # just above the threshold the column is not constant
    c = np.array([[2e-12, 1e-12], [1e-12, 1.0]])
    r = L.correlation_from_covariance(c)
    assert np.isfinite(r[0, 1]) and r[0, 1] == 1e-12 / np.sqrt(2e-12)


def test_pca_order_and_sign(L):
    rng = np.random.default_rng(4)
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    ev = np.array([9.0, 5.0, 3.0, 1.0, 0.5, 0.1])
    cov = (Q * ev) @ Q.T
    cov = (cov + cov.T) / 2
    pc = L.principal_components(cov, 4)
    assert pc.shape == (6, 4)
    for k in range(4):
        v = pc[:, k]
        assert abs(abs(v @ Q[:, k]) - 1.0) < 1e-12                   # descending eigenvalue order
        assert v[np.argmax(np.abs(v))] > 0                            # largest entry positive
    np.testing.assert_allclose(pc.T @ pc, np.eye(4), atol=1e-13)


def test_transform_mapping(L):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((40, 4)) * [1, 2, 3, 4] + [0, 1, -2, 5]
    s = np.array([0.5, 0.0, 2.0, 1.0 / 3.0])
    Xt = np.concatenate([X * s, np.ones((40, 1))], axis=1)
    for scale, bias in ((s, False), (None, True), (s, True)):
        direct = (X * s if scale is not None else X)
        if bias:
            direct = np.concatenate([direct, np.ones((40, 1))], axis=1)
        got = L.augmented_transformed(_aug(X), scale, bias, centered=False)
        np.testing.assert_allclose(got, _aug(direct), rtol=1e-13, atol=1e-12)
        gc = L.augmented_transformed(_centered_aug(X), scale, bias, centered=True)
        np.testing.assert_allclose(L.covariance_from_augmented(gc), np.cov(direct, rowvar=False, ddof=1), rtol=1e-12,
                                   atol=1e-12)
    # corr of a view with an intercept: NaN row and column for the bias, 1.0 on the diagonal (MLlib's constant column)
    gc = L.augmented_transformed(_centered_aug(X), s, True, centered=True)
    r = L.correlation_from_covariance(L.covariance_from_augmented(gc))
    assert r[4, 4] == 1.0 and np.all(np.isnan(r[4, :4])) and np.all(np.isnan(r[:4, 4]))
    assert np.all(np.isnan(r[1, [0, 2, 3]]))                          # a zero scale factor makes a constant column
    np.testing.assert_allclose(r[np.ix_([0, 2, 3], [0, 2, 3])], np.corrcoef(Xt[:, [0, 2, 3]], rowvar=False), rtol=1e-12)


def test_errors(L, agd):
    with pytest.raises(ValueError, match="no rows"):
        L.covariance_from_augmented(np.zeros((3, 3)))
    one = _aug(np.array([[1.0, 2.0]]))
    with pytest.raises(ValueError, match="<= 1 row"):
        L.covariance_from_augmented(one)
    cov = np.eye(3)
    for k in (0, 4, -1, 1.5):
        with pytest.raises(ValueError, match="out of range"):
            L.principal_components(cov, k)
    with pytest.raises(NotImplementedError, match="sort"):
        agd.Statistics.corr(None, method="spearman")
    with pytest.raises(ValueError, match="unknown correlation method"):
        agd.Statistics.corr(None, method="kendall")
    assert agd._native.GRAMIAN_MAX_DIM == 8192
