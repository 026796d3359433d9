"""RowMatrix.multiply / computeSVD host logic (no GPU): the fold of a transformed view into the projection, the (s, V) step of
computeSVD against numpy, the argument errors, and the agd_project symbol in the header and the binding."""
import numpy as np
import pytest

from test_abi import declared_symbols


def test_fold_matches_projecting_transformed_rows(agd):
    rng = np.random.default_rng(1)
    n, d, k = 50, 9, 4
    X = rng.standard_normal((n, d))
    s = rng.uniform(-2, 2, d)
    s[[2, 5]] = 0.0                      # zero scale (a constant column under StandardScaler)
    s[3] = -0.75                         # negative scale
    c0 = rng.standard_normal(k)
    for scale in (None, s):
        for bias in (False, True):
            Xt = X * (1.0 if scale is None else scale)
            if bias:
                Xt = np.concatenate([Xt, np.ones((n, 1))], axis=1)
            B = rng.standard_normal((Xt.shape[1], k))
            for off in (None, c0):
                P, c = agd.physical_projection(B, off, scale, bias, Xt.shape[1])
                assert P.shape == (d, k) and c.shape == (k,)
                ref = Xt @ B + (0.0 if off is None else off)
                np.testing.assert_allclose(X @ P + c, ref, rtol=1e-13, atol=1e-13 * np.abs(ref).max())
                if bias:
                    assert np.array_equal(c, (np.zeros(k) if off is None else off) + B[-1])
                if scale is not None:
                    assert np.all(P[[2, 5]] == 0.0)


def test_fold_errors(agd):
    B = np.ones((4, 2))
    for bad in (np.ones((3, 2)), np.ones((4, 0)), np.ones(4), np.ones((4, 2, 1))):
        with pytest.raises(ValueError, match="shape"):
            agd.physical_projection(bad, None, None, False, 4)
    for v in (np.nan, np.inf, -np.inf):
        Bb = B.copy()
        Bb[1, 1] = v
        with pytest.raises(ValueError, match="finite"):
            agd.physical_projection(Bb, None, None, False, 4)
        with pytest.raises(ValueError, match="finite"):
            agd.physical_projection(B, np.array([0.0, v]), None, False, 4)
    with pytest.raises(ValueError, match="shape"):
        agd.physical_projection(B, np.zeros(3), None, False, 4)
    with pytest.raises(ValueError, match="overflows"):
        agd.physical_projection(np.full((4, 2), 1e300), None, np.full(4, 1e10), False, 4)


def _svd_check(agd, A, k, rcond=1e-9):
    G = A.T @ A
    s, V = agd.linalg.svd_from_gramian(G, k, rcond)
    _, sr, vt = np.linalg.svd(A)
    m = s.shape[0]
    np.testing.assert_allclose(s, sr[:m], rtol=1e-12)
    for i in range(m):
        assert abs(V[:, i] @ vt[i]) >= 1 - 1e-9
        assert V[np.argmax(np.abs(V[:, i])), i] > 0                 # sign rule: the largest entry is positive
    return s, V


def test_svd_from_gramian(agd):
    rng = np.random.default_rng(2)
    n, d = 400, 12
    Q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    sv = np.linspace(10.0, 1.0, d)
    U, _ = np.linalg.qr(rng.standard_normal((n, d)))
    A = (U * sv) @ Q.T
    for k in (1, 5, d):
        s, V = _svd_check(agd, A, k)
        assert s.shape == (k,) and V.shape == (d, k)
        assert np.all(np.diff(s) <= 0)


def test_svd_rcond_truncation(agd):
    rng = np.random.default_rng(3)
    n, d = 300, 8
    U, _ = np.linalg.qr(rng.standard_normal((n, d)))
    Q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    sv = np.array([8.0, 4.0, 2.0, 1.0, 1e-3, 1e-4, 0.0, 0.0])
    A = (U * sv) @ Q.T
    s, V = agd.linalg.svd_from_gramian(A.T @ A, d, 1e-2)       # keeps sigma >= 0.08: four of them
    assert s.shape == (4,) and V.shape == (d, 4)
    np.testing.assert_allclose(s, sv[:4], rtol=1e-12)
    s, _ = agd.linalg.svd_from_gramian(A.T @ A, 3, 1e-2)        # at most k
    assert s.shape == (3,)
    s, _ = agd.linalg.svd_from_gramian(A.T @ A, d, 0.5)         # only 8 and 4 reach half of the largest
    assert s.shape == (2,)


def test_svd_k_errors(agd):
    G = np.eye(3)
    for k in (0, 4, -1, 1.5):
        with pytest.raises(ValueError, match="out of range"):
            agd.linalg.svd_from_gramian(G, k)


def test_principal_components_sign_rule_unchanged(agd):
    """principal_components shares the sign rule with svd_from_gramian: the first of two equal largest magnitudes decides."""
    cov = np.diag([3.0, 2.0, 1.0])
    pc = agd.linalg.principal_components(cov, 3)
    assert np.array_equal(pc, np.eye(3))
    m = agd.linalg._fix_signs(np.array([[-0.5, 0.5], [0.5, -0.5]]))
    assert np.array_equal(m, np.array([[0.5, 0.5], [-0.5, -0.5]]))


def test_symbol_in_header_and_binding(agd):
    assert "agd_project" in declared_symbols()
    assert "agd_project" in agd.exported_symbols()
    assert agd.SingularValueDecomposition._fields == ("U", "s", "V")
