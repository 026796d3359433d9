"""RowMatrix / Statistics.corr on the resident shards: agd_gramian (csrc/gramian.cu) against a reference over the rows as
stored (read back with agd_get_rows / agd_get_csr_rows, selected with row_mask on views).

Bounds, with u = 2^-53 and n rows.  The device rounds each product x_i x_j once and adds n of them in some order, so an
uncentered entry is within (n + 2) u sum |x_i x_j| of the exact sum.  Every entry is compared with an fp64 BLAS reference
(itself within n u sum |x_i x_j|), so within (2 n + 3) u sum |x_i x_j|; a sample of entries, every diagonal entry and the
augmented column are also compared with math.fsum of the products (exact for fp32 and bf16 storage, whose products have at
most 48 significant bits; within u sum |x_i x_j| for fp64), within (n + 3) u sum |x_i x_j|.
Covariance: the device centres about its own mu; any shift c leaves sum (x - c)(x - c)^T - sum (x - c) sum (x - c)^T / n
unchanged, so the error of mu does not enter.  Rounding z = x - mu costs u |z| per factor, then a product and a sum of n terms
as above, and the correction term sum z_i sum z_j / n carries each sum's error times the other sum.  With S_ij = sum |z_i z_j|
and T_ij = sum |z_i| sum |z_j| / n (z about the reference mean) the device is within (n + 8) u (S_ij + 2 T_ij) / (n - 1) of
the exact covariance, and the BLAS reference within as much again: (2 n + 16) u (S_ij + 2 T_ij) / (n - 1).  CSR shards derive
it from uncentered sums (MLlib's formula), so there S and T are taken over x instead of z and T counts twice more.  Count
exact; a non-finite entry has the reference's IEEE class."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_score_gpu import _stored_csr, _stored_dense, bits  # noqa: E402

U = 2.0 ** -53


def ref_aug(Z):
    """fp64 BLAS reference of the augmented matrix [Z^T Z, Z^T 1; 1^T Z, n] of the rows Z, and the magnitudes sum |z_i z_j|
    (augmented the same way)."""
    A = np.concatenate([np.asarray(Z, dtype=np.float64), np.ones((Z.shape[0], 1))], axis=1)
    with np.errstate(invalid="ignore", over="ignore"):
        return A.T @ A, np.abs(A).T @ np.abs(A)


def check_close(got, ref, tol, what):
    fin = np.isfinite(ref)
    with np.errstate(invalid="ignore"):
        bad = fin & ~(np.abs(got - ref) <= tol)
    assert not bad.any(), (what, np.argwhere(bad)[:5], got[bad][:5], ref[bad][:5], tol[bad][:5])
    nf = ~fin
    assert np.array_equal(np.isnan(got[nf]), np.isnan(ref[nf])), what
    assert np.array_equal(got[nf & ~np.isnan(ref)], ref[nf & ~np.isnan(ref)]), what


def check_gramian(aug, Xs, samples=3000):
    """aug from agd_gramian(centered=False) against the rows Xs (module docstring)."""
    n, d = Xs.shape
    ref, mag = ref_aug(Xs)
    assert aug[-1, -1] == n
    check_close(aug, ref, (2 * n + 3) * U * mag, "gramian")
    assert np.array_equal(bits(aug), bits(aug.T))
    A = np.concatenate([Xs, np.ones((n, 1))], axis=1)
    rng = np.random.default_rng(d)
    ii = np.concatenate([np.arange(d + 1), np.arange(d + 1), rng.integers(0, d + 1, samples)])
    jj = np.concatenate([np.arange(d + 1), np.full(d + 1, d), rng.integers(0, d + 1, samples)])
    for i, j in zip(ii, jj):
        with np.errstate(invalid="ignore"):
            p = A[:, i] * A[:, j]
        if np.all(np.isfinite(p)):
            assert abs(aug[i, j] - math.fsum(p)) <= (n + 3) * U * mag[i, j], ("fsum", i, j, aug[i, j], math.fsum(p))


def ref_cov_bound(Xs, csr=False):
    """Reference covariance and its bound (module docstring)."""
    n = Xs.shape[0]
    mu = np.array([math.fsum(c) for c in Xs.T]) / n
    Z = Xs if csr else Xs - mu
    refz, magz = ref_aug(Xs - mu)
    cov = (refz[:-1, :-1] - np.outer(refz[:-1, -1], refz[:-1, -1]) / n) / (n - 1)
    a = np.abs(Z).sum(0)
    S = (ref_aug(Z)[1] if csr else magz)[:-1, :-1]
    T = np.outer(a, a) / n
    return cov, (2 * n + 16) * U * (S + (4 if csr else 2) * T) / (n - 1)


def check_cov(agd, ds, Xs, csr=False):
    n = Xs.shape[0]
    cov = agd.RowMatrix(ds).computeCovariance()
    ref, tol = ref_cov_bound(Xs, csr)
    check_close(cov, ref, tol, "covariance")
    assert np.array_equal(bits(cov), bits(cov.T))
    return cov


def _matrix(rng, n, d):
    X = rng.standard_normal((n, d)) * np.exp(rng.uniform(-2, 2, d)) + rng.uniform(-3, 3, d)
    X[rng.random((n, d)) < 0.15] = 0.0
    if d > 2:
        X[:, 1] = 0.0
    return X


# aligned (16-byte rows: cp.async staging) for every padded width; 2051 (fp64) and 4099 (fp32, bf16) are left unpadded by the
# pad rule and take the plain-load staging form
DS = [1, 3, 127, 128, 129, 1001, 1024, 4096, "plain"]
PLAIN = {"f32": 4099, "f64": 2051, "bf16": 4099}


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", DS)
def test_dense(agd, ctx, store, d):
    d = PLAIN[store] if d == "plain" else d
    rng = np.random.default_rng(d * 5 + len(store))
    n1, n2 = (1, 37) if d >= 2048 else (1, 301)
    X = _matrix(rng, n1 + n2, d)
    y = np.zeros(n1 + n2)
    ds = ctx.parallelize(y[:n1], X[:n1], store=store)        # a one-row shard ...
    try:
        Xs = _stored_dense(ds, store)[0][:, :d]
        n, aug = ds.gramian(False)
        assert n == 1 and aug.shape == (d + 1, d + 1)         # padded columns are not reported
        check_gramian(aug, Xs)
        with pytest.raises(ValueError, match="<= 1 row"):
            agd.RowMatrix(ds).computeCovariance()
        ds.load_dense(y[n1:], X[n1:], store=store)            # ... and an appended, ragged partition
        Xs = _stored_dense(ds, store)[0][:, :d]
        n, aug = ds.gramian(False)
        check_gramian(aug, Xs)
        g = agd.RowMatrix(ds).computeGramianMatrix()
        assert np.array_equal(bits(g), bits(aug[:-1, :-1]))
        cov = check_cov(agd, ds, Xs)
        again = agd.RowMatrix(ds).computeCovariance()          # dense: bit-identical on a repeated call
        assert np.array_equal(bits(cov), bits(again))
        assert np.array_equal(bits(ds.gramian(False)[1]), bits(aug))
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_generated_shard(agd, ctx, store):
    ds = ctx.synthetic(3001, 256, agd.LogisticGradient(), seed=7, store=store)
    try:
        Xs = _stored_dense(ds, store)[0][:, :256]
        check_gramian(ds.gramian(False)[1], Xs)
        check_cov(agd, ds, Xs)
    finally:
        ds.close()


def _csr_rows(rp, ix, va, d, keep=None):
    n = rp.shape[0] - 1
    X = np.zeros((n, d))
    rows = np.repeat(np.arange(n), np.diff(rp))
    np.add.at(X, (rows, ix), va)
    return X if keep is None else X[keep]


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
@pytest.mark.parametrize("d", [1, 100, 1500])
def test_csr(agd, ctx, store, d):
    rng = np.random.default_rng(d + 17)
    n = 1201
    nnz = rng.integers(0, min(d, 40) + 1, size=n)
    nnz[[0, 9, n - 1]] = 0                                     # empty rows
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate([np.sort(rng.choice(d, k, replace=False)) for k in nnz]).astype(np.int32)
    va = rng.standard_normal(ix.shape[0]) * 3 - 1
    va[::7] = 0.0                                              # explicitly stored zeros
    y = np.zeros(n)
    h = 500
    ds = ctx.parallelize_csr(y[:h], rp[:h + 1], ix[:rp[h]], va[:rp[h]], d, store=store)
    try:
        ds.load_csr(y[h:], rp[h:] - rp[h], ix[rp[h]:], va[rp[h]:], d, store=store)   # appended partition
        rps, ixs, vas, _ = _stored_csr(ds, store)
        Xs = _csr_rows(rps, ixs, vas, d)
        n_, aug = ds.gramian(False)
        check_gramian(aug, Xs)
        check_cov(agd, ds, Xs, csr=True)
        view = ds.sample(False, 0.4, seed=3)
        keep = view.row_mask(0, 0, n)
        check_gramian(view.gramian(False)[1], Xs[keep])
        check_cov(agd, view, Xs[keep], csr=True)
    finally:
        ds.close()


@pytest.mark.gpu
def test_large_mean_covariance(agd, ctx):
    """mean 1e6 and unit spread: the centered device sums give the covariance within 1e-10 relative (MLlib's G - n mu mu^T
    loses most digits here)."""
    rng = np.random.default_rng(6)
    X = 1e6 + rng.standard_normal((20000, 3)) @ np.array([[1.0, 0.3, 0.0], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]])
    ds = ctx.parallelize(np.zeros(20000), X, store="f64")
    try:
        cov = agd.RowMatrix(ds).computeCovariance()
        Xc = X - np.array([math.fsum(c) for c in X.T]) / 20000
        ref = np.array([[math.fsum(Xc[:, i] * Xc[:, j]) for j in range(3)] for i in range(3)]) / 19999
        np.testing.assert_allclose(cov, ref, rtol=1e-10, atol=1e-10 * np.abs(ref).max())
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_views_and_nonfinite(agd, ctx, store):
    """±inf / NaN in rows outside a view leave no trace; inside it they follow IEEE arithmetic."""
    n, d = 2000, 130
    rng = np.random.default_rng(9)
    X = _matrix(rng, n, d)
    ds0 = ctx.parallelize(np.zeros(n), X, store=store)
    try:
        mask = ds0.sample(False, 0.5, seed=13).row_mask(0, 0, n)
    finally:
        ds0.close()
    out, kept = np.flatnonzero(~mask), np.flatnonzero(mask)
    inf, nan = float("inf"), float("nan")
    X[out[:3], 0] = [inf, -inf, nan]
    X[out[3:40], 5:129] = nan                                  # whole excluded rows across a block boundary
    ds = ctx.parallelize(np.zeros(n), X, store=store)
    try:
        view = ds.sample(False, 0.5, seed=13)
        assert np.array_equal(view.row_mask(0, 0, n), mask)
        Xs = _stored_dense(ds, store)[0][:, :d]
        _, aug = view.gramian(False)
        assert np.all(np.isfinite(aug))
        check_gramian(aug, Xs[mask])
        check_cov(agd, view, Xs[mask])
    finally:
        ds.close()
    X[kept[0], 2] = inf
    X[kept[1], 3], X[kept[2], 3] = inf, -inf
    ds = ctx.parallelize(np.zeros(n), X, store=store)
    try:
        view = ds.sample(False, 0.5, seed=13)
        Xs = _stored_dense(ds, store)[0][:, :d]
        _, aug = view.gramian(False)
        check_gramian(aug, Xs[mask])
        assert aug[2, 2] == inf and aug[3, 3] == inf and math.isnan(aug[3, d])     # sum x_3 = inf - inf
        assert np.isfinite(aug[0, 0]) and np.isfinite(aug[5, 6])
    finally:
        ds.close()


@pytest.mark.gpu
def test_corr_and_pca(agd, ctx):
    rng = np.random.default_rng(11)
    n, d = 5000, 40
    Q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    ev = np.concatenate([[50.0, 20.0, 8.0, 3.0], np.linspace(1.0, 0.1, d - 4)])
    X = (rng.standard_normal((n, d)) * np.sqrt(ev)) @ Q.T + rng.uniform(-10, 10, d)
    X[:, 7] = 4.0                                              # a constant column
    ds = ctx.parallelize(np.zeros(n), X, store="f64")
    try:
        Xs = _stored_dense(ds, "f64")[0]
        ref_cov, _ = ref_cov_bound(Xs)
        corr = agd.Statistics.corr(ds)
        assert agd.Statistics.corr(ds, "pearson").shape == (d, d)
        assert np.all(np.diag(corr) == 1.0)
        assert np.all(np.isnan(np.delete(corr[7], 7))) and np.all(np.isnan(np.delete(corr[:, 7], 7)))
        ref = agd.linalg.correlation_from_covariance(ref_cov)
        keep = np.delete(np.arange(d), 7)
        np.testing.assert_allclose(corr[np.ix_(keep, keep)], ref[np.ix_(keep, keep)], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(corr[np.ix_(keep, keep)], np.corrcoef(X[:, keep], rowvar=False), rtol=1e-10, atol=1e-12)
        pc = agd.RowMatrix(ds).computePrincipalComponents(3)
        w, v = np.linalg.eigh(ref_cov)
        for k in range(3):
            assert abs(pc[:, k] @ v[:, -1 - k]) >= 1 - 1e-9
            assert pc[np.argmax(np.abs(pc[:, k])), k] > 0
        with pytest.raises(ValueError, match="out of range"):
            agd.RowMatrix(ds).computePrincipalComponents(d + 1)
        with pytest.raises(NotImplementedError):
            agd.Statistics.corr(ds, method="spearman")
        rm = agd.RowMatrix(ds)
        assert rm.numRows() == n and rm.numCols() == d
        assert np.array_equal(rm.computeColumnSummaryStatistics().mean, agd.Statistics.colStats(ds).mean)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_transformed_views(agd, ctx, store):
    """StandardScaler + appendBias views: the statistics of the transformed rows [s o x, 1]."""
    n, d = 3000, 64
    rng = np.random.default_rng(12)
    X = _matrix(rng, n, d)
    ds = ctx.parallelize(np.zeros(n), X, store=store)
    try:
        Xs = _stored_dense(ds, store)[0][:, :d]
        model = agd.StandardScaler(withMean=False, withStd=True).fit(ds)
        tv = agd.MLUtils.appendBias(model.transform(ds))
        s = np.asarray(model.factor)
        Xt = np.concatenate([Xs * s, np.ones((n, 1))], axis=1)
        rm = agd.RowMatrix(tv)
        assert rm.numCols() == d + 1
        g = rm.computeGramianMatrix()
        ref, mag = ref_aug(Xt)
        check_close(g, ref[:-1, :-1], (2 * n + 8) * U * mag[:-1, :-1], "scaled gramian")
        cov = rm.computeCovariance()
        assert np.all(cov[d] == 0.0) and np.all(cov[:, d] == 0.0)
        ref_cov, tol = ref_cov_bound(Xt)
        check_close(cov[:d, :d], ref_cov[:d, :d], 4 * tol[:d, :d], "scaled covariance")
        corr = agd.Statistics.corr(tv)
        assert corr[d, d] == 1.0 and np.all(np.isnan(corr[d, :d])) and np.all(np.isnan(corr[:d, d]))
        live = np.flatnonzero(s != 0)
        np.testing.assert_allclose(corr[np.ix_(live, live)], np.corrcoef(Xt[:, live], rowvar=False), rtol=1e-9, atol=1e-12)
        sub = agd.MLUtils.appendBias(model.transform(ds.sample(False, 0.5, seed=2)))   # a row view of it too
        keep = sub.row_mask(0, 0, n)
        check_close(agd.RowMatrix(sub).computeGramianMatrix(), ref_aug(Xt[keep])[0][:-1, :-1],
                    (2 * n + 8) * U * ref_aug(Xt[keep])[1][:-1, :-1], "view gramian")
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_collectives_keep_their_bits(agd, ctx, store):
    """smooth, evaluate and colStats give the same bits before and after a gramian call (the exchange epochs stay in step)."""
    ds = ctx.synthetic(4001, 300, agd.LogisticGradient(), seed=5, store=store)
    try:
        w = np.linspace(-0.2, 0.2, 300)
        l1, g1, c1 = ds.smooth(agd.LogisticGradient(), w)
        e1 = ds.evaluate(agd.LogisticGradient(), w)
        s1 = agd.Statistics.colStats(ds)
        agd.RowMatrix(ds).computeCovariance()
        ds.gramian(False)
        l2, g2, c2 = ds.smooth(agd.LogisticGradient(), w)
        assert l1 == l2 and c1 == c2 and np.array_equal(bits(g1), bits(g2))
        e2 = ds.evaluate(agd.LogisticGradient(), w)
        assert np.array_equal(bits(list(e1.__dict__.values())), bits(list(e2.__dict__.values())))
        s2 = agd.Statistics.colStats(ds)
        assert np.array_equal(bits(s1.dev2), bits(s2.dev2)) and np.array_equal(bits(s1.sum), bits(s2.sum))
    finally:
        ds.close()


@pytest.mark.gpu
def test_errors(agd, ctx):
    ds = ctx.parallelize(np.zeros(3), np.ones((3, 8193)), store="f32")
    try:
        with pytest.raises(agd.NativeError, match="8192"):
            ds.gramian(False)
        with pytest.raises(agd.NativeError, match="8192"):
            agd.RowMatrix(ds).computeCovariance()
    finally:
        ds.close()
    ds = ctx.parallelize(np.zeros(50), np.ones((50, 4)), store="f32")
    try:
        empty = ds.sample(False, 0.0, seed=1)
        n, aug = empty.gramian(True)
        assert n == 0
        for call in (lambda: agd.RowMatrix(empty).computeCovariance(), lambda: agd.RowMatrix(empty).computeGramianMatrix(),
                     lambda: agd.Statistics.corr(empty)):
            with pytest.raises(ValueError, match="no rows"):
                call()
    finally:
        ds.close()
