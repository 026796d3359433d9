"""RowMatrix.multiply / DeviceDataset.project on the resident shards: agd_project (csrc/project.cu) against a reference over the
rows as stored (read back with agd_get_rows / agd_get_csr_rows, selected with row_mask on views), and computeSVD.

Bound.  With u = 2^-53 and gamma_n = n u / (1 - n u), the device forms y_ij = sum_l x_il b_lj (d products, each x widened
exactly to fp64) and then + c_j: d + 1 fp64 operations that each round at most once, so before the final rounding
|y_ij - exact| <= gamma_{d+1} (sum_l |x_il b_lj| + |c_j|) (padded columns add exact zeros).  The reference is the same sum in
np.longdouble (64-bit significand, u' = 2^-64), within gamma'_{d+1} of the same magnitude, so an fp64 destination is held to
(gamma_{d+1} + gamma'_{d+1}) (sum |x b| + |c|) of the reference.  fp32 / bf16 destinations must equal, bit for bit, the
round-to-nearest-even of the fp64 destination's values (the device rounds the same fp64 sum once).  A row whose reference is
non-finite must have the same IEEE class.
computeSVD: s and V from the device Gramian (within (2 n + 3) u sum |x_i x_j| per entry, tests/test_gramian_gpu.py) against
numpy's SVD of the stored rows.  U = A V diag(1 / s) on the device; U^T U = I up to the Gramian's and the projection's rounding
magnified by the conditioning of the kept block: |U^T U - I| <= 64 (n + d) u (s_0 / s_{k-1})^2."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gramian_gpu import _csr_rows  # noqa: E402
from test_score_gpu import _stored_csr, _stored_dense, bits  # noqa: E402

U = 2.0 ** -53
UL = float(np.finfo(np.longdouble).eps) / 2


def gamma(n, u):
    return n * u / (1 - n * u)


def rne_bf16(y):
    """fp64 -> bf16 bit patterns, round to nearest even (finite values in the normal range)."""
    u = np.ascontiguousarray(y, dtype=np.float64).view(np.uint64)
    lsb = (u >> np.uint64(45)) & np.uint64(1)
    r = (u + np.uint64((1 << 44) - 1) + lsb) & ~np.uint64((1 << 45) - 1)
    return (r.view(np.float64).astype(np.float32).view(np.uint32) >> np.uint32(16)).astype(np.uint16)


def rows_of(ds, store, k):
    """The projected rows as stored, and their labels (device 0)."""
    n = ds.local_rows(0)
    X, y = ds.get_rows(0, 0, n, dtype={"f32": np.float32, "f64": np.float64, "bf16": np.uint16}[store])
    assert X.shape == (n, k)
    return X, y


def check_projection(Y, Xs, B, c):
    """Y (fp64 destination) against the longdouble reference of Xs B + c (module docstring)."""
    n, d = Xs.shape
    assert Y.shape == (n, B.shape[1])
    XL, BL = Xs.astype(np.longdouble), B.astype(np.longdouble)
    with np.errstate(invalid="ignore", over="ignore"):
        ref = XL @ BL + c.astype(np.longdouble)
        mag = np.abs(Xs) @ np.abs(B) + np.abs(c)
    tol = (gamma(d + 1, U) + gamma(d + 1, UL)) * mag * (1 + 1e-9)
    fin = np.isfinite(ref)
    with np.errstate(invalid="ignore"):
        bad = fin & ~(np.abs(Y.astype(np.longdouble) - ref) <= tol)
    assert not bad.any(), (np.argwhere(bad)[:5], Y[bad][:5], ref[bad][:5], tol[bad][:5])
    nf = ~fin
    assert np.array_equal(np.isnan(Y[nf]), np.isnan(ref[nf]))
    assert np.array_equal(Y[nf & ~np.isnan(ref)], ref[nf & ~np.isnan(ref)].astype(np.float64))


def _matrix(rng, n, d):
    X = rng.standard_normal((n, d)) * np.exp(rng.uniform(-2, 2, d)) + rng.uniform(-3, 3, d)
    X[rng.random((n, d)) < 0.15] = 0.0
    return X


def _B(rng, d, k):
    B = rng.standard_normal((d, k)) * np.exp(rng.uniform(-3, 3, (d, 1)))
    B[rng.random((d, k)) < 0.1] = 0.0
    return B, rng.standard_normal(k) * 10


# (d, k): every d of the staging forms and padded widths, every k from one to several column tiles
CASES = [(1, 1), (1, 300), (7, 3), (7, 128), (16, 8), (16, 64), (127, 300), (127, 1), (1024, 64), (1024, 128), (4096, 3),
         (4096, 300), ("plain", 8), ("plain", 130)]
PLAIN = {"f32": 4099, "f64": 2051, "bf16": 4099}


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d,k", CASES)
def test_dense(agd, ctx, store, d, k):
    d = PLAIN[store] if d == "plain" else d
    rng = np.random.default_rng(d * 7 + k)
    n1, n2 = (3, 130) if d >= 2048 else (5, 300)
    X = _matrix(rng, n1 + n2, d)
    y = rng.standard_normal(n1 + n2)
    B, c = _B(rng, d, k)
    ds = ctx.parallelize(y[:n1], X[:n1], store=store)
    try:
        ds.load_dense(y[n1:], X[n1:], store=store)                 # two partitions: a ragged last row tile
        Xs, ys = _stored_dense(ds, store)
        Xs = Xs[:, :d]
        p64 = ds.project(B, c, store="f64")
        try:
            Y, yl = rows_of(p64, "f64", k)
            check_projection(Y, Xs, B, c)
            assert np.array_equal(bits(yl), bits(ys))                # labels carried exactly
            again = ds.project(B, c, store="f64")
            assert np.array_equal(bits(rows_of(again, "f64", k)[0]), bits(Y))   # repeated calls: identical bits
            again.close()
            p32 = ds.project(B, c, store="f32")
            assert np.array_equal(rows_of(p32, "f32", k)[0].view(np.uint32), Y.astype(np.float32).view(np.uint32))
            p32.close()
            pb = ds.project(B, c, store="bf16")
            assert np.array_equal(rows_of(pb, "bf16", k)[0], rne_bf16(Y))
            pb.close()
        finally:
            p64.close()
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_generated_and_split(agd, ctx, store):
    """A generated shard; randomSplit of the projection selects exactly the rows the same split of the source selects."""
    ds = ctx.synthetic(3001, 256, agd.LogisticGradient(), seed=7, store=store)
    try:
        Xs, ys = _stored_dense(ds, store)
        rng = np.random.default_rng(5)
        B, c = _B(rng, 256, 40)
        p = agd.RowMatrix(ds).multiply(B).data
        try:
            Y, yl = rows_of(p, "f64", 40)
            check_projection(Y, Xs[:, :256], B, np.zeros(40))
            assert np.array_equal(bits(yl), bits(ys))
            for a, b in zip(ds.randomSplit([0.3, 0.7], seed=9), p.randomSplit([0.3, 0.7], seed=9)):
                assert np.array_equal(a.row_mask(0, 0, 3001), b.row_mask(0, 0, 3001))
                assert a.count() == b.count()
            for (ta, va), (tb, vb) in zip(agd.MLUtils.kFold(ds, 3, seed=4), agd.MLUtils.kFold(p, 3, seed=4)):
                assert np.array_equal(va.row_mask(0, 0, 3001), vb.row_mask(0, 0, 3001))
        finally:
            p.close()
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
@pytest.mark.parametrize("d,k", [(1, 5), (100, 300), (1500, 64)])
def test_csr(agd, ctx, store, d, k):
    rng = np.random.default_rng(d + k)
    n = 1201
    nnz = rng.integers(0, min(d, 40) + 1, size=n)
    nnz[[0, 9, n - 1]] = 0                                           # empty rows
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate([np.sort(rng.choice(d, m, replace=False)) for m in nnz]).astype(np.int32)
    va = rng.standard_normal(ix.shape[0]) * 3 - 1
    va[::7] = 0.0
    r = int(np.flatnonzero(nnz >= 1)[3])                             # a row that stores one column three times
    ix = np.insert(ix, rp[r + 1], [ix[rp[r]], ix[rp[r]]])
    va = np.insert(va, rp[r + 1], [0.5, -2.25])
    rp[r + 1:] += 2
    y = rng.standard_normal(n)
    B, c = _B(rng, d, k)
    ds = ctx.parallelize_csr(y, rp, ix, va, d, store=store)
    try:
        rps, ixs, vas, ys = _stored_csr(ds, store)
        Xs = _csr_rows(rps, ixs, vas, d)
        p = ds.project(B, c)
        try:
            Y, yl = rows_of(p, "f64", k)
            check_projection(Y, Xs, B, c)
            assert np.array_equal(bits(yl), bits(ys))
        finally:
            p.close()
        view = ds.sample(False, 0.4, seed=3)
        keep = view.row_mask(0, 0, n)
        p = view.project(B, c, store="f32")
        try:
            Yv, yl = rows_of(p, "f32", k)
            assert np.array_equal(yl, ys[keep])
            assert np.array_equal(Yv.view(np.uint32), Y[keep].astype(np.float32).view(np.uint32))
        finally:
            p.close()
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_views_and_nonfinite(agd, ctx, store):
    """±inf / NaN in rows outside a view leave no trace; a NaN inside a kept row makes only that row NaN."""
    n, d, k = 2000, 130, 70
    rng = np.random.default_rng(9)
    X = _matrix(rng, n, d)
    y = rng.standard_normal(n)
    B, c = _B(rng, d, k)
    ds0 = ctx.parallelize(y, X, store=store)
    try:
        mask = ds0.sample(False, 0.5, seed=13).row_mask(0, 0, n)
    finally:
        ds0.close()
    out, kept = np.flatnonzero(~mask), np.flatnonzero(mask)
    X[out[:3], 0] = [np.inf, -np.inf, np.nan]
    X[out[3:40], 5:129] = np.nan
    X[kept[10], 17] = np.nan                                         # inside the view
    X[kept[11], 3] = np.inf
    ds = ctx.parallelize(y, X, store=store)
    try:
        view = ds.sample(False, 0.5, seed=13)
        Xs, ys = _stored_dense(ds, store)
        p = view.project(B, c)
        try:
            Y, yl = rows_of(p, "f64", k)
            assert Y.shape[0] == mask.sum()
            assert np.array_equal(bits(yl), bits(ys[mask]))
            check_projection(Y, Xs[mask][:, :d], B, c)
            assert np.all(np.isnan(Y[10]))
            fin = np.ones(Y.shape[0], bool)
            fin[[10, 11]] = False
            assert np.all(np.isfinite(Y[fin]))                       # every other row of its tile untouched
            full = ds.project(B, c)
            try:                                                     # a kept row's bits do not depend on the view
                assert np.array_equal(bits(rows_of(full, "f64", k)[0][mask][fin]), bits(Y[fin]))
            finally:
                full.close()
        finally:
            p.close()
        empty = ds.sample(False, 0.0, seed=1)
        p = empty.project(B, c)
        try:
            assert p.local_rows(0) == 0 and p.d == k and p.count() == 0
        finally:
            p.close()
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_transformed_views(agd, ctx, store):
    """StandardScaler + appendBias views: the projection of the transformed rows [s o x, 1]."""
    n, d, k = 1500, 64, 20
    rng = np.random.default_rng(12)
    X = _matrix(rng, n, d)
    X[:, 4] = 2.0                                                    # a constant column: scale 0
    ds = ctx.parallelize(np.zeros(n), X, store=store)
    try:
        Xs = _stored_dense(ds, store)[0][:, :d]
        model = agd.StandardScaler(withMean=False, withStd=True).fit(ds)
        s = np.asarray(model.factor)
        tv = agd.MLUtils.appendBias(model.transform(ds.sample(False, 0.6, seed=2)))
        keep = tv.row_mask(0, 0, n)
        B, c = _B(rng, d + 1, k)
        p = tv.project(B, c)
        try:
            P, cf = agd.physical_projection(B, c, s, True, d + 1)
            check_projection(rows_of(p, "f64", k)[0], Xs[keep], P, cf)
        finally:
            p.close()
        with pytest.raises(ValueError, match="shape"):
            tv.project(np.ones((d, k)))                              # the view is d + 1 wide
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_first_class_shard(agd, ctx, store):
    """A projected dataset is what a load of its rows gives: the same kernel, and training on it gives the bits of training on
    parallelize(labels, its rows); the source's collectives keep their bits."""
    n, d, k = 4000, 200, 64
    ds = ctx.synthetic(n, d, agd.LogisticGradient(), seed=3, store="f32")
    try:
        w = np.linspace(-0.2, 0.2, d)
        l1, g1, c1 = ds.smooth(agd.LogisticGradient(), w)
        e1 = ds.evaluate(agd.LogisticGradient(), w)
        s1 = agd.Statistics.colStats(ds)
        pc = agd.RowMatrix(ds).computePrincipalComponents(k)
        p = agd.RowMatrix(ds).multiply(pc, store=store).data
        try:
            Y, yl = p.get_rows(0, 0, n, dtype=np.uint16 if store == "bf16" else np.float32)
            Yh = agd.bf16_to_f32(Y) if store == "bf16" else Y
            q = ctx.parallelize(yl, Yh, store=store)
            try:
                assert p.kernel_name() == q.kernel_name() and p.d == q.d == k
                m1 = agd.LogisticRegressionWithAGD(numIterations=15).run(p)
                m2 = agd.LogisticRegressionWithAGD(numIterations=15).run(q)
                assert np.array_equal(bits(m1.weights), bits(m2.weights)) and m1.intercept == m2.intercept
            finally:
                q.close()
        finally:
            p.close()
        l2, g2, c2 = ds.smooth(agd.LogisticGradient(), w)
        assert l1 == l2 and c1 == c2 and np.array_equal(bits(g1), bits(g2))
        e2 = ds.evaluate(agd.LogisticGradient(), w)
        assert np.array_equal(bits(list(e1.__dict__.values())), bits(list(e2.__dict__.values())))
        s2 = agd.Statistics.colStats(ds)
        assert np.array_equal(bits(s1.dev2), bits(s2.dev2)) and np.array_equal(bits(s1.sum), bits(s2.sum))
    finally:
        ds.close()


@pytest.mark.gpu
def test_compute_svd(agd, ctx):
    rng = np.random.default_rng(11)
    n, d, k = 3000, 24, 5
    Q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    Ur, _ = np.linalg.qr(rng.standard_normal((n, d)))
    sv = np.concatenate([[40.0, 30.0, 20.0, 15.0, 10.0], np.linspace(5.0, 1.0, d - 5)])
    A = (Ur * sv) @ Q.T
    ds = ctx.parallelize(np.arange(n, dtype=np.float64), A, store="f64")
    try:
        mat = agd.RowMatrix(ds)
        svd = mat.computeSVD(k, computeU=True)
        _, sr, vt = np.linalg.svd(A)
        np.testing.assert_allclose(svd.s, sr[:k], rtol=1e-10)
        for i in range(k):
            assert abs(svd.V[:, i] @ vt[i]) >= 1 - 1e-9
            assert svd.V[np.argmax(np.abs(svd.V[:, i])), i] > 0
        Ud = svd.U.data
        try:
            assert Ud.local_rows(0) == n and svd.U.numCols() == k
            assert np.array_equal(Ud.get_labels(0, 0, n), np.arange(n, dtype=np.float64))
            G = agd.RowMatrix(Ud).computeGramianMatrix()
            tol = 64 * (n + d) * U * (svd.s[0] / svd.s[-1]) ** 2
            assert np.abs(G - np.eye(k)).max() <= tol, (np.abs(G - np.eye(k)).max(), tol)
        finally:
            Ud.close()
        nou = mat.computeSVD(d, rCond=0.3)                          # keeps sigma >= 12: four of them
        assert nou.U is None and nou.s.shape == (4,) and nou.V.shape == (d, 4)
        for bad in (0, d + 1):
            with pytest.raises(ValueError, match="out of range"):
                mat.computeSVD(bad)
    finally:
        ds.close()


@pytest.mark.gpu
def test_errors(agd, ctx):
    import ctypes as C
    N = agd._native
    X = np.arange(40.0).reshape(10, 4)
    ds = ctx.parallelize(np.zeros(10), X, store="f32")
    other = ctx.parallelize(np.ones(3), np.ones((3, 2)), store="f64")
    try:
        for bad in (np.ones((3, 2)), np.ones((4, 0)), np.full((4, 2), np.nan)):
            with pytest.raises(ValueError):
                agd.RowMatrix(ds).multiply(bad)
        with pytest.raises(ValueError):
            ds.project(np.ones((4, 2)), offset=np.array([0.0, np.inf]))
        B = np.ones((4, 2))
        ptr = B.ctypes.data_as(C.c_void_p)
        rc = N.lib().agd_project(ds.h, ptr, 2, None, other.h, N.F64)  # a destination that holds rows is refused, untouched
        assert rc != 0 and b"not empty" in N.lib().agd_last_error(ds.h)
        assert other.local_rows(0) == 3 and np.array_equal(other.get_rows(0, 0, 3, np.float64)[0], np.ones((3, 2)))
        fresh = agd.DeviceDataset(ctx)
        try:
            Bn = B.copy()
            Bn[2, 1] = np.inf
            rc = N.lib().agd_project(ds.h, Bn.ctypes.data_as(C.c_void_p), 2, None, fresh.h, N.F64)
            assert rc != 0 and b"not finite" in N.lib().agd_last_error(ds.h)
            assert N.lib().agd_project(ds.h, ptr, 0, None, fresh.h, N.F64) != 0
            assert fresh.local_rows(0) == 0 and fresh.d == 0                # left empty
            assert N.lib().agd_project(ds.h, ptr, 2, None, fresh.h, N.F64) == 0   # and still usable
            assert np.array_equal(fresh.get_rows(0, 0, 10, np.float64)[0], X @ B)
        finally:
            fresh.close()
    finally:
        other.close()
        ds.close()
