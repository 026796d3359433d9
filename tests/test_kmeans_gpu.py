"""KMeans on the resident shards: agd_kmeans_step / _assign / _costs / _sample (csrc/kmeans.cu) against numpy on the rows as
they are held (dense f64 / f32 / bf16 and CSR f32 / f64), views, transformed views, and KMeans.train end to end.

Exact design.  Features are small integers (|x| <= 7) and centres lie in 2^-10 Z with |c| <= 4, so every product, score,
distance, sum and cost is a multiple of 2^-20 far below 2^53 units: exact in fp64 in any order.  Under it the device must equal
numpy bit for bit: assignments (duplicated centres create ties, which go to the lowest index), sums, counts, cost, predict and
computeCost.

Random real data.  With u = 2^-53 and gamma_n = n u / (1 - n u), a score's cross term carries at most gamma_{D} sum_l |z_l c_l|
and ||c||^2 at most gamma_{D} ||c||^2, doubled and rounded once more, so the chosen centre a may lose to the exact best b by at
most 4 gamma_{D + 2} (|z| . |c_a| + |z| . |c_b| + ||c_a||^2 + ||c_b||^2).  A residual is a sum of D non-negative terms, so
its relative error is at most gamma_{D + 1}; the cost adds n of them (gamma_{n + D + 1})."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from view_reference import philox4x32_10  # noqa: E402

U = 2.0 ** -53
KM_STREAM = 8


def gamma(n):
    return n * U / (1 - n * U)


def km_draw(seed, grow):
    c = philox4x32_10([grow & 0xFFFFFFFF, (grow >> 32) & 0xFFFFFFFF, 0, KM_STREAM], [seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF])
    return float((((c[0] << 32) | c[1]) >> 11)) * 2.0 ** -53


def design(n, d, k, seed, dup=True):
    rng = np.random.default_rng(seed)
    X = rng.integers(-7, 8, (n, d)).astype(np.float64)
    X[rng.random((n, d)) < 0.2] = 0.0
    C = rng.integers(-4 * 1024, 4 * 1024 + 1, (k, d)) / 1024.0
    if dup and k >= 3:
        C[2] = C[1]                                   # a duplicated centre: every row it wins ties, lowest index first
    if k >= 2:
        C[0] = X[0]                                   # rows at distance 0
    return X, C


def ref_step(Z, C):
    dist = ((Z[:, None, :] - C[None, :, :]) ** 2).sum(axis=2)
    dist[np.isnan(dist)] = np.inf
    idx = np.argmin(dist, axis=1)
    sums = np.zeros_like(C)
    np.add.at(sums, idx, Z)
    counts = np.bincount(idx, minlength=C.shape[0]).astype(np.float64)
    own = ((Z - C[idx]) ** 2).sum(axis=1)
    return idx, sums, counts, own


def to_csr(X):
    rp = np.concatenate([[0], np.cumsum((X != 0).sum(axis=1))]).astype(np.int64)
    r, c = np.nonzero(X)
    return rp, c.astype(np.int32), X[r, c]


def load(ctx, X, store, y=None):
    y = np.zeros(X.shape[0]) if y is None else y
    if store.startswith("csr"):
        rp, ix, va = to_csr(X)
        return ctx.parallelize_csr(y, rp, ix, va.astype(np.float32 if store == "csr32" else np.float64), X.shape[1],
                                   store="f32" if store == "csr32" else "f64")
    return ctx.parallelize(y, X.astype(np.float32 if store != "f64" else np.float64), store=store)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def check_exact(agd, ds, Z, C):
    idx, sums, counts, own = ref_step(Z, C)
    s, cnt, cost = ds.kmeans_step(C)
    np.testing.assert_array_equal(cnt, counts)
    assert np.array_equal(bits(s), bits(sums))
    assert cost == own.sum()
    cl, dist = ds.kmeans_assign(C)
    np.testing.assert_array_equal(cl, idx)
    assert np.array_equal(bits(dist), bits(own))
    m = agd.KMeansModel(C)
    np.testing.assert_array_equal(m.predict(ds), idx)
    assert m.computeCost(ds) == own.sum()


STORES = ["f64", "f32", "bf16", "csr32", "csr64"]
SHAPES = [(1, 1), (1, 16), (17, 127), (17, 129), (1001, 300), (4099, 16), (4099, 129)]


@pytest.mark.gpu
@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("d,k", SHAPES)
def test_step_exact(agd, ctx, store, d, k):
    X, C = design(300 if d > 1000 else 700, d, k, seed=d * 1000 + k)
    ds = load(ctx, X, store)
    try:
        check_exact(agd, ds, X, C)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "csr64"])
@pytest.mark.parametrize("n,k", [(5, 16), (1, 3), (1, 130)])
def test_more_centres_than_rows(agd, ctx, store, n, k):
    X, C = design(n, 9, k, seed=n + k)
    ds = load(ctx, X, store)
    try:
        check_exact(agd, ds, X, C)
    finally:
        ds.close()


def _poisoned(X, keep):
    P = X.copy()
    out = np.nonzero(~keep)[0]
    P[out[0::3], 0] = np.inf
    P[out[1::3], -1] = -np.inf
    P[out[2::3], X.shape[1] // 2] = np.nan
    return P


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "csr64"])
def test_views_leave_no_trace(agd, ctx, store):
    X, C = design(900, 40, 20, seed=5)
    ds = load(ctx, X, store)
    try:
        views = [ds.randomSplit([0.3, 0.7], seed=9)[0], agd.MLUtils.kFold(ds, 3, seed=4)[1][0]]
        for v in views:
            keep = v.row_mask(0, 0, X.shape[0])
            P = _poisoned(X, keep)
            dp = load(ctx, P, store)
            try:
                vp = dp._view(None)
                vp._preds = v._preds
                for dv in (v, vp):
                    check_exact(agd, dv, X[keep], C)
            finally:
                dp.close()
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f64", "bf16", "csr32"])
def test_transformed_view(agd, ctx, store):
    n, d, k = 500, 24, 33
    X, _ = design(n, d, k, seed=8)
    rng = np.random.default_rng(8)
    s = 2.0 ** rng.integers(-2, 3, d)
    ds = load(ctx, X, store)
    try:
        v = agd.MLUtils.appendBias(agd.StandardScalerModel(1.0 / s).transform(ds)).sample(False, 0.8, seed=3)
        keep = v.row_mask(0, 0, n)
        Z = np.concatenate([X * s, np.ones((n, 1))], axis=1)[keep]
        C = rng.integers(-4 * 1024, 4 * 1024 + 1, (k, d + 1)) / 1024.0
        check_exact(agd, v, Z, C)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "f64"])
def test_real_data_bounds_and_repeat_bits(agd, ctx, store):
    rng = np.random.default_rng(21)
    n, d, k = 2000, 77, 37
    X = (rng.standard_normal((n, d)) * 3 + rng.standard_normal(d)).astype(np.float32)
    if store == "bf16":
        X = (((X.view(np.uint32) + np.uint32(0x8000)) >> np.uint32(16)) << np.uint32(16)).view(np.float32)
    C = X[rng.choice(n, k, replace=False)].astype(np.float64) + rng.standard_normal((k, d)) * 0.01
    ds = load(ctx, X, store)
    try:
        Z = X.astype(np.float64)
        cl, dist = ds.kmeans_assign(C)
        ex = ((Z[:, None, :].astype(np.longdouble) - C[None]) ** 2).sum(axis=2)
        best = np.argmin(ex, axis=1)
        az, ac = np.abs(Z), np.abs(C)
        cn = (C * C).sum(axis=1)
        rows = np.arange(n)
        tol = 4 * gamma(d + 2) * ((az * ac[cl]).sum(1) + (az * ac[best]).sum(1) + cn[cl] + cn[best])
        assert np.all(ex[rows, cl] - ex[rows, best] <= tol)
        np.testing.assert_allclose(dist, ex[rows, cl].astype(np.float64), rtol=gamma(d + 1), atol=0)
        s1, c1, cost1 = ds.kmeans_step(C)
        s2, c2, cost2 = ds.kmeans_step(C)
        assert np.array_equal(bits(s1), bits(s2)) and np.array_equal(c1, c2) and bits(cost1) == bits(cost2)
        np.testing.assert_array_equal(c1, np.bincount(cl, minlength=k))
        assert abs(cost1 - float(ex[rows, cl].sum())) <= gamma(n + d + 1) * float(ex[rows, cl].sum())
        sums = np.zeros_like(C)
        np.add.at(sums, cl, Z)
        np.testing.assert_allclose(s1, sums, rtol=1e-12, atol=1e-9)
        cl2, dist2 = ds.kmeans_assign(C)
        assert np.array_equal(cl, cl2) and np.array_equal(bits(dist), bits(dist2))
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "csr64"])
def test_sample_and_costs(agd, ctx, store):
    n, d = 600, 12
    X, _ = design(n, d, 4, seed=2)
    ds = load(ctx, X, store)
    try:
        v = ds.sample(False, 0.7, seed=12)
        keep = v.row_mask(0, 0, n)
        u = np.array([km_draw(99, r) for r in range(n)])
        rows, draws = v.kmeans_sample(99, 0.25, weighted=False)
        sel = keep & (u < 0.25)
        np.testing.assert_array_equal(rows, X[sel])
        np.testing.assert_array_equal(draws, u[sel])
        assert v.kmeans_sample(99, 1.0, weighted=False)[0].shape[0] == keep.sum()
        cand = X[[3, 50]] + 0.5
        _, _, _, d1 = ref_step(X, cand)
        total = v.kmeans_costs(cand, keep=False)
        assert total == d1[keep].sum()
        f = 2.0 / total
        rows, draws = v.kmeans_sample(7, f, weighted=True)
        u7 = np.array([km_draw(7, r) for r in range(n)])
        sel = keep & (u7 < f * d1)
        np.testing.assert_array_equal(rows, X[sel])
        cand2 = X[[100]] - 0.25
        _, _, _, d2 = ref_step(X, cand2)
        total2 = v.kmeans_costs(cand2, keep=True)
        assert total2 == np.minimum(d1, d2)[keep].sum()
        with pytest.raises(agd.NativeError, match="factor"):
            v.kmeans_sample(1, float("nan"), weighted=False)
    finally:
        ds.close()


def blobs(n_per, d, centres, seed, scale=0.2):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.normal(c, scale, (n_per, d)) for c in centres]), rng


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["k-means||", "random"])
@pytest.mark.parametrize("store", ["f32", "csr64"])
def test_train_recovers_blobs(agd, ctx, mode, store):
    rng = np.random.default_rng(1)
    d = 6
    k = 5 if mode == "k-means||" else 2     # k random rows of k equal blobs land in k different blobs with odds k! / k^k
    truth = rng.uniform(-20, 20, (k, d))
    X, _ = blobs(400, d, truth, seed=2)
    ds = load(ctx, X, store)
    try:
        model = agd.KMeans.train(ds, k, 20, runs=3 if mode == "random" else 1, initializationMode=mode, seed=31)
        got = model.clusterCenters
        assert got.shape == (k, d)
        dist = ((truth[:, None, :] - got[None]) ** 2).sum(2)
        assert np.all(dist.min(axis=1) < 0.05), dist.min(axis=1)
        pred = model.predict(ds)
        assert np.all(np.bincount(pred, minlength=k) == 400)
        Xs = X.astype(np.float32).astype(np.float64) if store == "f32" else X      # the rows as held
        assert model.computeCost(ds) == pytest.approx(((Xs - got[pred]) ** 2).sum(), rel=1e-12)
    finally:
        ds.close()


@pytest.mark.gpu
def test_initial_model_matches_host_loop(agd, ctx):
    from spark_agd_b200.clustering import lloyd
    from test_kmeans_host import ExactStep
    rng = np.random.default_rng(4)
    truth = rng.uniform(-10, 10, (4, 3))
    X, _ = blobs(250, 3, truth, seed=5, scale=1.5)
    start = X[[0, 1, 2, 3]]
    ds = load(ctx, X, "f64")
    try:
        model = agd.KMeans(k=4, maxIterations=15, epsilon=0.0).setInitialModel(agd.KMeansModel(start)).run(ds)
        ref, _, _ = lloyd(ExactStep(X), start, 15, 0.0)
        np.testing.assert_allclose(model.clusterCenters, ref, rtol=1e-12, atol=1e-12)
    finally:
        ds.close()


@pytest.mark.gpu
def test_errors(agd, ctx):
    X, C = design(50, 4, 3, seed=1)
    ds = load(ctx, X, "f32")
    try:
        with pytest.raises(ValueError, match="features"):
            ds.kmeans_step(np.zeros((2, 5)))
        Cn = C.copy()
        Cn[1, 2] = np.inf
        with pytest.raises(agd.NativeError, match="not finite"):
            ds.kmeans_step(Cn)
        with pytest.raises(agd.NativeError, match="keep = 1"):
            ds.kmeans_costs(C, keep=True)
        with pytest.raises(agd.NativeError, match="weighted = 1"):
            ds.kmeans_sample(1, 1.0, weighted=True)
        with pytest.raises(ValueError, match="no rows"):
            agd.KMeans.train(ds.sample(False, 0.0, seed=1), 2, 5, seed=1)
        with pytest.raises(ValueError, match="features"):
            agd.KMeans(k=3).setInitialModel(agd.KMeansModel(np.zeros((3, 7)))).run(ds)
        # collective calls after the k-means ones keep their bits
        w = np.linspace(-1, 1, 4)
        e1 = ds.evaluate(agd.LeastSquaresGradient(), w).__dict__
        ds.kmeans_step(C)
        assert ds.evaluate(agd.LeastSquaresGradient(), w).__dict__ == e1
    finally:
        ds.close()
