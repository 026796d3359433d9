"""NaiveBayes and MulticlassMetrics on the resident shards: agd_label_classes / agd_class_sums / agd_linear_argmax /
agd_linear_confusion (csrc/classify.cu and the k-means kernels' modes) against numpy on the rows as they are held (dense f64 /
f32 / bf16 and CSR f32 / f64), views, transformed views, and NaiveBayes.train end to end.

Exact design.  Features are small nonnegative integers (0 <= x <= 7), labels a few distinct doubles (negative, non-integer, and
0.0 stored as -0.0 in some rows), and a hand-built model has theta in 2^-10 Z with |theta| <= 4 and pi in 2^-10 Z with
|pi| <= 8.  Every class sum, count and score is then a multiple of 2^-10 far below 2^53 units: exact in fp64 in any order.
Under it the device must equal numpy bit for bit: the distinct labels and counts, the class sums, the trained pi / theta (the
same host formulas on the same sums), the predicted labels (a duplicated class creates ties, which go to the lowest index), the
confusion counts and every metric.

Real data.  With u = 2^-53 and gamma_n = n u / (1 - n u), a score pi_c + z . theta_c computed in fp64 in any order differs from
the exact one by at most e_c = gamma_{D + 1} (|pi_c| + sum_l |z_l theta_cl|), so the predicted class a may lose to the exact
best b only when s*_b - s*_a <= e_a + e_b: away from such rows the prediction must equal the longdouble argmax."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

U = 2.0 ** -53


def gamma(n):
    return n * U / (1 - n * U)


def label_values(C):
    return (np.arange(C) - C // 2) * 0.75     # 0.0 at C // 2; -0.75, -1.5, ... below it


def design(n, d, C, seed):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 8, (n, d)).astype(np.float64)
    X[rng.random((n, d)) < 0.3] = 0.0
    y = label_values(C)[rng.integers(0, C, n)]
    y[(y == 0.0) & (rng.random(n) < 0.5)] = -0.0
    theta = rng.integers(-4 * 1024, 1, (C, d)) / 1024.0
    pi = rng.integers(-8 * 1024, 1, C) / 1024.0
    if C >= 3:
        theta[2], pi[2] = theta[1], pi[1]        # a duplicated class: every row it wins is a tie, lowest index first
    return X, y, theta, pi


def to_csr(X):
    rp = np.concatenate([[0], np.cumsum((X != 0).sum(axis=1))]).astype(np.int64)
    r, c = np.nonzero(X)
    return rp, c.astype(np.int32), X[r, c]


def load(ctx, X, store, y):
    if store.startswith("csr"):
        rp, ix, va = to_csr(X)
        return ctx.parallelize_csr(y, rp, ix, va.astype(np.float32 if store == "csr32" else np.float64), X.shape[1],
                                   store="f32" if store == "csr32" else "f64")
    return ctx.parallelize(y, X.astype(np.float32 if store != "f64" else np.float64), store=store)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def ref_aggregate(Z, y):
    yn = np.asarray(y, dtype=np.float64) + 0.0
    labels, counts = np.unique(yn, return_counts=True)
    sums = np.zeros((labels.shape[0], Z.shape[1]))
    np.add.at(sums, np.searchsorted(labels, yn), Z)
    return labels, counts, sums


def metric_values(m):
    out = [m.confusionMatrix.ravel(), m.labels, [m.precision(), m.recall(), m.fMeasure(), m.weightedPrecision,
                                                  m.weightedRecall, m.weightedFMeasure(), m.weightedFMeasure(0.5),
                                                  m.weightedTruePositiveRate, m.weightedFalsePositiveRate]]
    for lab in m.labels:
        out.append([m.precision(lab), m.recall(lab), m.fMeasure(lab), m.fMeasure(lab, 2.5), m.truePositiveRate(lab),
                    m.falsePositiveRate(lab)])
    return np.concatenate([np.asarray(v, dtype=np.float64).ravel() for v in out])


def check_exact(agd, ds, Z, y, theta, pi, lam=1.0):
    from spark_agd_b200.classification import argmax_scores, naive_bayes_model
    labels, counts, sums = ref_aggregate(Z, y)
    got_l, got_c, nan = ds.label_classes()
    assert same(got_l, labels) and nan == 0
    np.testing.assert_array_equal(got_c, counts)
    s, c, neg = ds.class_sums(labels)
    assert same(s, sums) and neg == 0
    np.testing.assert_array_equal(c, counts)
    m = agd.NaiveBayes.train(ds, lambda_=lam)
    pi_ref, theta_ref = naive_bayes_model(counts, sums, lam)
    assert same(m.labels, labels) and same(m.pi, pi_ref) and same(m.theta, theta_ref)
    model = agd.NaiveBayesModel(label_values(pi.shape[0]), pi, theta)
    idx = argmax_scores(pi[None, :] + Z @ theta.T)
    np.testing.assert_array_equal(ds.linear_argmax(theta, pi), idx)
    assert same(model.predict(ds), model.labels[idx])
    host = agd.MulticlassMetrics(np.stack([model.labels[idx], y], axis=1))
    dev = agd.MulticlassMetrics(model, ds)
    assert same(metric_values(dev), metric_values(host))


STORES = ["f64", "f32", "bf16", "csr32", "csr64"]
SHAPES = [(1, 1), (3, 2), (16, 3), (127, 17), (129, 130), (300, 300), (4099, 16), (4099, 129)]


@pytest.mark.gpu
@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("d,C", SHAPES)
def test_exact(agd, ctx, store, d, C):
    X, y, theta, pi = design(300 if d > 1000 else 700, d, C, seed=d * 1000 + C)
    ds = load(ctx, X, store, y)
    try:
        check_exact(agd, ds, X, y, theta, pi)
    finally:
        ds.close()


def _poisoned(X, y, keep, seed=3):
    rng = np.random.default_rng(seed)
    P, yp = X.copy(), y.copy()
    out = np.nonzero(~keep)[0]
    for i in out:
        j = rng.integers(0, X.shape[1])
        P[i, j] = [np.inf, -np.inf, np.nan, -3.0][i % 4]
    yp[out[::3]] = np.nan
    return P, yp


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "csr64"])
def test_views_leave_no_trace(agd, ctx, store):
    X, y, theta, pi = design(900, 40, 20, seed=5)
    ds = load(ctx, X, store, y)
    try:
        views = [ds.randomSplit([0.3, 0.7], seed=9)[0], agd.MLUtils.kFold(ds, 3, seed=4)[1][0]]
        for v in views:
            keep = v.row_mask(0, 0, X.shape[0])
            P, yp = _poisoned(X, y, keep)
            for labels, msg in ((yp, "NaN label"), (y, "nonnegative")):
                dp = load(ctx, P, store, labels)
                try:
                    vp = dp._view(None)
                    vp._preds = v._preds
                    check_exact(agd, vp, X[keep], y[keep], theta, pi)
                    with pytest.raises(ValueError, match=msg):   # the same rows inside a view are refused
                        agd.NaiveBayes.train(dp)
                finally:
                    dp.close()
            check_exact(agd, v, X[keep], y[keep], theta, pi)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f64", "bf16", "csr32"])
def test_transformed_view(agd, ctx, store):
    n, d, C = 500, 24, 7
    X, y, _, _ = design(n, d, C, seed=8)
    rng = np.random.default_rng(8)
    s = 2.0 ** rng.integers(-2, 3, d)
    ds = load(ctx, X, store, y)
    try:
        v = agd.MLUtils.appendBias(agd.StandardScalerModel(1.0 / s).transform(ds)).sample(False, 0.8, seed=3)
        keep = v.row_mask(0, 0, n)
        Z = np.concatenate([X * s, np.ones((n, 1))], axis=1)[keep]
        theta = rng.integers(-4 * 1024, 1, (C, d + 1)) / 1024.0
        pi = rng.integers(-8 * 1024, 1, C) / 1024.0
        check_exact(agd, v, Z, y[keep], theta, pi, lam=0.5)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "csr64"])
def test_errors_and_empty_view(agd, ctx, store):
    X, y, theta, pi = design(200, 9, 4, seed=11)
    Xn = X.copy()
    Xn[5, 3] = -1.0
    Xn[7, 2] = np.nan
    ds = load(ctx, Xn, store, y)
    try:
        with pytest.raises(ValueError, match="2 entries"):
            agd.NaiveBayes.train(ds)
        assert ds.class_sums(np.unique(y + 0.0))[2] == 2
        e = ds.sample(False, 0.0, seed=1)
        assert e.label_classes()[0].shape[0] == 0
        with pytest.raises(ValueError, match="no rows"):
            agd.NaiveBayes.train(e)
        assert e.linear_argmax(theta, pi).shape[0] == 0
        assert agd.MulticlassMetrics(agd.NaiveBayesModel(label_values(4), pi, theta), e).confusionMatrix.shape == (0, 0)
        bad = theta.copy()
        bad[1, 4] = -np.inf                       # lambda = 0 with an empty column gives this
        with pytest.raises(ValueError, match=r"theta\[1, 4\]"):
            agd.NaiveBayesModel(label_values(4), pi, bad).predict(ds)
        with pytest.raises(agd.NativeError, match="not finite"):
            ds.linear_argmax(bad, pi)
        with pytest.raises(agd.NativeError, match="ascend"):
            ds.class_sums(np.array([1.0, 1.0]))
        with pytest.raises(agd.NativeError, match="classes"):
            ds.class_sums(np.arange(agd._native.MAX_CLASSES + 1.0))
        yn = y.copy()
        yn[3] = np.nan
        dn = load(ctx, X, store, yn)
        try:
            assert dn.label_classes()[2] == 1
            with pytest.raises(ValueError, match="1 rows of the data have a NaN label"):
                agd.NaiveBayes.train(dn)
            with pytest.raises(ValueError, match="NaN label"):
                agd.MulticlassMetrics(agd.NaiveBayesModel(label_values(4), pi, theta), dn)
        finally:
            dn.close()
    finally:
        ds.close()


def _neighbours(ds, C0, w, B, csr):
    """kmeans_step, binary_curve and project on the same handle, as bits (CSR k-means sums and cost add by RED.ADD, so
    there only the counts repeat their bits)"""
    s, c, cost = ds.kmeans_step(C0)
    summary, m, tp, fp = ds.binary_curve(w, 0.25)
    pj = ds.project(B)
    try:
        rows = pj.get_rows(0, 0, pj.local_rows(0), dtype=np.float64)[0]
    finally:
        pj.close()
    exact = (c, summary, m, rows) if csr else (s, c, [cost], summary, m, rows)
    return [bits(v).tolist() for v in exact] + [tp.tolist(), fp.tolist()]


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "csr64"])
def test_repeat_bits_and_neighbours_keep_theirs(agd, ctx, store):
    X, y, _, _ = design(3000, 64, 9, seed=14)
    rng = np.random.default_rng(14)
    ds = load(ctx, X * rng.random(X.shape), store, y)    # real-valued, nonnegative
    try:
        C0, w, B = rng.standard_normal((5, 64)), rng.standard_normal(64), rng.standard_normal((64, 3))
        csr = store.startswith("csr")
        before = _neighbours(ds, C0, w, B, csr)
        m1, m2 = agd.NaiveBayes.train(ds), agd.NaiveBayes.train(ds)
        assert same(m1.pi, m2.pi)                                   # counts are exact
        if csr:                                                     # RED.ADD sums: equal to rounding
            np.testing.assert_allclose(m1.theta, m2.theta, rtol=1e-13, atol=0)
        else:
            assert same(m1.theta, m2.theta)
        assert same(m1.predict(ds), m1.predict(ds))
        assert same(metric_values(agd.MulticlassMetrics(m1, ds)), metric_values(agd.MulticlassMetrics(m1, ds)))
        assert _neighbours(ds, C0, w, B, csr) == before
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f64", "f32", "bf16", "csr32"])
def test_trained_model_predicts_the_exact_argmax(agd, ctx, store):
    rng = np.random.default_rng(31)
    n, d, C = 4000, 50, 12
    X, y, _, _ = design(n, d, C, seed=31)
    Xr = np.round(X * rng.random(X.shape) * 64) / 64    # real-valued, nonnegative, exact in bf16 up to 8 bits
    if store == "bf16":
        Xr = X
    ds = load(ctx, Xr, store, y)
    try:
        m = agd.NaiveBayes.train(ds, lambda_=0.3)
        Z = Xr.astype(np.float32).astype(np.float64) if store in ("f32", "csr32") else Xr
        got = ds.linear_argmax(m.theta, m.pi)
        exact = m.pi.astype(np.longdouble)[None, :] + Z.astype(np.longdouble) @ m.theta.T.astype(np.longdouble)
        best = np.argmax(exact, axis=1)
        e = gamma(d + 1) * (np.abs(m.pi)[None, :] + np.abs(Z) @ np.abs(m.theta).T)
        top = exact[np.arange(n), best]
        close = ((top[:, None] - exact) <= (e + e[np.arange(n), best][:, None])) & (np.arange(C)[None, :] != best[:, None])
        clear = ~close.any(axis=1)
        assert clear.mean() > 0.9
        np.testing.assert_array_equal(got[clear], best[clear])
        assert np.all(close[~clear, got[~clear]] | (got[~clear] == best[~clear]))
        np.testing.assert_array_equal(m.predict(Z)[clear], m.labels[best[clear]])
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "csr32"])
def test_train_separates_multinomial_classes(agd, ctx, store):
    rng = np.random.default_rng(41)
    C, d, n = 6, 30, 6000
    probs = rng.dirichlet(np.full(d, 0.3), C)
    probs = 0.9 * probs + 0.1 / d
    cls = rng.integers(0, C, n)
    X = np.stack([rng.multinomial(40, probs[c]) for c in cls]).astype(np.float64)
    y = label_values(C)[cls]
    ds = load(ctx, X, store, y)
    try:
        tr, te = ds.randomSplit([0.7, 0.3], seed=5)
        m = agd.NaiveBayes.train(tr)
        mm = agd.MulticlassMetrics(m, te)
        assert mm.precision() > 0.95 and mm.weightedFMeasure() > 0.95
        np.testing.assert_allclose(np.exp(m.theta), probs, atol=0.03)
    finally:
        ds.close()
