"""BinaryClassificationMetrics on the device (agd_binary_curve, csrc/rank.cu and the key form of csrc/score.cu).

The curve (descending margins, cumulative tp / fp) must equal, bit for bit, the numpy restatement (tests/binmetrics_reference.py)
built from agd_margins output of the same rows; the areas must agree with an fsum trapezoid reference and with the Mann-Whitney
U statistic to 1e-12."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import binmetrics_reference as R  # noqa: E402


def _rows(ds):
    """Margins-independent: the labels of the view's rows on device 0, in the order DeviceDataset.margins uses."""
    n = ds.local_rows(0)
    if ds.kernel_name(0).startswith("k1_csr"):
        y = ds.get_csr_rows(0, 0, n, 1 << 22)[3]
    else:
        y = ds.get_labels(0, 0, n)
    return y[ds.row_mask(0, 0, n)] if ds.is_view and ds._preds else y


def check(ds, w, b=0.0, expect_nan=None):
    """agd_binary_curve of (w, b) on ds against the reference from ds.margins; returns (summary, K)."""
    summary, m, tp, fp = ds.binary_curve(w, b)
    ref_m = ds.margins(w, b)
    y = _rows(ds)
    rm, rtp, rfp, rnan = R.curve(ref_m, y)
    assert np.array_equal(m.view(np.uint64), rm.view(np.uint64))
    assert np.array_equal(tp, rtp) and np.array_equal(fp, rfp)
    P, N = (int(rtp[-1]), int(rfp[-1])) if len(rtp) else (0, 0)
    assert summary[0] == P and summary[1] == N and summary[2] == rnan
    if expect_nan is not None:
        assert rnan == expect_nan
    au, ap = R.areas(rtp, rfp)
    for got, ref in ((summary[3], au), (summary[4], ap)):
        if math.isnan(ref):
            assert math.isnan(got)
        else:
            assert abs(got - ref) <= 1e-12 * abs(ref), (got, ref)
    if P > 0 and N > 0 and not np.any(np.isinf(ref_m)):
        from scipy.stats import mannwhitneyu
        keep = ~np.isnan(ref_m)
        pos, neg = ref_m[keep][y[keep] > 0.5], ref_m[keep][y[keep] <= 0.5]
        u = mannwhitneyu(pos, neg).statistic / (len(pos) * len(neg))
        assert abs(summary[3] - u) <= 1e-12 * u, (summary[3], u)
    again = ds.binary_curve(w, b)
    assert np.array_equal(again[0].view(np.uint64), summary.view(np.uint64))
    assert np.array_equal(again[1].view(np.uint64), m.view(np.uint64))
    return summary, len(m)


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 3, 100, 1024, 4096])
def test_dense_curve(ctx, store, d):
    rng = np.random.default_rng(d)
    n = 37 if d >= 4096 else 5003
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = (rng.random(n) < 0.3).astype(np.float64)
    ds = ctx.parallelize(y, X, store=store)
    w = rng.standard_normal(d) * 0.1
    check(ds, w, 0.25)
    ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_csr_curve(ctx, store):
    rng = np.random.default_rng(11)
    n, d = 4001, 300
    nnz = rng.integers(0, 9, n)
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate([np.sort(rng.choice(d, k, replace=False)) for k in nnz]).astype(np.int32)
    va = rng.standard_normal(rp[-1])
    y = (rng.random(n) < 0.5).astype(np.float64)
    ds = ctx.parallelize_csr(y, rp, ix, va, d, store=store)
    check(ds, rng.standard_normal(d), -0.5)
    ds.close()


@pytest.mark.gpu
def test_generated_and_appended(agd, ctx):
    g = ctx.synthetic(20000, 64, agd.LogisticGradient(), seed=7, store="f32")
    check(g, np.random.default_rng(1).standard_normal(64))
    g.close()
    rng = np.random.default_rng(2)
    ds = ctx.parallelize((rng.random(300) < 0.5).astype(np.float64), rng.standard_normal((300, 17)), store="f64")
    ds.load_dense((rng.random(501) < 0.5).astype(np.float64), rng.standard_normal((501, 17)), store="f64")
    check(ds, rng.standard_normal(17), 0.1)
    ds.close()


@pytest.mark.gpu
def test_heavy_ties_and_infinite_margins(ctx):
    rng = np.random.default_rng(4)
    n, d = 6007, 5
    X = rng.integers(-2, 3, (n, d)).astype(np.float64)
    X[::97, 0] = np.inf
    X[1::89, 0] = -np.inf
    y = (rng.random(n) < 0.5).astype(np.float64)
    ds = ctx.parallelize(y, X, store="f64")
    _, K = check(ds, np.array([1.0, -1.0, 2.0, 0.0, 1.0]), 0.0, expect_nan=0)
    assert K < 40
    ds.close()


@pytest.mark.gpu
def test_nan_margins_counted(agd, ctx):
    rng = np.random.default_rng(6)
    n, d = 3001, 4
    X = rng.standard_normal((n, d))
    X[::50, 1] = np.nan
    X[3::70, 3] = np.inf        # inf * 0 = NaN
    y = (rng.random(n) < 0.5).astype(np.float64)
    ds = ctx.parallelize(y, X, store="f64")
    w = np.array([0.3, 1.0, -0.2, 0.0])
    expect = int(np.sum(np.isnan(X[:, 1]) | np.isinf(X[:, 3])))
    check(ds, w, 0.0, expect_nan=expect)
    with pytest.raises(ValueError, match="NaN"):
        agd.BinaryClassificationMetrics(agd.SVMModel(w, 0.0), ds)
    ds.close()


@pytest.mark.gpu
def test_views_and_excluded_nonfinite_rows(agd, ctx):
    rng = np.random.default_rng(8)
    n, d = 8000, 12
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[::13, 2] = np.nan
    X[5::17, 4] = np.inf
    y = (rng.random(n) < 0.4).astype(np.float64)
    ds = ctx.parallelize(y, X, store="f32")
    w = rng.standard_normal(d)
    bad = np.isnan(X[:, 2])        # the inf rows score +-inf (w[4] != 0)
    for v in ds.randomSplit([0.7, 0.3], seed=3):
        mask = v.row_mask(0, 0, n)
        check(v, w, 0.0, expect_nan=int(np.sum(bad & mask)))
    for tr, va in agd.MLUtils.kFold(ds, 3, seed=5):
        check(tr, w)
        check(va, w)
    empty = ds.sample(False, 0.0)
    s, K = check(empty, w)
    assert K == 0 and s[0] == 0 and s[1] == 0 and math.isnan(s[3]) and math.isnan(s[4])
    ds.close()


@pytest.mark.gpu
def test_scaled_bias_views_and_models(agd, ctx):
    rng = np.random.default_rng(10)
    n, d = 5000, 20
    X = (rng.standard_normal((n, d)) * rng.uniform(0.1, 10, d)).astype(np.float32)
    y = (X[:, 0] + rng.standard_normal(n) > 0).astype(np.float64)
    ds = ctx.parallelize(y, X, store="f32")
    train, test = ds.randomSplit([0.8, 0.2], seed=1)
    sc = agd.StandardScaler().fit(train)
    tv = agd.MLUtils.appendBias(sc.transform(test))
    w = rng.standard_normal(d + 1)
    check(tv, w, 0.0)
    model = agd.LogisticRegressionWithAGD(numIterations=20).run(agd.MLUtils.appendBias(sc.transform(train)))
    bm = model.binaryMetrics(tv)
    s, m, tp, fp = tv.binary_curve(model.weights, model.intercept)
    assert bm.areaUnderROC() == s[3] and bm.areaUnderPR() == s[4] and 0.5 < bm.areaUnderROC() <= 1.0
    np.testing.assert_array_equal(bm.thresholds(), 1.0 / (1.0 + np.exp(-m)))
    svm = agd.SVMModel(model.weights, model.intercept)
    np.testing.assert_array_equal(svm.binaryMetrics(tv).thresholds(), m)
    binned = model.binaryMetrics(tv, numBins=10)
    assert binned.thresholds().shape[0] <= len(m) // (len(m) // 10) + 1
    ds.close()


@pytest.mark.gpu
def test_capacity_smaller_than_curve(ctx):
    import ctypes as C
    from spark_agd_b200 import _native as N
    rng = np.random.default_rng(12)
    ds = ctx.parallelize((rng.random(700) < 0.5).astype(np.float64), rng.standard_normal((700, 3)), store="f64")
    w = np.array([1.0, 2.0, 3.0])
    full = ds.binary_curve(w)
    K = len(full[1])
    m = np.full(K, -7.0)
    tp = np.full(K, -7, dtype=np.int64)
    fp = np.full(K, -7, dtype=np.int64)
    out = np.empty(N.BIN_N)
    k = C.c_int64()
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    N.check(N.lib().agd_binary_curve(ds.h, p(w), 0.0, K - 1, p(m), p(tp), p(fp), C.byref(k), p(out)), ds.h)
    assert k.value == K and np.all(m == -7.0) and np.all(tp == -7) and np.all(fp == -7)
    assert np.array_equal(out.view(np.uint64), full[0].view(np.uint64))
    ds.close()


def _sort_case(ctx, x, y):
    """d = 1 fp64 rows, w = 1: every margin is the feature itself (fma(x, 1, 0) + 0), so the keys are chosen directly."""
    ds = ctx.parallelize(y, x.reshape(-1, 1), store="f64")
    out = check(ds, np.array([1.0]), 0.0)
    ds.close()
    return out


@pytest.mark.gpu
def test_sort_adversarial_keys(ctx):
    rng = np.random.default_rng(13)
    # one row, and 2 rows
    _sort_case(ctx, np.array([0.5]), np.array([1.0]))
    _sort_case(ctx, np.array([0.5, 0.25]), np.array([0.0, 1.0]))
    # every key equal (no pass runs), sizes off the tile
    for n in (2047, 2049, 10001):
        _, K = _sort_case(ctx, np.full(n, 1.5), (rng.random(n) < 0.5).astype(np.float64))
        assert K == 1
    # keys differing only in the lowest byte: consecutive doubles
    x = 1.0 + np.arange(255) * np.finfo(np.float64).eps
    rng.shuffle(x)
    _, K = _sort_case(ctx, np.tile(x, 20), (rng.random(255 * 20) < 0.5).astype(np.float64))
    assert K == 255
    # keys differing only in the highest byte: sign and the top exponent bits (2^(16 j), low exponent bits fixed)
    x = 2.0 ** (np.arange(-60, 61) * 16.0)
    k = R.margin_key(x)
    assert np.all((k & np.uint64((1 << 56) - 1)) == (k[0] & np.uint64((1 << 56) - 1)))
    rng.shuffle(x)
    _sort_case(ctx, np.tile(x, 30), (rng.random(x.shape[0] * 30) < 0.5).astype(np.float64))
    # many distinct keys over several tiles
    _sort_case(ctx, rng.standard_normal(100003) * 1e3, (rng.random(100003) < 0.5).astype(np.float64))
