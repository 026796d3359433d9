"""BinaryClassificationMetrics on the host: the key map, the curve algebra, the numBins grouping and the metrics derived from a
curve (spark-agd_b200/evaluation.py), against the numpy restatement in tests/binmetrics_reference.py.  No GPU."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import binmetrics_reference as R  # noqa: E402


@pytest.fixture(scope="module")
def ev():
    from spark_agd_b200 import evaluation
    return evaluation


def _special():
    tiny = np.finfo(np.float64).tiny
    den = 5e-324
    return np.array([0.0, -0.0, den, -den, 2 * den, -2 * den, tiny, -tiny, tiny - den, -(tiny - den), 1.0, -1.0,
                     np.nextafter(1.0, 2.0), np.nextafter(1.0, 0.0), np.finfo(np.float64).max, -np.finfo(np.float64).max,
                     np.inf, -np.inf])


def test_key_order_is_descending_fp64_order():
    rng = np.random.default_rng(5)
    m = np.concatenate([_special(), rng.standard_normal(2000) * 10.0 ** rng.integers(-300, 300, 2000),
                        rng.integers(-5, 5, 200).astype(np.float64)])
    k = R.margin_key(m)
    for i in range(0, m.shape[0], 7):
        a, b = m[i], m
        ka, kb = k[i], k
        assert np.array_equal(ka < kb, a > b), i
        assert np.array_equal(ka == kb, a == b), i
    assert R.margin_key(np.array([-0.0]))[0] == R.margin_key(np.array([0.0]))[0]
    back = R.margin_of_key(k)
    same = np.where(m == 0.0, 0.0, m)
    assert np.array_equal(back.view(np.uint64), same.view(np.uint64))


def test_key_of_nonnan_never_all_ones():
    assert np.all(R.margin_key(_special()) != np.uint64(0xFFFFFFFFFFFFFFFF))


def test_curve_algebra_ties():
    m = np.array([3.0, 1.0, 1.0, -0.0, 0.0, 3.0, np.nan, -2.0])
    y = np.array([1.0, 0.0, 1.0, 1.0, 0.0, 0.0, 1.0, 0.0])
    mm, tp, fp, nan = R.curve(m, y)
    assert nan == 1
    assert mm.tolist() == [3.0, 1.0, 0.0, -2.0]
    assert tp.tolist() == [1, 2, 3, 3] and fp.tolist() == [1, 2, 3, 4]
    auroc, aupr = R.areas(tp, fp)
    # ROC (0,0) (1/4,1/3) (1/2,2/3) (3/4,1) (1,1) (1,1)
    assert auroc == pytest.approx(0.5 * (0.25 * (1 / 3) + 0.25 * (1 / 3 + 2 / 3) + 0.25 * (2 / 3 + 1)) + 0.25, abs=1e-15)
    pos, neg = m[(y > 0.5) & ~np.isnan(m)], m[(y <= 0.5) & ~np.isnan(m)]
    u = sum((1.0 if p > q else 0.5 if p == q else 0.0) for p in pos for q in neg)
    assert auroc == pytest.approx(u / (len(pos) * len(neg)), abs=1e-15)
    assert aupr == pytest.approx(math.fsum([(1 / 3) * (1 + 0.5) / 2, (1 / 3) * (0.5 + 0.5) / 2, (1 / 3) * (0.5 + 0.5) / 2]),
                                 abs=1e-15)


def test_endpoints_and_degenerate_classes(ev):
    assert math.isnan(R.areas(np.array([2]), np.array([0]))[0])
    assert R.areas(np.array([2]), np.array([0]))[1] == 1.0
    assert all(math.isnan(a) for a in R.areas(np.array([0]), np.array([3])))
    assert ev.trapezoid([[0.0, 0.0], [1.0, 1.0]]) == 0.5
    assert ev.trapezoid([[0.0, 1.0]]) == 0.0


class _Fake:
    """A DeviceDataset stand-in returning a fixed curve."""

    def __init__(self, m, y):
        self.m, self.tp, self.fp, self.nan = R.curve(m, y)

    def binary_curve(self, w, intercept):
        P = int(self.tp[-1]) if len(self.tp) else 0
        N = int(self.fp[-1]) if len(self.fp) else 0
        au = R.areas(self.tp, self.fp)
        return np.array([P, N, self.nan, au[0], au[1]], dtype=np.float64), self.m, self.tp, self.fp


class _Model:
    weights = np.zeros(1)
    intercept = 0.0


def test_metrics_from_curve(ev):
    rng = np.random.default_rng(3)
    m = rng.integers(-20, 20, 500).astype(np.float64)
    y = (rng.random(500) < 0.4).astype(np.float64)
    fake = _Fake(m, y)
    bm = ev.BinaryClassificationMetrics(_Model(), fake)
    P, N = int(fake.tp[-1]), int(fake.fp[-1])
    roc = bm.roc()
    assert roc[0].tolist() == [0.0, 0.0] and roc[-1].tolist() == [1.0, 1.0] and roc[-2].tolist() == [1.0, 1.0]
    np.testing.assert_array_equal(roc[1:-1, 0], fake.fp / N)
    pr = bm.pr()
    assert pr[0].tolist() == [0.0, 1.0]
    np.testing.assert_array_equal(pr[1:, 1], fake.tp / (fake.tp + fake.fp))
    np.testing.assert_array_equal(bm.thresholds(), fake.m)
    p, r = fake.tp / (fake.tp + fake.fp), fake.tp / P
    for beta in (1.0, 0.5, 2.0):
        f = bm.fMeasureByThreshold(beta)
        b2 = beta * beta
        np.testing.assert_allclose(f[:, 1], (1 + b2) * p * r / (b2 * p + r), rtol=1e-15)
        np.testing.assert_array_equal(f[:, 0], fake.m)
    np.testing.assert_array_equal(bm.precisionByThreshold()[:, 1], p)
    np.testing.assert_array_equal(bm.recallByThreshold()[:, 1], r)
    assert bm.areaUnderROC() == R.areas(fake.tp, fake.fp)[0]
    assert abs(ev.trapezoid(roc) - bm.areaUnderROC()) < 1e-13
    assert abs(ev.trapezoid(pr) - bm.areaUnderPR()) < 1e-13


def test_logistic_thresholds_are_probabilities(ev):
    from spark_agd_b200 import LogisticRegressionModel
    fake = _Fake(np.array([2.0, -1.0, 0.5]), np.array([1.0, 0.0, 1.0]))
    bm = ev.BinaryClassificationMetrics(LogisticRegressionModel(np.zeros(1), 0.0), fake)
    np.testing.assert_array_equal(bm.thresholds(), 1.0 / (1.0 + np.exp(-fake.m)))


def test_nan_margins_raise(ev):
    with pytest.raises(ValueError, match="NaN"):
        ev.BinaryClassificationMetrics(_Model(), _Fake(np.array([1.0, np.nan]), np.array([1.0, 0.0])))


@pytest.mark.parametrize("K,bins", [(100, 10), (101, 10), (19, 10), (20, 10), (7, 3), (1000, 7)])
def test_numbins_grouping(ev, K, bins):
    s = -np.arange(K, dtype=np.float64)
    tp = np.cumsum(np.arange(K) % 3 == 0).astype(np.int64)
    fp = np.arange(1, K + 1) - tp
    bs, btp, bfp = ev.downsample(s, tp, fp, bins)
    g = K // bins
    if g < 2:
        assert np.array_equal(bs, s)
        return
    groups = [list(range(i, min(i + g, K))) for i in range(0, K, g)]
    assert bs.tolist() == [s[grp[0]] for grp in groups]
    assert btp.tolist() == [tp[grp[-1]] for grp in groups]
    assert bfp.tolist() == [fp[grp[-1]] for grp in groups]


def test_numbins_areas_from_downsampled_curve(ev):
    rng = np.random.default_rng(9)
    m = rng.standard_normal(3000)
    y = (rng.random(3000) < 0.5).astype(np.float64)
    fake = _Fake(m, y)
    bm = ev.BinaryClassificationMetrics(_Model(), fake, numBins=50)
    assert bm.thresholds().shape[0] == math.ceil(3000 / 60)
    assert bm.areaUnderROC() == ev.trapezoid(bm.roc())
    assert abs(bm.areaUnderROC() - R.areas(fake.tp, fake.fp)[0]) < 0.02
