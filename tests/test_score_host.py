"""Host side of scoring (no GPU): the metrics Evaluation derives from the AGD_EVAL_* sums, the threshold logic of the
GLM models on host matrices, and the argument checks of run(DeviceDataset)."""
import math

import numpy as np
import pytest


def test_evaluation_derived_metrics(agd):
    N = agd._native
    assert N.EVAL_N == 11 and (N.EVAL_COUNT, N.EVAL_LOSS, N.EVAL_SUM_Y2) == (0, 1, 10)
    rng = np.random.default_rng(0)
    m = rng.standard_normal(1000)
    y = (rng.random(1000) > 0.4).astype(np.float64)
    pos = m > 0.1
    e = m - y
    sums = np.zeros(N.EVAL_N)
    sums[N.EVAL_COUNT] = len(m)
    sums[N.EVAL_LOSS] = np.sum(np.maximum(0, 1 - (2 * y - 1) * m))
    sums[N.EVAL_TP] = np.sum(pos & (y == 1))
    sums[N.EVAL_FP] = np.sum(pos & (y == 0))
    sums[N.EVAL_TN] = np.sum(~pos & (y == 0))
    sums[N.EVAL_FN] = np.sum(~pos & (y == 1))
    sums[N.EVAL_SUM_ERR], sums[N.EVAL_SUM_ERR2], sums[N.EVAL_SUM_ABS_ERR] = e.sum(), (e * e).sum(), np.abs(e).sum()
    sums[N.EVAL_SUM_Y], sums[N.EVAL_SUM_Y2] = y.sum(), (y * y).sum()
    ev = agd.Evaluation.from_sums(sums)
    assert ev.count == 1000 and ev.tp == sums[N.EVAL_TP]
    assert ev.mean_loss == pytest.approx(np.mean(np.maximum(0, 1 - (2 * y - 1) * m)), rel=1e-14)
    assert ev.accuracy == pytest.approx(np.mean(pos == (y == 1)), rel=1e-15)
    assert ev.precision == pytest.approx(np.sum(pos & (y == 1)) / np.sum(pos), rel=1e-15)
    assert ev.recall == pytest.approx(np.sum(pos & (y == 1)) / np.sum(y == 1), rel=1e-15)
    assert ev.mse == pytest.approx(np.mean(e * e), rel=1e-14)
    assert ev.rmse == pytest.approx(math.sqrt(np.mean(e * e)), rel=1e-14)
    assert ev.mae == pytest.approx(np.mean(np.abs(e)), rel=1e-14)
    r2 = 1 - np.sum(e * e) / np.sum((y - y.mean()) ** 2)
    assert ev.r2 == pytest.approx(r2, rel=1e-12)


def test_evaluation_empty_and_degenerate(agd):
    ev = agd.Evaluation.from_sums(np.zeros(11))
    for v in (ev.mean_loss, ev.accuracy, ev.precision, ev.recall, ev.mse, ev.rmse, ev.mae, ev.r2):
        assert math.isnan(v)
    # no positive prediction: precision is undefined, recall is 0
    ev = agd.Evaluation(4, 1.0, 0, 0, 2, 2, 0.0, 1.0, 1.0, 2.0, 2.0)
    assert math.isnan(ev.precision) and ev.recall == 0.0 and ev.accuracy == 0.5


def test_model_thresholds_on_host(agd):
    X = np.array([[1.0, 0.0], [0.0, 1.0], [-1.0, -1.0], [0.2, 0.1]])
    w = np.array([2.0, -1.0])
    lr = agd.LogisticRegressionModel(w, 0.1)
    m = X @ w + 0.1
    p = 1 / (1 + np.exp(-m))
    assert agd.LogisticRegressionModel.threshold == 0.5 and agd.SVMModel.threshold == 0.0
    np.testing.assert_array_equal(lr.predict(X), (p > 0.5).astype(float))
    assert lr.setThreshold(0.9) is lr and lr.getThreshold() == 0.9
    np.testing.assert_array_equal(lr.predict(X), (p > 0.9).astype(float))
    assert agd.LogisticRegressionModel.threshold == 0.5                # the class default is untouched
    np.testing.assert_array_equal(agd.LogisticRegressionModel(w, 0.1).predict(X), (p > 0.5).astype(float))
    lr.clearThreshold()
    assert lr.getThreshold() is None
    np.testing.assert_allclose(lr.predict(X), p, rtol=1e-15)
    assert lr._eval_threshold() == 0.5                                  # confusion counts fall back to the class default
    svm = agd.SVMModel(w, -0.5)
    np.testing.assert_array_equal(svm.predict(X), (X @ w - 0.5 > 0.0).astype(float))
    svm.setThreshold(1.0)
    np.testing.assert_array_equal(svm.predict(X), (X @ w - 0.5 > 1.0).astype(float))
    assert svm._eval_threshold() == 1.0
    svm.clearThreshold()
    np.testing.assert_array_equal(svm.predict(X), X @ w - 0.5)
    np.testing.assert_array_equal(agd.LinearRegressionModel(w, 0.25).predict(X), X @ w + 0.25)
    assert isinstance(agd.SVMModel.loss, agd.HingeGradient) and isinstance(agd.LogisticRegressionModel.loss, agd.LogisticGradient)


def test_run_keeps_host_form(agd):
    """run(sc, labels, X) is unchanged; a DeviceDataset with a second matrix is a usage error."""
    alg = agd.SVMWithAGD()
    ds = agd.DeviceDataset.__new__(agd.DeviceDataset)     # no handle needed: rejected before any native call
    with pytest.raises(TypeError, match="DeviceDataset"):
        alg.run(ds, np.zeros(3), np.zeros((3, 2)))


def test_run_resident_form_takes_only_initial_weights(agd):
    """run(data[, initialWeights]): the weights may follow positionally or by name; nothing else may."""
    alg = agd.SVMWithAGD()
    ds = agd.DeviceDataset.__new__(agd.DeviceDataset)
    for kwargs in ({"labels": np.zeros(3)}, {"X": np.zeros((3, 2))}, {"initialWeights": np.zeros(2), "labels": None}):
        with pytest.raises(TypeError, match="only the initial weights"):
            alg.run(ds, **kwargs)
    with pytest.raises(TypeError, match="only the initial weights"):
        alg.run(ds, np.zeros(2), initialWeights=np.zeros(2))


def test_evaluate_needs_a_named_loss(agd):
    class Custom(agd.GeneralizedLinearModel):
        pass

    ds = agd.DeviceDataset.__new__(agd.DeviceDataset)
    with pytest.raises(TypeError, match="names no loss"):
        Custom(np.zeros(2), 0.0).evaluate(ds)
