"""NaiveBayes / NaiveBayesModel / MulticlassMetrics on the host (no GPU): the argument errors, pi / theta against an
element-by-element restatement of MLlib's NaiveBayes.run, host predict's tie and NaN rules, and host MulticlassMetrics against
a restatement of MLlib's formulas (mllib 1.3.0, as recalled)."""
import math

import numpy as np
import pytest


def mllib_run(labels, counts, sums, lam):
    """NaiveBayes.run's driver loop over the aggregated (label, (n, sumTermFreqs)) pairs."""
    num_labels, num_features = len(labels), len(sums[0])
    num_documents = 0
    for n in counts:
        num_documents += int(n)
    pi_log_denom = math.log(num_documents + num_labels * lam)
    pi, theta = [], []
    for i in range(num_labels):
        total = 0.0
        for v in sums[i]:
            total += v
        theta_log_denom = math.log(total + num_features * lam)
        pi.append(math.log(int(counts[i]) + lam) - pi_log_denom)
        theta.append([math.log(sums[i][j] + lam) - theta_log_denom for j in range(num_features)])
    return np.array(pi), np.array(theta)


def test_pi_theta_match_the_restatement(agd):
    from spark_agd_b200.classification import naive_bayes_model
    rng = np.random.default_rng(3)
    for C, D, lam in [(1, 1, 1.0), (3, 7, 0.5), (10, 33, 1.0), (4, 5, 0.0), (17, 200, 2.25)]:
        counts = rng.integers(1, 1000, C).astype(np.float64)
        sums = rng.random((C, D)) * rng.integers(0, 50, (C, D))
        if lam == 0.0:
            sums += 0.5
        pi, theta = naive_bayes_model(counts, sums, lam)
        rp, rt = mllib_run(list(range(C)), counts, sums.tolist(), lam)
        np.testing.assert_allclose(pi, rp, rtol=4e-16, atol=4e-16)
        np.testing.assert_allclose(theta, rt, rtol=4e-16, atol=4e-16)


def test_lambda_and_model_errors(agd):
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="lambda"):
            agd.NaiveBayes(bad)
        with pytest.raises(ValueError, match="lambda"):
            agd.NaiveBayes().setLambda(bad)
    assert agd.NaiveBayes(0.0).getLambda() == 0.0 and agd.NaiveBayes().getLambda() == 1.0
    with pytest.raises(ValueError, match="C classes"):
        agd.NaiveBayesModel([1.0, 2.0], [0.0], [[0.0], [0.0]])
    with pytest.raises(ValueError, match="C classes"):
        agd.NaiveBayesModel([], [], np.zeros((0, 3)))
    m = agd.NaiveBayesModel([0.0, 1.0], [0.0, 0.0], [[0.0, 0.0], [0.0, 0.0]])
    with pytest.raises(ValueError, match="features"):
        m.predict(np.zeros((2, 3)))


def test_host_predict_ties_and_nan():
    import spark_agd_b200 as agd
    labels = [-2.5, -0.0, 1.25]
    theta = np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 1.0]])
    m = agd.NaiveBayesModel(labels, [0.0, 0.0, 0.0], theta)
    assert m.labels[1] == 0.0 and not np.signbit(m.labels[1])
    assert m.predict([2.0, 1.0]) == -2.5                        # classes 0 and 1 tie: the lowest index
    assert m.predict([1.0, 2.0]) == 1.25
    X = np.array([[np.nan, 0.0], [np.inf, 1.0], [np.nan, np.nan], [0.0, np.nan]])
    # a NaN feature times a 0 weight is NaN: rows 0, 2 and 3 score NaN everywhere and go to 0; row 1: +inf ties for 0 and 1
    np.testing.assert_array_equal(m.predict(X), [-2.5, -2.5, -2.5, -2.5])
    mi = agd.NaiveBayesModel(labels, [np.nan, -1.0, 2.0], theta)   # a NaN score never wins
    np.testing.assert_array_equal(mi.predict(np.zeros((2, 2))), [1.25, 1.25])
    mi = agd.NaiveBayesModel(labels, [np.nan, -np.inf, np.nan], theta)
    assert mi.predict([0.0, 0.0]) == -2.5


def mllib_metrics(pl, beta=1.0):
    """MulticlassMetrics' formulas over (prediction, label) pairs, labels by value, weighted sums in ascending label order."""
    pred = [p + 0.0 for p in pl[:, 0]]
    lab = [y + 0.0 for y in pl[:, 1]]
    label_count_by_class, tp_by_class, fp_by_class = {}, {}, {}
    for p, y in zip(pred, lab):
        label_count_by_class[y] = label_count_by_class.get(y, 0) + 1
        tp_by_class[y] = tp_by_class.get(y, 0) + (1 if p == y else 0)
        fp_by_class[p] = fp_by_class.get(p, 0) + (1 if p != y else 0)
    label_count = sum(label_count_by_class.values())
    labels = sorted(tp_by_class)

    def precision(c):
        tp, fp = tp_by_class[c], fp_by_class.get(c, 0)
        return 0.0 if tp + fp == 0 else tp / (tp + fp)

    def recall(c):
        return tp_by_class[c] / label_count_by_class[c]

    def fpr(c):   # a Scala Double division: 0 / 0 is NaN (a single label)
        den = label_count - label_count_by_class[c]
        return fp_by_class.get(c, 0) / den if den else float("nan")

    def f(c, b):
        p, r = precision(c), recall(c)
        return 0.0 if p + r == 0 else (1 + b * b) * p * r / (b * b * p + r)

    def weighted(fn):
        total = 0.0
        for c in labels:
            total += fn(c) * label_count_by_class[c] / label_count
        return total

    conf = np.zeros((len(labels), len(labels)))
    for p, y in zip(pred, lab):
        if p in labels:
            conf[labels.index(y), labels.index(p)] += 1
    out = {"labels": labels, "confusion": conf, "precision": sum(tp_by_class.values()) / label_count,
           "weightedPrecision": weighted(precision), "weightedRecall": weighted(recall),
           "weightedF": weighted(lambda c: f(c, 1.0)), "weightedFbeta": weighted(lambda c: f(c, beta)),
           "weightedFPR": weighted(fpr)}
    for c in labels:
        out[("p", c)], out[("r", c)], out[("fpr", c)] = precision(c), recall(c), fpr(c)
        out[("f", c)], out[("fb", c)] = f(c, 1.0), f(c, beta)
    return out


def same(a, b):
    return a == b or (math.isnan(a) and math.isnan(b))


CASES = {
    "never predicted and non-labels": np.array([[1.0, 1.0], [1.0, 2.0], [7.0, 2.0], [1.0, 3.0], [3.0, 3.0], [9.0, 1.0]]),
    "single class": np.array([[4.0, 4.0], [4.0, 4.0], [5.0, 4.0]]),
    "signed zero": np.array([[-0.0, 0.0], [0.0, -0.0], [0.0, 1.5], [1.5, -0.0], [1.5, 1.5]]),
    "random": np.stack([np.random.default_rng(2).integers(-3, 5, 500) * 0.5,
                        np.random.default_rng(3).integers(-3, 4, 500) * 0.5], axis=1),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("beta", [1.0, 0.5, 3.0])
def test_multiclass_metrics_match_the_formulas(agd, case, beta):
    pl = CASES[case]
    m = agd.MulticlassMetrics(pl)
    r = mllib_metrics(pl, beta)
    np.testing.assert_array_equal(m.labels, r["labels"])
    assert not np.signbit(m.labels[m.labels == 0]).any()
    np.testing.assert_array_equal(m.confusionMatrix, r["confusion"])
    assert m.precision() == m.recall() == m.fMeasure() == r["precision"]
    assert m.weightedPrecision == r["weightedPrecision"]
    assert m.weightedRecall == m.weightedTruePositiveRate == r["weightedRecall"]
    assert m.weightedFMeasure() == r["weightedF"] and m.weightedFMeasure(beta) == r["weightedFbeta"]
    assert same(m.weightedFalsePositiveRate, r["weightedFPR"])
    for c in r["labels"]:
        assert m.precision(c) == r[("p", c)] and m.recall(c) == m.truePositiveRate(c) == r[("r", c)]
        assert m.fMeasure(c) == r[("f", c)] and m.fMeasure(c, beta) == r[("fb", c)]
        assert same(m.falsePositiveRate(c), r[("fpr", c)])


def test_multiclass_metrics_errors(agd):
    with pytest.raises(ValueError, match=r"\(n, 2\)"):
        agd.MulticlassMetrics(np.zeros((3, 3)))
    with pytest.raises(ValueError, match="NaN label"):
        agd.MulticlassMetrics(np.array([[1.0, np.nan], [1.0, 1.0]]))
    m = agd.MulticlassMetrics(np.array([[1.0, 1.0], [np.nan, 2.0]]))   # a NaN prediction is a false positive of nothing
    assert m.recall(2.0) == 0.0 and m.precision(1.0) == 1.0
    with pytest.raises(ValueError, match="not one of the labels"):
        m.precision(3.0)
    with pytest.raises(TypeError):
        agd.MulticlassMetrics()
