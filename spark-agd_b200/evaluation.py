"""org.apache.spark.mllib.evaluation.BinaryClassificationMetrics and MulticlassMetrics [mllib-1.3.0] over the shards already in
HBM.

The curve is computed on the device (agd_binary_curve): one point per distinct margin of the rows of a view, over every shard
of the world, in descending order, with exact cumulative counts of true and false positives.  This module derives MLlib's
metrics from it on the host.

Deviations from MLlib, on purpose:
  * rows are ranked by their margin m = x . w + b.  For a logistic model MLlib ranks by sigmoid(m), which is the same order
    except where distinct margins round to the same probability; the thresholds are still reported as sigmoid(m);
  * with numBins > 0 the points are grouped globally (MLlib groups within each partition): groups of distinct // numBins
    consecutive points, each taking its first (highest) score and the counts at its end;
  * a row whose margin is NaN is not ranked: the constructor raises ValueError when there is one.

MulticlassMetrics follows MLlib's formulas over one confusion matrix (rows: actual labels, columns: predicted, over the distinct
actual labels, ascending) and the count of each label; on the device both come from agd_label_classes and agd_linear_confusion.
Deviations from MLlib, on purpose:
  * labels are compared by value: -0.0 is read as 0.0 (MLlib's maps key -0.0 and 0.0 apart);
  * the weighted metrics add their terms in ascending label order (MLlib: hash-map order);
  * a NaN label raises ValueError; a label that is not one of `labels` raises ValueError where MLlib raises
    NoSuchElementException.
"""
from __future__ import annotations

import numpy as np

from . import _native as N


def downsample(scores, tp, fp, numBins: int):
    """MLlib's numBins grouping of a descending curve with cumulative counts: groups of len // numBins consecutive points (no
    grouping when that is below 2), a group taking its first score and its last point's counts."""
    scores, tp, fp = np.asarray(scores), np.asarray(tp), np.asarray(fp)
    if numBins <= 0:
        return scores, tp, fp
    grouping = scores.shape[0] // int(numBins)
    if grouping < 2:
        return scores, tp, fp
    first = np.arange(0, scores.shape[0], grouping)
    last = np.minimum(first + grouping, scores.shape[0]) - 1
    return scores[first], tp[last], fp[last]


def trapezoid(points) -> float:
    """AreaUnderCurve.of: the trapezoid sum (x1 - x0) (y0 + y1) / 2 over consecutive points, added in order."""
    p = np.asarray(points, dtype=np.float64)
    if p.shape[0] < 2:
        return 0.0
    seg = (p[1:, 0] - p[:-1, 0]) * (p[1:, 1] + p[:-1, 1]) / 2.0
    total = 0.0
    for v in seg.tolist():
        total += v
    return total


class BinaryClassificationMetrics:
    """BinaryClassificationMetrics(model, data, numBins=0): the ROC and PR curves of a binary model (LogisticRegressionModel,
    SVMModel, or any GeneralizedLinearModel) over the rows of a DeviceDataset or view, every shard of the world (collective:
    every rank constructs it with the same arguments, and every rank gets the same bits).  On a transformed view the model is
    one of the view's features, mapped to the stored ones the way scoring maps it."""

    def __init__(self, model, data, numBins: int = 0):
        numBins = int(numBins)
        if numBins < 0:
            raise ValueError(f"numBins must be >= 0, got {numBins}")
        summary, m, tp, fp = data.binary_curve(model.weights, model.intercept)
        nan = int(summary[N.BIN_NAN])
        if nan:
            raise ValueError(f"{nan} rows of the data have a NaN margin under this model and cannot be ranked")
        self.numBins = numBins
        self.numPositives = int(summary[N.BIN_POS])
        self.numNegatives = int(summary[N.BIN_NEG])
        self._margins, self._tp, self._fp = downsample(m, tp, fp, numBins)
        self._logistic = type(model).__name__ == "LogisticRegressionModel"
        if numBins > 0:
            self._auroc, self._aupr = trapezoid(self.roc()), trapezoid(self.pr())
        else:
            self._auroc, self._aupr = float(summary[N.BIN_AUROC]), float(summary[N.BIN_AUPR])

    def thresholds(self) -> np.ndarray:
        """The score of every point, descending: sigmoid(margin) for a logistic model, the margin otherwise."""
        if self._logistic:
            return 1.0 / (1.0 + np.exp(-self._margins))
        return self._margins.copy()

    @staticmethod
    def _ratio(a, b) -> np.ndarray:
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.asarray(a, dtype=np.float64) / np.asarray(b, dtype=np.float64)

    def _recall(self) -> np.ndarray:
        return self._ratio(self._tp, self.numPositives)

    def _precision(self) -> np.ndarray:
        return self._ratio(self._tp, self._tp + self._fp)

    def roc(self) -> np.ndarray:
        """(false positive rate, recall) per point, between (0, 0) and (1, 1)."""
        pts = np.stack([self._ratio(self._fp, self.numNegatives), self._recall()], axis=1)
        return np.concatenate([[[0.0, 0.0]], pts, [[1.0, 1.0]]])

    def pr(self) -> np.ndarray:
        """(recall, precision) per point, after (0, 1)."""
        return np.concatenate([[[0.0, 1.0]], np.stack([self._recall(), self._precision()], axis=1)])

    def areaUnderROC(self) -> float:
        return self._auroc

    def areaUnderPR(self) -> float:
        return self._aupr

    def precisionByThreshold(self) -> np.ndarray:
        return np.stack([self.thresholds(), self._precision()], axis=1)

    def recallByThreshold(self) -> np.ndarray:
        return np.stack([self.thresholds(), self._recall()], axis=1)

    def fMeasureByThreshold(self, beta: float = 1.0) -> np.ndarray:
        """(1 + beta^2) p r / (beta^2 p + r) per threshold, 0 where p + r = 0."""
        b2 = float(beta) * float(beta)
        p, r = self._precision(), self._recall()
        with np.errstate(divide="ignore", invalid="ignore"):
            f = np.where(p + r == 0, 0.0, (1.0 + b2) * (p * r / (b2 * p + r)))
        return np.stack([self.thresholds(), f], axis=1)


class MulticlassMetrics:
    """MulticlassMetrics(predictionAndLabels): from a host (n, 2) array of (prediction, label) rows.
    MulticlassMetrics(model, data): from a NaiveBayesModel's predictions on the rows of a DeviceDataset or view, over every
    shard of the world (collective: every rank constructs it with the same arguments and gets the same bits).  A prediction
    that is none of the labels is a false positive of no label in `labels`, as in MLlib."""

    def __init__(self, *args):
        if len(args) == 1:
            labels, counts, confusion = self._host(args[0])
        elif len(args) == 2:
            labels, counts, confusion = self._device(*args)
        else:
            raise TypeError("MulticlassMetrics(predictionAndLabels) or MulticlassMetrics(model, data)")
        self.labels = labels
        self._count = counts.astype(np.float64)
        self._n = float(counts.sum())
        self.confusionMatrix = confusion
        self._tp = np.diagonal(confusion).copy()
        self._fp = confusion.sum(axis=0) - self._tp   # column sums of integers: exact

    @staticmethod
    def _host(predictionAndLabels):
        pl = np.asarray(predictionAndLabels, dtype=np.float64)
        if pl.ndim != 2 or pl.shape[1] != 2:
            raise ValueError(f"predictionAndLabels must be an (n, 2) array, got shape {pl.shape}")
        pred, lab = pl[:, 0] + 0.0, pl[:, 1] + 0.0
        if np.isnan(lab).any():
            raise ValueError(f"{int(np.isnan(lab).sum())} rows have a NaN label")
        labels, li, counts = np.unique(lab, return_inverse=True, return_counts=True)
        L = labels.shape[0]
        pj = np.searchsorted(labels, pred) if L else np.zeros(pred.shape[0], dtype=np.int64)
        hit = (pj < L) & (labels[np.minimum(pj, max(L - 1, 0))] == pred) if L else np.zeros(pred.shape[0], dtype=bool)
        confusion = np.zeros((L, L), dtype=np.float64)
        np.add.at(confusion, (li[hit], pj[hit]), 1.0)
        return labels, counts.astype(np.int64), confusion

    @staticmethod
    def _device(model, data):
        labels, counts, nan = data.label_classes()
        if nan:
            raise ValueError(f"{nan} rows of the data have a NaN label")
        L = labels.shape[0]
        confusion = np.zeros((L, L), dtype=np.float64)
        if L == 0:
            return labels, counts, confusion
        if L > N.MAX_CLASSES:
            raise ValueError(f"{L} distinct labels, more than the {N.MAX_CLASSES} classes MulticlassMetrics takes on the device")
        W, b = model._device_model()
        cnt = data.linear_confusion(W, b, labels)                 # (L, C) by the model's class index
        cols = np.searchsorted(labels, model.labels)
        for c in range(model.labels.shape[0]):                    # a model class that is no data label counts nowhere
            j = int(cols[c])
            if j < L and labels[j] == model.labels[c]:
                confusion[:, j] += cnt[:, c]
        return labels, counts, confusion

    def _index(self, label) -> int:
        v = float(label) + 0.0
        j = int(np.searchsorted(self.labels, v))
        if j >= self.labels.shape[0] or self.labels[j] != v:
            raise ValueError(f"{label} is not one of the labels")
        return j

    def truePositiveRate(self, label) -> float:
        return self.recall(label)

    def _fpr(self, j: int) -> float:
        with np.errstate(divide="ignore", invalid="ignore"):   # a single label: 0 / 0, NaN as in MLlib
            return self._fp[j] / np.float64(self._n - self._count[j])

    def falsePositiveRate(self, label) -> float:
        return self._fpr(self._index(label))

    def _precision(self, j: int) -> float:
        tp, fp = self._tp[j], self._fp[j]
        return 0.0 if tp + fp == 0 else tp / (tp + fp)

    def _recall(self, j: int) -> float:
        return self._tp[j] / self._count[j]

    def _f(self, j: int, beta: float) -> float:
        p, r = self._precision(j), self._recall(j)
        b2 = float(beta) * float(beta)
        return 0.0 if p + r == 0 else (1.0 + b2) * p * r / (b2 * p + r)

    def _weighted(self, metric) -> float:
        total = 0.0
        for j in range(self.labels.shape[0]):
            total += metric(j) * self._count[j] / self._n
        return total

    def precision(self, label=None) -> float:
        """precision(label), or with no label the overall precision (the fraction of rows predicted right)."""
        if label is None:
            return float(self._tp.sum()) / self._n if self._n else float("nan")
        return self._precision(self._index(label))

    def recall(self, label=None) -> float:
        if label is None:
            return self.precision()
        return self._recall(self._index(label))

    def fMeasure(self, label=None, beta: float = 1.0) -> float:
        if label is None:
            return self.precision()
        return self._f(self._index(label), beta)

    @property
    def weightedTruePositiveRate(self) -> float:
        return self.weightedRecall

    @property
    def weightedFalsePositiveRate(self) -> float:
        return self._weighted(self._fpr)

    @property
    def weightedRecall(self) -> float:
        return self._weighted(self._recall)

    @property
    def weightedPrecision(self) -> float:
        return self._weighted(self._precision)

    def weightedFMeasure(self, beta: float = 1.0) -> float:
        return self._weighted(lambda j: self._f(j, beta))
