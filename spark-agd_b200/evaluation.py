"""org.apache.spark.mllib.evaluation.BinaryClassificationMetrics [mllib-1.3.0] over the shards already in HBM.

The curve is computed on the device (agd_binary_curve): one point per distinct margin of the rows of a view, over every shard
of the world, in descending order, with exact cumulative counts of true and false positives.  This module derives MLlib's
metrics from it on the host.

Deviations from MLlib, on purpose:
  * rows are ranked by their margin m = x . w + b.  For a logistic model MLlib ranks by sigmoid(m), which is the same order
    except where distinct margins round to the same probability; the thresholds are still reported as sigmoid(m);
  * with numBins > 0 the points are grouped globally (MLlib groups within each partition): groups of distinct // numBins
    consecutive points, each taking its first (highest) score and the counts at its end;
  * a row whose margin is NaN is not ranked: the constructor raises ValueError when there is one.
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
