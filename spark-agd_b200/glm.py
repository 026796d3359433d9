"""Callers of the Optimizer interface (SURVEY.md 8(f).4): the GeneralizedLinearAlgorithm.run recipe of
spark-mllib 1.3.0 restated over this package's optimizer, so that
`LogisticRegressionWithAGD().run(sc, labels, X)` reads like `new LogisticRegressionWithSGD().run(rdd)`.

What run() does, following GeneralizedLinearAlgorithm.run [mllib-1.3.0]:
  * useFeatureScaling: features are divided by their sample standard deviation (StandardScaler(withStd = true,
    withMean = false), unbiased variance; a zero-variance column is left as is -- multiplied by 0 upstream, i.e. dropped);
  * addIntercept: MLUtils.appendBias appends a constant 1.0 as the LAST feature; the intercept is the last weight;
  * the optimizer runs from zero initial weights; weights are mapped back to the original feature scale.
The transformed rows are what gets pinned in HBM; the optimizer itself is untouched.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .optimization import (AcceleratedGradientDescent, Context, DeviceDataset, Evaluation, HingeGradient,
                           LeastSquaresGradient, LogisticGradient, SimpleUpdater, SquaredL2Updater)


@dataclass
class GeneralizedLinearModel:
    weights: np.ndarray
    intercept: float
    loss = None    # the Gradient whose loss evaluate() reports; the concrete models below name theirs

    def margin(self, X) -> np.ndarray:
        """x . weights + intercept per row; X is a host matrix or a DeviceDataset (scored where it is resident)."""
        if isinstance(X, DeviceDataset):
            return X.margins(self.weights, self.intercept)
        return np.asarray(X, dtype=np.float64) @ self.weights + self.intercept

    def evaluate(self, data: DeviceDataset) -> Evaluation:
        """The model's loss, confusion counts (at its threshold) and error moments over every shard of `data`'s world
        (collective)."""
        if self.loss is None:
            raise TypeError(f"{type(self).__name__} names no loss: evaluate() needs a model class with a `loss` Gradient "
                            "(LogisticRegressionModel, SVMModel, LinearRegressionModel)")
        return data.evaluate(self.loss, self.weights, self.intercept, self._eval_threshold())

    def _eval_threshold(self) -> float:
        return 0.5


class _ThresholdModel(GeneralizedLinearModel):
    """setThreshold / clearThreshold of the binary classification models (mllib 1.3.0): with the threshold cleared,
    predict returns the raw score.  Until set, the class default applies."""

    def setThreshold(self, threshold: float):
        self.threshold = float(threshold)
        return self

    def clearThreshold(self):
        self.threshold = None
        return self

    def getThreshold(self):
        return self.threshold

    def score(self, X) -> np.ndarray:
        raise NotImplementedError

    def predict(self, X) -> np.ndarray:
        score = self.score(X)
        if self.threshold is None:
            return score
        return (score > self.threshold).astype(np.float64)

    def binaryMetrics(self, data: DeviceDataset, numBins: int = 0):
        """BinaryClassificationMetrics of this model over every shard of `data` (a DeviceDataset or view; collective)."""
        from .evaluation import BinaryClassificationMetrics
        return BinaryClassificationMetrics(self, data, numBins)

    def _eval_threshold(self) -> float:
        # the confusion counts need a cut even when predict returns raw scores: the class default then
        return type(self).threshold if self.threshold is None else self.threshold


class LogisticRegressionModel(_ThresholdModel):
    threshold = 0.5
    loss = LogisticGradient()

    def score(self, X) -> np.ndarray:
        return 1.0 / (1.0 + np.exp(-self.margin(X)))


class SVMModel(_ThresholdModel):
    threshold = 0.0
    loss = HingeGradient()

    def score(self, X) -> np.ndarray:
        return self.margin(X)


class LinearRegressionModel(GeneralizedLinearModel):
    loss = LeastSquaresGradient()

    def predict(self, X) -> np.ndarray:
        return self.margin(X)


def append_bias(X: np.ndarray) -> np.ndarray:
    """MLUtils.appendBias: a constant 1.0 as the last feature."""
    return np.concatenate([X, np.ones((X.shape[0], 1), dtype=X.dtype)], axis=1)


def column_std(X: np.ndarray) -> np.ndarray:
    """StandardScaler(withStd = true).fit: unbiased sample standard deviation per column (fp64)."""
    Xd = np.asarray(X, dtype=np.float64)
    n = Xd.shape[0]
    if n < 2:
        return np.zeros(Xd.shape[1])
    return np.sqrt(Xd.var(axis=0, ddof=1))


class GeneralizedLinearAlgorithm:
    """Holds an Optimizer (here: AcceleratedGradientDescent) plus the intercept / scaling switches."""
    model_class = GeneralizedLinearModel

    def __init__(self, optimizer: AcceleratedGradientDescent):
        self.optimizer = optimizer
        self.addIntercept = False
        self.useFeatureScaling = False
        self.store = "f64"

    def setIntercept(self, addIntercept: bool):
        self.addIntercept = addIntercept
        return self

    def setFeatureScaling(self, useFeatureScaling: bool):
        self.useFeatureScaling = useFeatureScaling
        return self

    def prepare(self, X):
        """The host-side part of run(): returns (X_transformed, scale) with scale = 1/std per original column."""
        X = np.asarray(X)
        if X.dtype not in (np.float32, np.float64):
            X = X.astype(np.float64)
        d = X.shape[1]
        scale = np.ones(d)
        if self.useFeatureScaling:
            std = column_std(X)
            scale = np.where(std != 0.0, 1.0 / np.where(std != 0.0, std, 1.0), 0.0)
            X = (X.astype(np.float64) * scale).astype(X.dtype)
        if self.addIntercept:
            X = append_bias(X)
        return X, scale

    def run(self, sc, *args, **kwargs):
        """Two forms:
          run(sc, labels, X, initialWeights=None)  pins the transformed host rows on the context's GPUs and trains on them;
          run(data, initialWeights=None)           trains on a DeviceDataset where it is resident (e.g. MLUtils.loadLibSVMFile).
        The second form takes nothing but the initial weights (positionally or by that name)."""
        if isinstance(sc, DeviceDataset):
            if len(args) + len(kwargs) > 1 or set(kwargs) - {"initialWeights"}:
                raise TypeError("run(data[, initialWeights]): a DeviceDataset already holds the labels and the rows; "
                                "only the initial weights may follow it")
            return self._run_resident(sc, *args, **kwargs)
        return self._run_host(sc, *args, **kwargs)

    def _run_host(self, sc: Context, labels, X, initialWeights=None):
        Xt, scale = self.prepare(X)
        d = np.asarray(X).shape[1]
        # GeneralizedLinearAlgorithm.run [mllib-1.3.0]: initialWeights default to zeros(numFeatures), and with addIntercept
        # the optimizer starts from appendBias(initialWeights) -- i.e. the initial INTERCEPT is 1.0, not 0.0
        w0 = np.zeros(d) if initialWeights is None else np.asarray(initialWeights, dtype=np.float64)
        if w0.ndim != 1 or w0.shape[0] != d:
            raise ValueError(f"initialWeights has size {w0.shape}, data has {d} features")
        if self.addIntercept:
            w0 = np.concatenate([w0, [1.0]])
        data = sc.parallelize(labels, Xt, store=self.store).cache()
        try:
            w = self.optimizer.optimize(data, w0)
        finally:
            data.close()
        intercept = float(w[-1]) if self.addIntercept else 0.0
        weights = np.array(w[:d], dtype=np.float64)
        if self.useFeatureScaling:
            weights = weights * scale          # back to the original feature scale
        return self.model_class(weights, intercept)

    def _run_resident(self, data: DeviceDataset, initialWeights=None):
        # both switches rewrite every row (appendBias / StandardScaler); the resident shard is used as it is
        if self.addIntercept:
            raise ValueError("run(DeviceDataset) cannot add an intercept: it needs a copy of the resident shard with a "
                             "column of ones appended; train from host rows (run(sc, labels, X)) instead, or train on "
                             "the view MLUtils.appendBias(data), whose last weight is the intercept")
        if self.useFeatureScaling:
            raise ValueError("run(DeviceDataset) cannot scale features: it needs a rescaled copy of the resident shard; "
                             "train from host rows (run(sc, labels, X)) instead, or train on the view "
                             "StandardScaler().fit(data).transform(data)")
        d = data.d
        w0 = np.zeros(d) if initialWeights is None else np.asarray(initialWeights, dtype=np.float64)
        if w0.ndim != 1 or w0.shape[0] != d:
            raise ValueError(f"initialWeights has size {w0.shape}, data has {d} features")
        w = self.optimizer.optimize(data, w0)
        return self.model_class(np.array(w, dtype=np.float64), 0.0)


class LogisticRegressionWithAGD(GeneralizedLinearAlgorithm):
    """LogisticRegressionWithSGD's shape with the accelerated optimizer (binary labels in {0, 1})."""
    model_class = LogisticRegressionModel

    def __init__(self, numIterations: int = 100, regParam: float = 0.0, convergenceTol: float = 1e-4):
        super().__init__(AcceleratedGradientDescent(LogisticGradient(), SquaredL2Updater())
                         .setNumIterations(numIterations).setRegParam(regParam).setConvergenceTol(convergenceTol))


class SVMWithAGD(GeneralizedLinearAlgorithm):
    model_class = SVMModel

    def __init__(self, numIterations: int = 100, regParam: float = 1.0, convergenceTol: float = 1e-4):
        super().__init__(AcceleratedGradientDescent(HingeGradient(), SquaredL2Updater())
                         .setNumIterations(numIterations).setRegParam(regParam).setConvergenceTol(convergenceTol))


class LinearRegressionWithAGD(GeneralizedLinearAlgorithm):
    model_class = LinearRegressionModel

    def __init__(self, numIterations: int = 100, convergenceTol: float = 1e-4):
        super().__init__(AcceleratedGradientDescent(LeastSquaresGradient(), SimpleUpdater())
                         .setNumIterations(numIterations).setConvergenceTol(convergenceTol))
