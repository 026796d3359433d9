"""org.apache.spark.mllib.classification.NaiveBayes / NaiveBayesModel [mllib-1.3.0] (multinomial) on the resident shards (as
recalled), over a DeviceDataset or any view of it, dense or CSR.

  model = NaiveBayes.train(data, lambda_=1.0)
  model.labels, model.pi, model.theta   # C, C and C x D
  model.predict(data)                   # each row's label, rank-local, in margins' order

Every pass over the rows runs on the device: the distinct labels and their counts (agd_label_classes), the per-label feature sums
(agd_class_sums) and the argmax of pi_c + theta_c . z (agd_linear_argmax).  The host computes the logarithms from the C (D + 1)
sums, as MLlib's driver does.  Deviations from MLlib:
  * labels are sorted ascending (MLlib keeps collect() order): this changes only which label wins an exact tie;
  * labels are compared by value: -0.0 is read as 0.0;
  * a NaN label in the data raises ValueError, and so does an empty view;
  * lambda must be finite and >= 0;
  * more than MAX_CLASSES (1,024) distinct labels raise ValueError.

Prediction rounding.  z . theta_c is an fp64 sum of D terms in an order of the kernel's (gamma_n = n u / (1 - n u), u = 2^-53),
plus pi_c, so a computed score s_c differs from the exact one by at most e_c = gamma_{D + 1} (|pi_c| + sum_l |z_l theta_cl|).  The
predicted class can differ from the exact argmax b only when a class a != b has s*_b - s*_a <= e_a + e_b.
"""
from __future__ import annotations

import math

import numpy as np

from . import _native as N
from .optimization import DeviceDataset

MAX_CLASSES = N.MAX_CLASSES


def naive_bayes_model(counts, sums, lambda_: float):
    """MLlib's run on the aggregate: pi_c = log(n_c + lambda) - log(N + C lambda) and theta_cl = log(S_cl + lambda) -
    log(sum_l S_cl + D lambda), the sum added in column order."""
    n = np.asarray(counts, dtype=np.float64)
    S = np.atleast_2d(np.asarray(sums, dtype=np.float64))
    C, D = S.shape
    pi = np.log(n + lambda_) - math.log(float(n.sum()) + C * lambda_)
    tot = np.cumsum(S, axis=1)[:, -1] if D else np.zeros(C)
    theta = np.log(S + lambda_) - np.log(tot + D * lambda_)[:, None]
    return pi, theta


def argmax_scores(scores) -> np.ndarray:
    """The lowest index of the largest score per row; a NaN score never wins, a row no class wins goes to index 0."""
    s = np.array(scores, dtype=np.float64, copy=True)
    s[np.isnan(s)] = -np.inf
    return np.argmax(s, axis=1) if s.shape[0] else np.zeros(0, dtype=np.int64)


def _lambda(lambda_) -> float:
    v = float(lambda_)
    if not (math.isfinite(v) and v >= 0.0):
        raise ValueError(f"lambda must be finite and >= 0, got {lambda_}")
    return v


class NaiveBayesModel:
    """NaiveBayesModel [mllib-1.3.0]: labels (C, ascending), pi (C log priors) and theta (C x D log conditional
    probabilities)."""

    def __init__(self, labels, pi, theta):
        lab = np.array(labels, dtype=np.float64, copy=True) + 0.0
        p = np.array(pi, dtype=np.float64, copy=True)
        t = np.array(theta, dtype=np.float64, copy=True)
        if lab.ndim != 1 or lab.shape[0] < 1 or p.shape != lab.shape or t.ndim != 2 or t.shape[0] != lab.shape[0]:
            raise ValueError(f"labels {lab.shape}, pi {p.shape} and theta {t.shape} do not describe C classes")
        for a in (lab, p, t):
            a.setflags(write=False)
        self.labels, self.pi, self.theta = lab, p, t

    def _device_model(self):
        for name, a in (("pi", self.pi), ("theta", self.theta)):
            bad = np.argwhere(~np.isfinite(a))
            if bad.shape[0]:
                i = tuple(int(v) for v in bad[0])
                raise ValueError(f"NaiveBayesModel: {name}{list(i)} = {a[i]} is not finite; the device scores finite models only")
        return self.theta, self.pi

    def predict(self, x):
        """The label of a host vector (a float), of the rows of a host matrix, or of this process's rows of a DeviceDataset /
        view (rank-local, in DeviceDataset.margins' order)."""
        if isinstance(x, DeviceDataset):
            W, b = self._device_model()
            return self.labels[x.linear_argmax(W, b)]
        a = np.asarray(x, dtype=np.float64)
        one = a.ndim == 1
        a = np.atleast_2d(a)
        if a.shape[1] != self.theta.shape[1]:
            raise ValueError(f"rows have {a.shape[1]} features, the model {self.theta.shape[1]}")
        with np.errstate(invalid="ignore", over="ignore"):
            idx = argmax_scores(self.pi[None, :] + a @ self.theta.T)
        out = self.labels[idx]
        return float(out[0]) if one else out


class NaiveBayes:
    """NaiveBayes [mllib-1.3.0], multinomial: NaiveBayes(lambda_).run(data) or NaiveBayes.train(data, lambda_)."""

    def __init__(self, lambda_: float = 1.0):
        self.setLambda(lambda_)

    def setLambda(self, lambda_: float):
        self.lambda_ = _lambda(lambda_)
        return self

    def getLambda(self) -> float:
        return self.lambda_

    def run(self, data: DeviceDataset) -> NaiveBayesModel:
        """Train on every row of `data` (a DeviceDataset or view; collective: every rank calls it and gets the same model, or
        the same error)."""
        labels, _, nan = data.label_classes()
        if nan:
            raise ValueError(f"NaiveBayes: {nan} rows of the data have a NaN label")
        if labels.shape[0] == 0:
            raise ValueError("NaiveBayes: the data has no rows")
        if labels.shape[0] > MAX_CLASSES:
            raise ValueError(f"NaiveBayes: {labels.shape[0]} distinct labels, more than the {MAX_CLASSES} classes it takes")
        sums, counts, negative = data.class_sums(labels)
        if negative:
            raise ValueError(f"NaiveBayes requires nonnegative feature values: {negative} entries of the data are negative "
                             "or NaN")
        pi, theta = naive_bayes_model(counts, sums, self.lambda_)
        return NaiveBayesModel(labels, pi, theta)

    @staticmethod
    def train(data: DeviceDataset, lambda_: float = 1.0) -> NaiveBayesModel:
        return NaiveBayes(lambda_).run(data)
