"""org.apache.spark.mllib.stat [mllib-1.3.0]: column statistics of the resident shards.

  summary = Statistics.colStats(data)            # collective; two reads of X on the device, no host copy of X
  summary.mean, summary.variance, summary.numNonzeros, summary.max, summary.min, summary.normL1, summary.normL2

The device returns sums (agd_col_stats); the statistics are derived from them on the host, as Evaluation does for
agd_evaluate.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .optimization import DeviceDataset, _ptr


@dataclass(frozen=True)
class MultivariateStatisticalSummary:
    """MultivariateStatisticalSummary of MultivariateOnlineSummarizer (mllib 1.3.0), from the sums agd_col_stats reduces
    over the world.  Zeros count as values: explicit zeros, a CSR row's implicit zeros and zeros of dense rows.

    One deviation: a column whose every entry is NaN reports NaN as its max and min, where MLlib reports its
    Double.MinValue / Double.MaxValue sentinels."""
    n: float                 # rows
    sum: np.ndarray          # sum x
    sum_sq: np.ndarray       # sum x^2
    sum_abs: np.ndarray      # sum |x|
    nnz: np.ndarray          # entries with x != 0 (a NaN is nonzero)
    dev: np.ndarray          # sum (x - mu), mu = fl(sum / n)
    dev2: np.ndarray         # sum (x - mu)^2
    col_max: np.ndarray
    col_min: np.ndarray

    @classmethod
    def from_sums(cls, count, sums) -> "MultivariateStatisticalSummary":
        """count: rows; sums: AGD_COLSTAT_N x d (statistic-major).  An empty dataset raises ValueError, as MLlib's
        require(count > 0) does."""
        n = float(count)
        if not (n > 0):
            raise ValueError("Nothing has been added to this summarizer.")
        s = np.array(sums, dtype=np.float64, copy=True)
        if s.ndim != 2 or s.shape[0] != N.COLSTAT_N:
            raise ValueError(f"sums must be {N.COLSTAT_N} x d, got shape {s.shape}")
        s.setflags(write=False)
        return cls(n, *(s[k] for k in range(N.COLSTAT_N)))

    @property
    def count(self) -> int:
        return int(self.n)

    @property
    def mean(self) -> np.ndarray:
        return self.sum / self.n

    @property
    def variance(self) -> np.ndarray:
        """The unbiased sample variance by the corrected two-pass formula (sum (x-mu)^2 - (sum (x-mu))^2 / n) / (n - 1),
        exact to fp64 rounding also where the mean is large next to the spread; 0 when there is one row."""
        if self.n <= 1:
            return np.zeros_like(self.sum)
        return (self.dev2 - self.dev * self.dev / self.n) / (self.n - 1.0)

    @property
    def numNonzeros(self) -> np.ndarray:
        return self.nnz.copy()

    @property
    def max(self) -> np.ndarray:
        return self.col_max.copy()

    @property
    def min(self) -> np.ndarray:
        return self.col_min.copy()

    @property
    def normL1(self) -> np.ndarray:
        return self.sum_abs.copy()

    @property
    def normL2(self) -> np.ndarray:
        return np.sqrt(self.sum_sq)

    def transformed(self, scale=None, bias: bool = False) -> "MultivariateStatisticalSummary":
        """The summary of appendBias(s o x) from that of x, in O(d): sums scale by s, squares by s^2 (so mean, max, min, normL1
        and normL2 scale by |s| -- max and min swap where s < 0 -- and the variance by s^2); a column with s = 0 has no
        nonzeros.  The bias column: count rows of 1.0 (mean 1, variance 0, max = min = 1, normL1 = n, normL2 = sqrt(n))."""
        cols = [self.sum, self.sum_sq, self.sum_abs, self.nnz, self.dev, self.dev2, self.col_max, self.col_min]
        if scale is not None:
            s = np.asarray(scale, dtype=np.float64)
            neg = s < 0
            hi, lo = self.col_max * s, self.col_min * s
            cols = [self.sum * s, self.sum_sq * (s * s), self.sum_abs * np.abs(s), np.where(s != 0, self.nnz, 0.0),
                    self.dev * s, self.dev2 * (s * s), np.where(neg, lo, hi), np.where(neg, hi, lo)]
        if bias:
            n = self.n
            cols = [np.append(c, v) for c, v in zip(cols, [n, n, n, n, 0.0, 0.0, 1.0, 1.0])]
        return MultivariateStatisticalSummary.from_sums(self.n, np.stack(cols))


class Statistics:
    """org.apache.spark.mllib.stat.Statistics [mllib-1.3.0] (column summaries and correlations)."""

    @staticmethod
    def corr(data: DeviceDataset, method: str = "pearson") -> np.ndarray:
        """The d x d correlation matrix of the columns of a DeviceDataset or view (collective), derived from the covariance
        as MLlib's computeCorrelationMatrixFromCovariance does: a column with variance <= 1e-12 has NaN correlations and
        1.0 on the diagonal."""
        from .linalg import RowMatrix, correlation_from_covariance
        if method == "spearman":
            raise NotImplementedError("method='spearman' ranks every column's values over all rows: that needs a per-column "
                                      "sort of the resident rows, a different kernel; only 'pearson' is implemented")
        if method != "pearson":
            raise ValueError(f"unknown correlation method {method!r}: 'pearson' or 'spearman'")
        return correlation_from_covariance(RowMatrix(data).computeCovariance())

    @staticmethod
    def colStats(data: DeviceDataset) -> MultivariateStatisticalSummary:
        """Column statistics of a DeviceDataset or view over every shard of the world (collective: every rank calls it and
        every rank gets the same bits).  A view's filter is set for this call only.  On a transformed view the statistics
        are those of the transformed features, derived from the stored features' (MultivariateStatisticalSummary.transformed)."""
        d = data._phys_d
        sums = np.empty((N.COLSTAT_N, d), dtype=np.float64)
        count = C.c_double()
        data._ensure_exchange()
        with data._filtered():
            N.check(N.lib().agd_col_stats(data.h, C.byref(count), _ptr(sums)), data.h)
        summary = MultivariateStatisticalSummary.from_sums(count.value, sums)
        if data._scale is not None or data._bias:
            summary = summary.transformed(data._scale, data._bias)
        return summary
