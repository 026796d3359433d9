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


class Statistics:
    """org.apache.spark.mllib.stat.Statistics [mllib-1.3.0] (column summaries)."""

    @staticmethod
    def colStats(data: DeviceDataset) -> MultivariateStatisticalSummary:
        """Column statistics of a DeviceDataset or view over every shard of the world (collective: every rank calls it and
        every rank gets the same bits).  A view's filter is set for this call only."""
        d = data.d
        sums = np.empty((N.COLSTAT_N, d), dtype=np.float64)
        count = C.c_double()
        data._ensure_exchange()
        with data._filtered():
            N.check(N.lib().agd_col_stats(data.h, C.byref(count), _ptr(sums)), data.h)
        return MultivariateStatisticalSummary.from_sums(count.value, sums)
