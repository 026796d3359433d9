"""org.apache.spark.mllib.feature [mllib-1.3.0]: StandardScaler on host arrays and on the resident shards.

  scaler = StandardScaler(withMean=False, withStd=True).fit(train)     # colStats on the device for a DeviceDataset
  model = SVMWithAGD(...).run(MLUtils.appendBias(scaler.transform(train)))

On a DeviceDataset, transform returns a view: the stored rows are never rewritten.  Training on it runs on appendBias(s o x)
through agd_set_feature_transform (the gradient kernels see the stored x, a scaled point and an intercept), scoring maps the
weights back to the stored features, and its colStats are derived from the stored features' statistics.
"""
from __future__ import annotations

import numpy as np

from .glm import column_std
from .optimization import DeviceDataset
from .stat import Statistics


class StandardScalerModel:
    """StandardScalerModel(std, withMean = false, withStd): x -> x * factor with factor_j = 1 / std_j, or 0 where std_j = 0
    (MLlib's rule; such a column is dropped).  Built by StandardScaler.fit, or from a given std."""

    def __init__(self, std, withMean: bool = False, withStd: bool = True):
        if withMean:
            raise NotImplementedError("withMean=True would densify sparse rows; only withMean=False is supported")
        std = np.array(std, dtype=np.float64, copy=True)
        if std.ndim != 1:
            raise ValueError(f"std must be a vector, got shape {std.shape}")
        std.setflags(write=False)
        self.std = std
        self.withMean = False
        self.withStd = bool(withStd)

    @property
    def factor(self) -> np.ndarray:
        """The multiplier of each feature: 1 / std, 0 where std == 0 (all ones without withStd)."""
        if not self.withStd:
            return np.ones_like(self.std)
        nz = self.std != 0.0
        return np.where(nz, 1.0 / np.where(nz, self.std, 1.0), 0.0)

    def transform(self, x):
        """The scaled features: a new array for a host matrix or vector, a view for a DeviceDataset (or view of one)."""
        if isinstance(x, DeviceDataset):
            return x._transformed(scale=self.factor) if self.withStd else x
        x = np.asarray(x, dtype=np.float64)
        if x.shape[-1] != self.std.shape[0]:
            raise ValueError(f"x has {x.shape[-1]} features, the scaler {self.std.shape[0]}")
        return x * self.factor


class StandardScaler:
    """StandardScaler(withMean = false, withStd = true) [mllib-1.3.0]: fit computes the unbiased standard deviation of every
    column (0 when there are fewer than two rows)."""

    def __init__(self, withMean: bool = False, withStd: bool = True):
        if withMean:
            raise NotImplementedError("withMean=True would densify sparse rows; only withMean=False is supported")
        self.withMean = False
        self.withStd = bool(withStd)

    def fit(self, data) -> StandardScalerModel:
        """data: a DeviceDataset or view (Statistics.colStats on the device, collective) or a host matrix."""
        if isinstance(data, DeviceDataset):
            std = np.sqrt(Statistics.colStats(data).variance)
        else:
            std = column_std(np.asarray(data))
        return StandardScalerModel(std, withMean=False, withStd=self.withStd)
