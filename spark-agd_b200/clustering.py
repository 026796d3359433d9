"""org.apache.spark.mllib.clustering.KMeans / KMeansModel [mllib-1.3.0] on the resident shards (as recalled), over a DeviceDataset
or any view of it, dense or CSR.  Labels are ignored.

  model = KMeans.train(data, k=8, maxIterations=20, seed=7)
  model.clusterCenters                  # k x d
  model.predict(data)                   # each row's centre, rank-local, in margins' order
  model.computeCost(data)               # collective: the sum of squared distances to the closest centre

Every pass over the rows runs on the device (agd_kmeans_step / _costs / _sample / _assign); the host keeps what MLlib keeps on
the driver: the k centres, the k-means|| candidates and LocalKMeans.kMeansPlusPlus over them.  Deviations from MLlib:
  * "random" takes the k rows with the smallest draws under the seed: a row is never repeated (MLlib's takeSample with
    replacement can repeat one); when k exceeds the rows of the view, the rows are cycled.
  * k-means|| draws each row's number from its global row and the round's seed only (MLlib: XORShiftRandom(seed ^ (step << 16)
    ^ partition)), so the candidates do not depend on the partitioning.  The host's random stream is numpy's.
  * runs > 1 executes the runs one after another with seeds derived from `seed` and keeps the lowest cost.
  * In a multi-process world every rank must pass the same seed: a seed drawn on each rank would select different rows.
"""
from __future__ import annotations

from typing import Callable, Optional

import numpy as np

from .optimization import DeviceDataset

K_MEANS_PARALLEL = "k-means||"
RANDOM = "random"
LOCAL_MAX_ITERATIONS = 30          # LocalKMeans' Lloyd iterations on the k-means|| candidates
_MASK64 = (1 << 64) - 1


def squared_distances(points, centers) -> np.ndarray:
    """(n, k) exact squared Euclidean distances sum_l (p_l - c_l)^2, in fp64, in chunks of points."""
    p = np.asarray(points, dtype=np.float64)
    c = np.asarray(centers, dtype=np.float64)
    out = np.empty((p.shape[0], c.shape[0]), dtype=np.float64)
    step = max(1, (1 << 22) // max(1, c.shape[0] * c.shape[1]))
    for i in range(0, p.shape[0], step):
        out[i:i + step] = ((p[i:i + step, None, :] - c[None, :, :]) ** 2).sum(axis=2)
    return out


def closest(points, centers) -> np.ndarray:
    """MLlib's findClosest: the lowest index of the smallest distance; a NaN distance never wins, a point no centre wins
    goes to 0."""
    dist = squared_distances(points, centers)
    dist[np.isnan(dist)] = np.inf
    return np.argmin(dist, axis=1) if dist.shape[0] else np.zeros(0, dtype=np.int64)


def lloyd(step: Callable, centers, max_iterations: int, epsilon: float):
    """One run of MLlib's Lloyd loop from `centers`: step(centers) -> (sums, counts, cost) over every row.  A centre with rows
    moves to sum * (1 / count), one without keeps its value; the run stops when no centre moved by more than epsilon^2 in
    squared distance, or after max_iterations steps.  Returns (centers, cost, iterations), cost from the last step (that of
    the centres it started from), or of `centers` when no step ran."""
    c = np.array(centers, dtype=np.float64, copy=True)
    cost, it, converged = None, 0, False
    while it < max_iterations and not converged:
        sums, counts, cost = step(c)
        converged = True
        for j in range(c.shape[0]):
            if counts[j] != 0:
                new = sums[j] * (1.0 / counts[j])
                if float(((new - c[j]) ** 2).sum()) > epsilon * epsilon:
                    converged = False
                c[j] = new
        it += 1
    if cost is None:
        cost = step(c)[2]
    return c, cost, it


class LocalKMeans:
    """LocalKMeans [mllib-1.3.0]: weighted k-means++ seeding, then at most max_iterations weighted Lloyd iterations, on the
    host, with numpy's random stream."""

    @staticmethod
    def _pick_weighted(rng, points, weights):
        r = rng.random() * float(np.sum(weights))
        i, cur = 0, 0.0
        while i < len(points) and cur < r:
            cur += weights[i]
            i += 1
        return points[max(i - 1, 0)]

    @staticmethod
    def kMeansPlusPlus(seed: int, points, weights, k: int, maxIterations: int) -> np.ndarray:
        rng = np.random.default_rng(seed)
        pts = np.asarray(points, dtype=np.float64)
        w = np.asarray(weights, dtype=np.float64)
        n = pts.shape[0]
        centers = np.empty((k, pts.shape[1]), dtype=np.float64)
        centers[0] = LocalKMeans._pick_weighted(rng, pts, w)
        for i in range(1, k):
            cost = w * squared_distances(pts, centers[:i]).min(axis=1)
            r = rng.random() * float(np.sum(cost))
            cum, j = 0.0, 0
            while j < n and cum < r:
                cum += cost[j]
                j += 1
            centers[i] = pts[0] if j == 0 else pts[j - 1]
        old = np.full(n, -1)
        it, moved = 0, True
        while moved and it < maxIterations:
            idx = closest(pts, centers)
            sums = np.zeros_like(centers)
            counts = np.zeros(k)
            for i in range(n):
                sums[idx[i]] += w[i] * pts[i]
                counts[idx[i]] += w[i]
            moved = bool(np.any(idx != old))
            old = idx
            for j in range(k):
                if counts[j] == 0.0:
                    centers[j] = pts[rng.integers(n)]
                else:
                    centers[j] = sums[j] * (1.0 / counts[j])
            it += 1
        return centers


class KMeansModel:
    """KMeansModel [mllib-1.3.0]: clusterCenters (k x d) and k."""

    def __init__(self, clusterCenters):
        c = np.array(clusterCenters, dtype=np.float64, copy=True)
        if c.ndim != 2 or c.shape[0] < 1:
            raise ValueError(f"clusterCenters must be a non-empty (k, d) matrix, got shape {c.shape}")
        c.setflags(write=False)
        self.clusterCenters = c

    @property
    def k(self) -> int:
        return self.clusterCenters.shape[0]

    def predict(self, x):
        """The closest centre of a host vector (an int), of the rows of a host matrix, or of this process's rows of a
        DeviceDataset / view (rank-local, in DeviceDataset.margins' order)."""
        if isinstance(x, DeviceDataset):
            return x.kmeans_assign(self.clusterCenters)[0]
        a = np.asarray(x, dtype=np.float64)
        if a.ndim == 1:
            return int(closest(a[None, :], self.clusterCenters)[0])
        return closest(a, self.clusterCenters)

    def computeCost(self, data) -> float:
        """The sum of squared distances of the rows to their closest centre: collective on a DeviceDataset / view."""
        if isinstance(data, DeviceDataset):
            return data.kmeans_step(self.clusterCenters, sums=False)[2]
        a = np.atleast_2d(np.asarray(data, dtype=np.float64))
        idx = closest(a, self.clusterCenters)
        return float(((a - self.clusterCenters[idx]) ** 2).sum())


class KMeans:
    """KMeans [mllib-1.3.0] (setInitialModel as in mllib >= 1.4)."""

    def __init__(self, k: int = 2, maxIterations: int = 20, runs: int = 1, initializationMode: str = K_MEANS_PARALLEL,
                 initializationSteps: int = 5, epsilon: float = 1e-4, seed: Optional[int] = None):
        self.setK(k).setMaxIterations(maxIterations).setRuns(runs).setInitializationMode(initializationMode)
        self.setInitializationSteps(initializationSteps).setEpsilon(epsilon)
        self.seed = None if seed is None else int(seed) & _MASK64
        self.initialModel = None

    def setK(self, k: int):
        if int(k) < 1:
            raise ValueError(f"k must be at least 1, got {k}")
        self.k = int(k)
        return self

    def getK(self) -> int:
        return self.k

    def setMaxIterations(self, maxIterations: int):
        if int(maxIterations) < 0:
            raise ValueError(f"maxIterations must be >= 0, got {maxIterations}")
        self.maxIterations = int(maxIterations)
        return self

    def getMaxIterations(self) -> int:
        return self.maxIterations

    def setRuns(self, runs: int):
        if int(runs) < 1:
            raise ValueError(f"runs must be at least 1, got {runs}")
        self.runs = int(runs)
        return self

    def getRuns(self) -> int:
        return self.runs

    def setInitializationMode(self, initializationMode: str):
        if initializationMode not in (K_MEANS_PARALLEL, RANDOM):
            raise ValueError(f"unknown initialization mode {initializationMode!r} (\"{RANDOM}\" or \"{K_MEANS_PARALLEL}\")")
        self.initializationMode = initializationMode
        return self

    def getInitializationMode(self) -> str:
        return self.initializationMode

    def setInitializationSteps(self, initializationSteps: int):
        if int(initializationSteps) < 1:
            raise ValueError(f"initializationSteps must be at least 1, got {initializationSteps}")
        self.initializationSteps = int(initializationSteps)
        return self

    def getInitializationSteps(self) -> int:
        return self.initializationSteps

    def setEpsilon(self, epsilon: float):
        if not (float(epsilon) >= 0.0):
            raise ValueError(f"epsilon must be >= 0, got {epsilon}")
        self.epsilon = float(epsilon)
        return self

    def getEpsilon(self) -> float:
        return self.epsilon

    def setSeed(self, seed: int):
        self.seed = int(seed) & _MASK64
        return self

    def getSeed(self) -> Optional[int]:
        return self.seed

    def setInitialModel(self, model: KMeansModel):
        """Start from these centres (one run; mllib >= 1.4).  Their count must equal k, their width the data's."""
        c = model.clusterCenters
        if c.shape[0] != self.k:
            raise ValueError(f"the initial model has {c.shape[0]} centres, k is {self.k}")
        if not np.all(np.isfinite(c)):
            raise ValueError("the initial model's centres must be finite")
        self.initialModel = model
        return self

    # --- initialisation ---
    @staticmethod
    def _smallest_draws(data: DeviceDataset, seed: int, k: int, n: int) -> np.ndarray:
        """The k rows with the smallest draws under `seed` (rows cycled when the view has fewer than k)."""
        f = min(1.0, (2.0 * k + 16.0) / n)
        while True:
            rows, draws = data.kmeans_sample(seed, f, weighted=False)
            if rows.shape[0] >= k or f >= 1.0:
                break
            f = min(1.0, 4.0 * f)
        rows = rows[np.argsort(draws, kind="stable")]
        return rows[np.arange(k) % rows.shape[0]]

    def _init_random(self, data, seed, n):
        return self._smallest_draws(data, seed, self.k, n)

    def _init_parallel(self, data, seed, n):
        k = self.k
        centers = self._smallest_draws(data, seed, 1, n)
        new = centers
        total = 0.0
        for step in range(self.initializationSteps):
            if new is not None:
                total = data.kmeans_costs(new, keep=step > 0)
            if not (total > 0.0 and np.isfinite(total)):
                break
            rows, _ = data.kmeans_sample(seed ^ ((step + 1) << 16), 2.0 * k / total, weighted=True)
            new = rows if rows.shape[0] else None
            if new is not None:
                centers = np.vstack([centers, rows])
        _, weights, _ = data.kmeans_step(centers, sums=False)
        return LocalKMeans.kMeansPlusPlus(seed, centers, weights, k, LOCAL_MAX_ITERATIONS)

    def run(self, data: DeviceDataset) -> KMeansModel:
        """Train on every row of `data` (a DeviceDataset or view; collective: every rank calls it and gets the same model)."""
        n = data.count()
        if n == 0:
            raise ValueError("KMeans: the data has no rows")
        if self.initialModel is not None and self.initialModel.clusterCenters.shape[1] != data.d:
            raise ValueError(f"the initial model's centres have {self.initialModel.clusterCenters.shape[1]} features, the data "
                             f"{data.d}")
        seed = self.seed
        if seed is None:
            if data.ctx.world_size > len(data.ctx.devices):
                raise ValueError("KMeans: pass a seed in a multi-process world (every rank must draw the same rows)")
            seed = int(np.random.default_rng().integers(0, 2 ** 63))
        step = lambda c: data.kmeans_step(c)   # noqa: E731
        best = None
        for r in range(1 if self.initialModel is not None else self.runs):
            rs = (seed + 0x9E3779B97F4A7C15 * r) & _MASK64
            if self.initialModel is not None:
                init = self.initialModel.clusterCenters
            elif self.initializationMode == RANDOM:
                init = self._init_random(data, rs, n)
            else:
                init = self._init_parallel(data, rs, n)
            centers, cost, _ = lloyd(step, init, self.maxIterations, self.epsilon)
            if best is None or cost < best[1]:
                best = (centers, cost)
        return KMeansModel(best[0])

    @staticmethod
    def train(data: DeviceDataset, k: int, maxIterations: int, runs: int = 1, initializationMode: str = K_MEANS_PARALLEL,
              seed: Optional[int] = None) -> KMeansModel:
        return KMeans(k=k, maxIterations=maxIterations, runs=runs, initializationMode=initializationMode, seed=seed).run(data)
