"""org.apache.spark.mllib.linalg.distributed.RowMatrix [mllib-1.3.0] on the resident shards: Gramian, covariance and principal
components of a DeviceDataset or view.

  mat = RowMatrix(data)
  mat.computeGramianMatrix()            # d x d, sum x x^T
  mat.computeCovariance()               # d x d, unbiased
  mat.computePrincipalComponents(k)     # d x k
  mat.multiply(B)                       # RowMatrix of the rows times B, resident on the same devices
  mat.computeSVD(k, computeU=True)      # SingularValueDecomposition(U, s, V)

The device returns the augmented cross-products [sum z z^T, sum z; sum z^T, count] over every shard of the world
(agd_gramian); everything else is derived from that (d + 1) x (d + 1) matrix on the host, in O(d^2) (O(d^3) for the
eigendecomposition, which MLlib also runs on the driver).  multiply projects the rows on the device (agd_project) into a new
resident dataset.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np

from .optimization import DeviceDataset

# MLlib's computeCorrelationMatrixFromCovariance: a variance at most this large in magnitude is a constant column
CORR_VARIANCE_EPS = 1e-12


def _count(aug) -> float:
    n = float(aug[-1, -1])
    if not (n > 0):
        raise ValueError("RowMatrix has no rows (count is 0)")
    return n


def augmented_transformed(aug, scale=None, bias: bool = False, centered: bool = False) -> np.ndarray:
    """The augmented matrix of appendBias(s o x) from that of the stored features x, in O(d^2): sum z z^T scales to
    diag(s) G diag(s) and sum z to s o sum z.  The appended column is 1 in every row: uncentered, its cross-products are
    [s o sum x, n] and its sum n; centered, z = 1 - 1 = 0, so its row and column are 0."""
    a = np.asarray(aug, dtype=np.float64)
    d = a.shape[0] - 1
    G, s, n = a[:d, :d], a[:d, d], a[d, d]
    if scale is not None:
        sc = np.asarray(scale, dtype=np.float64)
        G = G * sc[:, None] * sc[None, :]
        s = s * sc
    if not bias:
        out = np.empty_like(a)
        out[:d, :d], out[:d, d], out[d, :d], out[d, d] = G, s, s, n
        return out
    out = np.zeros((d + 2, d + 2), dtype=np.float64)
    out[:d, :d] = G
    out[:d, d + 1] = out[d + 1, :d] = s
    out[d + 1, d + 1] = n
    if not centered:
        out[:d, d] = out[d, :d] = s
        out[d, d] = out[d, d + 1] = out[d + 1, d] = n
    return out


def covariance_from_augmented(aug) -> np.ndarray:
    """The unbiased covariance (sum z z^T - (sum z)(sum z)^T / n) / (n - 1).  From centered sums this is the corrected
    two-pass formula (accurate where a mean is large next to the spread); from uncentered ones it is MLlib's (G - n mu mu^T) /
    (n - 1).  Exactly symmetric.  One row raises ValueError, as MLlib's require(m > 1) does."""
    a = np.asarray(aug, dtype=np.float64)
    n = _count(a)
    if n <= 1:
        raise ValueError(f"Cannot compute the covariance of a RowMatrix with <= 1 row (it has {int(n)}).")
    d = a.shape[0] - 1
    s = a[:d, d]
    return (a[:d, :d] - np.outer(s, s) / n) / (n - 1.0)


def correlation_from_covariance(cov) -> np.ndarray:
    """Pearson correlation as MLlib's computeCorrelationMatrixFromCovariance: sigma_i = 0 where |cov_ii| <= 1e-12, else
    sqrt(cov_ii); an off-diagonal entry is NaN where either sigma is 0; the diagonal is 1.0."""
    c = np.asarray(cov, dtype=np.float64)
    v = np.diag(c)
    small = np.abs(v) <= CORR_VARIANCE_EPS
    with np.errstate(divide="ignore", invalid="ignore"):   # a negative variance gives a NaN sigma, as in IEEE arithmetic
        sigma = np.where(small, 0.0, np.sqrt(np.where(small, 1.0, v)))
        r = c / (sigma[:, None] * sigma[None, :])
    zero = sigma == 0.0
    r[zero[:, None] | zero[None, :]] = np.nan
    np.fill_diagonal(r, 1.0)
    return r


def principal_components(cov, k: int) -> np.ndarray:
    """d x k: the top-k eigenvectors of the covariance (numpy.linalg.eigh) in descending eigenvalue order, each column's sign
    fixed so that its entry of largest magnitude (the first of equals) is positive."""
    c = np.asarray(cov, dtype=np.float64)
    d = c.shape[0]
    if not (isinstance(k, (int, np.integer)) and 1 <= k <= d):
        raise ValueError(f"k = {k} out of range 1 <= k <= n = {d}")
    w, v = np.linalg.eigh(c)
    order = np.argsort(w, kind="stable")[::-1][:k]
    return _fix_signs(v[:, order])


def _fix_signs(m):
    """Each column times -1 where its entry of largest magnitude (the first of equals) is negative."""
    big = np.argmax(np.abs(m), axis=0)
    signs = np.where(m[big, np.arange(m.shape[1])] < 0, -1.0, 1.0)
    return m * signs[None, :]


class SingularValueDecomposition(NamedTuple):
    """SingularValueDecomposition(U, s, V) of mllib 1.3.0: U a RowMatrix (None unless computeU), s the singular values in
    descending order, V the d x len(s) right singular vectors."""
    U: Optional["RowMatrix"]
    s: np.ndarray
    V: np.ndarray


def svd_from_gramian(G, k: int, rCond: float = 1e-9):
    """(s, V) of RowMatrix.computeSVD's local path (mllib 1.3.0) from the Gramian G = A^T A: sigma = sqrt of G's singular
    values, descending; the leading sigma_i >= rCond sigma_0 are kept, at most k of them; V holds the matching singular vectors
    of G, each column's sign fixed as in principal_components."""
    g = np.asarray(G, dtype=np.float64)
    d = g.shape[0]
    if not (isinstance(k, (int, np.integer)) and 1 <= k <= d):
        raise ValueError(f"k = {k} out of range 1 <= k <= n = {d}")
    u, sig2, _ = np.linalg.svd(g)
    sigma = np.sqrt(sig2)
    threshold = float(rCond) * sigma[0]
    sk = 0
    while sk < k and sigma[sk] >= threshold:
        sk += 1
    return sigma[:sk].copy(), _fix_signs(u[:, :sk])


class RowMatrix:
    """RowMatrix(rows) of mllib 1.3.0 over a DeviceDataset or view: its rows are the dataset's feature vectors over every
    shard of the world.  Every method is collective (every rank calls it; every rank gets the same bits).  On a transformed
    view (StandardScaler / appendBias) the rows are the transformed features."""

    def __init__(self, data: DeviceDataset):
        self.data = data

    def numRows(self) -> int:
        return self.data.count()

    def numCols(self) -> int:
        return self.data.d

    def _augmented(self, centered: bool) -> np.ndarray:
        data = self.data
        _, aug = data.gramian(centered)
        if data._scale is not None or data._bias:
            aug = augmented_transformed(aug, data._scale, data._bias, centered)
        return aug

    def computeGramianMatrix(self) -> np.ndarray:
        """d x d: sum x x^T over the rows."""
        aug = self._augmented(False)
        _count(aug)
        return aug[:-1, :-1].copy()

    def computeCovariance(self) -> np.ndarray:
        """d x d unbiased covariance.  Dense shards: from the sums of x - mu, mu from a first pass on the device (more accurate
        than MLlib's G - n mu mu^T where a mean is large next to the spread); CSR shards: from the uncentered sums, MLlib's
        own formula."""
        return covariance_from_augmented(self._augmented(True))

    def computePrincipalComponents(self, k: int) -> np.ndarray:
        """d x k: the top-k principal components (see principal_components)."""
        d = self.numCols()
        if not (isinstance(k, (int, np.integer)) and 1 <= k <= d):
            raise ValueError(f"k = {k} out of range 1 <= k <= n = {d}")
        return principal_components(self.computeCovariance(), k)

    def multiply(self, B, store: str = "f64") -> "RowMatrix":
        """The rows times B ((d, k) array, d = numCols()) as a RowMatrix whose .data is a new resident DeviceDataset (labels
        kept, stored as `store`), projected on the device without a host copy of the rows (DeviceDataset.project).  A wrong
        shape, a non-finite entry or k < 1 raises ValueError."""
        return RowMatrix(self.data.project(B, store=store))

    def computeSVD(self, k: int, computeU: bool = False, rCond: float = 1e-9) -> SingularValueDecomposition:
        """The top-k singular values and right singular vectors (svd_from_gramian of computeGramianMatrix()), with U =
        multiply(V diag(1 / s)) when computeU.  MLlib 1.3.0 takes this local path for small or wide requests and ARPACK on the
        distributed Gramian otherwise; here the Gramian is cheap on the device, so it is always taken and s and V are the exact
        top k to rounding.  k outside 1 <= k <= numCols() raises ValueError."""
        d = self.numCols()
        if not (isinstance(k, (int, np.integer)) and 1 <= k <= d):
            raise ValueError(f"k = {k} out of range 1 <= k <= n = {d}")
        s, V = svd_from_gramian(self.computeGramianMatrix(), k, rCond)
        U = self.multiply(V * (1.0 / s)[None, :]) if computeU else None
        return SingularValueDecomposition(U, s, V)

    def computeColumnSummaryStatistics(self):
        from .stat import Statistics
        return Statistics.colStats(self.data)
