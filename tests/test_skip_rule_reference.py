"""CPU check of the skip rule's two references: k1_reference.fold_shard and the C oracle (oracle/agd_oracle.c) are
independent restatements of which rows the reference folds into applySmooth, and must agree bit for bit -- on finite
shards, and on shards whose skipped rows hold +-inf or NaN.

  dense: a row whose multiplier is exactly 0 adds nothing (netlib DAXPY returns when DA == 0);
  CSR:   a sampled row adds mult * x unless it is a hinge row outside the margin (the sparse axpy has no zero test)."""
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import k1_reference as R  # noqa: E402

INF, NAN = np.inf, np.nan


def _shard(rng, n, d, kind):
    X = rng.standard_normal((n, d))
    w = rng.standard_normal(d) / np.sqrt(d)
    w[0] = 0.0
    m = X @ w
    y = m + 0.1 * rng.standard_normal(n) if kind.startswith("least") else (m + rng.logistic(size=n) > 0).astype(float)
    return X, y, w


def _poison(X, y, w, kind, rng):
    """Rows the reference skips on dense storage, holding +-inf / NaN: hinge rows outside the margin (one with a NaN margin
    through w_0 = 0), saturated logistic rows (y = 1, m = +inf: multiplier exactly 0)."""
    X, y = X.copy(), y.copy()
    rows = rng.choice(len(y), 6, replace=False)
    j = 1 + int(np.argmax(np.abs(w[1:])))
    sj = np.sign(w[j])
    for t, i in enumerate(rows):
        if kind == "hinge":
            if t % 3 == 0:
                X[i, 0] = INF if t % 2 else -INF           # 0 * inf: NaN margin, outside the margin
            elif t % 3 == 1:
                X[i, j], y[i] = INF, (1.0 if sj > 0 else 0.0)
            else:
                X[i, j], y[i] = -INF, (0.0 if sj > 0 else 1.0)
                X[i, 0] = NAN
        elif kind == "logistic":
            X[i, j], y[i] = INF * sj, 1.0                    # m = +inf, y = 1: multiplier exactly 0
    return X, y


def _oracle_fold(oracle, kind, y, w, X=None, csr=None, sample=None):
    D = oracle.Data(y, X=X) if X is not None else oracle.Data(y, csr=csr, d=len(w))
    if sample is not None:
        D._s.sample_seed, D._s.sample_thresh = sample[0], sample[1]
    loss, g, cnt = oracle.smooth(D, kind, w, partitions=1, threads=1)
    return loss, g, cnt


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64)[np.isfinite(a)], b.view(np.uint64)[np.isfinite(b)]) and \
        np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b)) and \
        np.array_equal(np.isneginf(a), np.isneginf(b))


def _to_csr(X, rng):
    mask = rng.random(X.shape) < 0.5
    mask |= ~np.isfinite(X)                               # non-finite entries are stored
    rowptr = np.concatenate([[0], np.cumsum(mask.sum(axis=1))]).astype(np.int64)
    idx = np.nonzero(mask)[1].astype(np.int32)
    return rowptr, idx, X[mask]


@pytest.mark.parametrize("store", ["f64", "f32", "csr-f64", "csr-f32"])
@pytest.mark.parametrize("kind", list(R.KINDS))
@pytest.mark.parametrize("masked", [False, True])
def test_fold_matches_oracle_on_finite_shards(oracle, store, kind, masked):
    rng = np.random.default_rng(zlib.crc32(f"{store}-{kind}-{masked}".encode()))
    X, y, w = _shard(rng, 300, 9, kind)
    if store.endswith("f32"):
        X = X.astype(np.float32)
    sample = (43, int(np.ldexp(0.3, 64)), np.arange(300)) if masked else None
    if store.startswith("csr"):
        csr = _to_csr(X, rng)
        l, c, g = R.fold_shard(kind, y, w, csr=csr, sample=sample)
        lo, go, co = _oracle_fold(oracle, kind, y, w, csr=csr, sample=sample)
    else:
        l, c, g = R.fold_shard(kind, y, w, X=X, sample=sample)
        lo, go, co = _oracle_fold(oracle, kind, y, w, X=X, sample=sample)
    assert c == co and 0 < c <= 300
    assert _same(l / c, lo) and _same(g / float(c), go)
    assert np.all(np.isfinite(g))


@pytest.mark.parametrize("kind", ["hinge", "logistic"])
@pytest.mark.parametrize("store", ["f64", "f32", "csr-f64", "csr-f32"])
def test_fold_matches_oracle_on_poisoned_skipped_rows(oracle, store, kind):
    """Dense: the poisoned rows are skipped and the gradient stays finite.  CSR: the hinge rows are skipped too, but a
    saturated logistic row adds 0 * inf = NaN at its infinite feature."""
    rng = np.random.default_rng(5 if kind == "hinge" else 6)
    X, y, w = _shard(rng, 200, 7, kind)
    X, y = _poison(X, y, w, kind, rng)
    if store.endswith("f32"):
        X = X.astype(np.float32)
    if store.startswith("csr"):
        csr = _to_csr(X, rng)
        l, c, g = R.fold_shard(kind, y, w, csr=csr)
        lo, go, co = _oracle_fold(oracle, kind, y, w, csr=csr)
    else:
        l, c, g = R.fold_shard(kind, y, w, X=X)
        lo, go, co = _oracle_fold(oracle, kind, y, w, X=X)
    assert c == co == 200
    assert _same(l / c, lo) and _same(g / float(c), go)
    assert np.isfinite(l)
    if kind == "logistic" and store.startswith("csr"):
        assert np.isnan(g).sum() == 1                     # the one poisoned feature; the rest stays finite
    else:
        assert np.all(np.isfinite(g))


def test_mask_drops_poisoned_rows(oracle):
    """Rows the mini-batch mask drops are never touched, on either storage."""
    rng = np.random.default_rng(9)
    X, y, w = _shard(rng, 256, 6, "least_squares")
    sample = (44, int(np.ldexp(0.25, 64)), np.arange(256))
    dropped = ~R.row_selected(*sample)
    X[np.nonzero(dropped)[0][:5], 2] = [INF, -INF, NAN, INF, NAN]
    for csr in (None, _to_csr(X, rng)):
        kw = {"csr": csr} if csr is not None else {"X": X}
        l, c, g = R.fold_shard("least_squares", y, w, sample=sample, **kw)
        lo, go, co = _oracle_fold(oracle, "least_squares", y, w, sample=sample, **kw)
        assert c == co == int((~dropped).sum())
        assert _same(l / c, lo) and _same(g / float(c), go) and np.all(np.isfinite(g))
