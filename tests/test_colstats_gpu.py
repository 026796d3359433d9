"""Statistics.colStats on the resident shards: agd_col_stats (csrc/colstats.cu) against a math.fsum reference over the
rows as stored (read back with agd_get_rows / agd_get_csr_rows, selected with row_mask on views).

count, numNonzeros, max and min must match exactly.  A sum of n terms is held to (n + 2) 2^-53 times the sum of its terms'
magnitudes; the variance to 1e-11 relative (it is derived with the corrected two-pass formula, so the error of mu cancels).
Non-finite results must have the reference's IEEE class."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_score_gpu import _stored_csr, _stored_dense, bits  # noqa: E402

U = 2.0 ** -53


def ref_column(v, n):
    """Reference statistics of one column: v = its stored values (fp64), n = rows (n - len(v) implicit zeros)."""
    v = np.asarray(v, dtype=np.float64)
    z = n - v.shape[0]
    fin = bool(np.all(np.isfinite(v)))
    f = math.fsum if fin else (lambda t: float(np.sum(np.asarray(list(t), dtype=np.float64))))
    s = f(v)
    r = {"sum": (s, float(np.sum(np.abs(v)))), "sum_sq": (f(v * v), float(np.sum(v * v))),
         "sum_abs": (f(np.abs(v)), float(np.sum(np.abs(v))))}
    r["nnz"] = int(np.count_nonzero(v))
    mx = float(np.fmax.reduce(v)) if v.shape[0] else float("nan")
    mn = float(np.fmin.reduce(v)) if v.shape[0] else float("nan")
    if z > 0:
        mx, mn = float(np.fmax(mx, 0.0)), float(np.fmin(mn, 0.0))
    r["max"], r["min"] = mx, mn
    if n > 1:
        m = s / n
        d1 = f(list(v - m) + [-m] * z)
        d2 = f(list((v - m) ** 2) + [m * m] * z)
        r["var"] = (d2 - d1 * d1 / n) / (n - 1) if fin else float(np.sum(v) * 0.0 + d2)
        r["mean2"] = m * m
    else:
        r["var"] = 0.0 if fin else float("nan")
        r["mean2"] = 0.0
    return r


def _class_or_close(got, ref, tol, what):
    if not math.isfinite(ref):
        assert (math.isnan(got) and math.isnan(ref)) or got == ref, (what, got, ref)
    else:
        assert abs(got - ref) <= tol, (what, got, ref, tol)


def check_summary(st, cols, n):
    """cols: list of per-column stored-value arrays (dense: the whole column)."""
    assert st.count == n
    d = len(cols)
    assert st.mean.shape == (d,)
    mean, var, nnz, mx, mn = st.mean, st.variance, st.numNonzeros, st.max, st.min
    l1, l2sq = st.normL1, st.sum_sq
    for j, v in enumerate(cols):
        r = ref_column(v, n)
        tol = lambda mag: (n + 2) * U * mag  # noqa: E731
        _class_or_close(st.sum[j], r["sum"][0], tol(r["sum"][1]), ("sum", j))
        _class_or_close(mean[j], r["sum"][0] / n, tol(r["sum"][1]) / n + U * abs(r["sum"][0] / n), ("mean", j))
        _class_or_close(l2sq[j], r["sum_sq"][0], tol(r["sum_sq"][1]), ("sum_sq", j))
        _class_or_close(l1[j], r["sum_abs"][0], tol(r["sum_abs"][1]), ("sum_abs", j))
        assert nnz[j] == r["nnz"], ("nnz", j, nnz[j], r["nnz"])
        assert (math.isnan(mx[j]) and math.isnan(r["max"])) or mx[j] == r["max"], ("max", j, mx[j], r["max"])
        assert (math.isnan(mn[j]) and math.isnan(r["min"])) or mn[j] == r["min"], ("min", j, mn[j], r["min"])
        _class_or_close(var[j], r["var"], 1e-11 * abs(r["var"]) + 16 * n * U * U * r["mean2"], ("var", j))


def dense_cols(X):
    return [X[:, j] for j in range(X.shape[1])]


def csr_cols(rp, ix, va, d, keep=None):
    """Per-column stored values of the rows in `keep` (bool mask, default all)."""
    n = rp.shape[0] - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    sel = np.ones(ix.shape[0], bool) if keep is None else keep[rows]
    ixs, vas = ix[sel], va[sel]
    order = np.argsort(ixs, kind="stable")
    ixs, vas = ixs[order], vas[order]
    bounds = np.searchsorted(ixs, np.arange(d + 1))
    return [vas[bounds[j]:bounds[j + 1]] for j in range(d)]


def _matrix(rng, n, d):
    X = rng.standard_normal((n, d)) * np.exp(rng.uniform(-2, 2, d)) + rng.uniform(-3, 3, d)
    X[rng.random((n, d)) < 0.15] = 0.0                       # explicit zeros
    if d > 2:
        X[:, 1] = 0.0                                        # an all-zero column
    return X


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", [1, 3, 1001, 1024, 4096, 20000])
def test_dense(agd, ctx, store, d):
    rng = np.random.default_rng(d * 3 + len(store))
    n1, n2 = (1, 37) if d >= 4096 else (1, 301)
    X = _matrix(rng, n1 + n2, d)
    y = np.zeros(n1 + n2)
    ds = ctx.parallelize(y[:n1], X[:n1], store=store)        # a one-row shard ...
    try:
        Xs, _ = _stored_dense(ds, store)
        st = agd.Statistics.colStats(ds)
        check_summary(st, dense_cols(Xs[:, :d]), n1)
        assert np.all(st.variance == 0.0)
        ds.load_dense(y[n1:], X[n1:], store=store)            # ... and an appended, ragged partition
        Xs, _ = _stored_dense(ds, store)
        st = agd.Statistics.colStats(ds)
        assert st.mean.shape == (d,)                           # padded columns are not reported
        check_summary(st, dense_cols(Xs[:, :d]), n1 + n2)
        again = agd.Statistics.colStats(ds)                    # dense: bit-identical on a repeated call
        for f in ("sum", "sum_sq", "sum_abs", "nnz", "dev", "dev2", "col_max", "col_min"):
            assert np.array_equal(bits(getattr(st, f)), bits(getattr(again, f))), f
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
@pytest.mark.parametrize("d", [1, 100, 1_000_000])
def test_csr(agd, ctx, store, d):
    rng = np.random.default_rng(d + 11)
    n = 2001
    nnz = rng.integers(0, min(d, 30) + 1, size=n)
    nnz[[0, 9, n - 1]] = 0                                     # empty rows
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate([np.sort(rng.choice(d, k, replace=False)) for k in nnz]).astype(np.int32)
    if d == 100:
        keep = ix != 5
        ix = ix[keep]                                          # column 5 has no stored entry at all
        rp = np.concatenate([[0], np.cumsum(np.bincount(np.repeat(np.arange(n), nnz)[keep], minlength=n))]).astype(np.int64)
    va = rng.standard_normal(ix.shape[0]) * 3 - 1
    va[::7] = 0.0                                              # explicitly stored zeros
    y = np.zeros(n)
    h = 700
    ds = ctx.parallelize_csr(y[:h], rp[:h + 1], ix[:rp[h]], va[:rp[h]], d, store=store)
    try:
        ds.load_csr(y[h:], rp[h:] - rp[h], ix[rp[h]:], va[rp[h]:], d, store=store)   # appended partition
        rps, ixs, vas, _ = _stored_csr(ds, store)
        st = agd.Statistics.colStats(ds)
        if d >= 100:
            cols = csr_cols(rps, ixs, vas, d)
            touched = np.unique(ixs)
            sub = touched[:3000] if d > 100 else np.arange(d)
            # every column is reported; an empty column is all implicit zeros
            empty = np.setdiff1d(np.arange(d), touched)[:50]
            assert np.all(st.sum[empty] == 0) and np.all(st.max[empty] == 0) and np.all(st.min[empty] == 0)
            assert np.all(st.numNonzeros[empty] == 0) and np.all(st.variance[empty] == 0)
            check_summary(_Sub(st, sub), [cols[j] for j in sub], n)
        else:
            check_summary(st, csr_cols(rps, ixs, vas, d), n)
        assert st.count == n
    finally:
        ds.close()


class _Sub:
    """The columns `idx` of a summary (the reference for d = 10^6 checks the touched columns and samples the rest)."""

    def __init__(self, st, idx):
        self.count = st.count
        for f in ("sum", "sum_sq", "mean", "variance", "numNonzeros", "max", "min", "normL1"):
            setattr(self, f, getattr(st, f)[idx])


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16"])
def test_generated_shard(agd, ctx, store):
    ds = ctx.synthetic(3001, 256, agd.LogisticGradient(), seed=7, store=store)
    try:
        Xs, _ = _stored_dense(ds, store)
        check_summary(agd.Statistics.colStats(ds), dense_cols(Xs[:, :256]), 3001)
    finally:
        ds.close()


@pytest.mark.gpu
def test_generated_csr_shard(agd, ctx):
    ds = agd.optimization._synthetic_csr(ctx, 4001, 5000, 16, agd.HingeGradient(), seed=3, store="f32")
    try:
        rps, ixs, vas, _ = _stored_csr(ds, "f32")
        check_summary(agd.Statistics.colStats(ds), csr_cols(rps, ixs, vas, 5000), 4001)
    finally:
        ds.close()


@pytest.mark.gpu
def test_large_mean_variance(agd, ctx):
    """mean 1e6 and unit spread: within 1e-12 of the exact variance (sum x^2 - (sum x)^2 / n would lose ~all digits)."""
    rng = np.random.default_rng(5)
    X = 1e6 + rng.standard_normal((20000, 2))
    ds = ctx.parallelize(np.zeros(20000), X, store="f64")
    try:
        st = agd.Statistics.colStats(ds)
        for j in range(2):
            m = math.fsum(X[:, j]) / 20000
            exact = math.fsum((X[:, j] - m) ** 2) / 19999
            assert abs(st.variance[j] - exact) <= 1e-12 * exact, (j, st.variance[j], exact)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dense", "csr"])
def test_nonfinite_kept_and_excluded_rows(agd, ctx, kind):
    """±inf / NaN in rows of a view follow IEEE arithmetic in the sums and are ignored by max / min when NaN; in rows
    outside the view they leave no trace."""
    rng = np.random.default_rng(9)
    n, d = 4000, 6
    X = rng.standard_normal((n, d))
    ds0 = ctx.parallelize(np.zeros(n), X, store="f64")
    try:
        mask = ds0.sample(False, 0.5, seed=13).row_mask(0, 0, n)
    finally:
        ds0.close()
    kept, out = np.flatnonzero(mask), np.flatnonzero(~mask)
    inf, nan = float("inf"), float("nan")
    X[out[:3], 0] = [inf, -inf, nan]                            # excluded rows: column 0 must stay finite
    X[out[3:], 1] = nan                                         # column 1: NaN in every excluded row
    X[kept[0], 2] = inf                                         # kept rows: IEEE sums
    X[kept[1], 3], X[kept[2], 3] = inf, -inf                    # inf - inf = NaN
    X[kept[3], 4] = nan                                         # NaN: nonzero, ignored by max / min
    X[kept, 5] = nan                                            # every kept value NaN: max / min NaN
    if kind == "dense":
        ds = ctx.parallelize(np.zeros(n), X, store="f64")
    else:
        rp = np.arange(0, n * d + 1, d, dtype=np.int64)
        ds = ctx.parallelize_csr(np.zeros(n), rp, np.tile(np.arange(d, dtype=np.int32), n), X.ravel(), d, store="f64")
    try:
        view = ds.sample(False, 0.5, seed=13)
        assert np.array_equal(view.row_mask(0, 0, n), mask)
        st = agd.Statistics.colStats(view)
        check_summary(st, dense_cols(X[kept]), kept.shape[0])
        assert math.isfinite(st.mean[0]) and math.isfinite(st.variance[0]) and math.isfinite(st.mean[1])
        assert st.mean[2] == inf and math.isnan(st.mean[3]) and math.isnan(st.mean[4])
        assert math.isfinite(st.max[4]) and math.isnan(st.max[5]) and math.isnan(st.min[5])
        assert st.numNonzeros[5] == kept.shape[0]
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "csr"])
def test_views_add_up(agd, ctx, store):
    """randomSplit parts: counts add up to the whole, sums to rounding; each part matches its rows; kFold too; an empty
    view raises."""
    rng = np.random.default_rng(17)
    n, d = 6007, 64
    X = _matrix(rng, n, d)
    if store == "csr":
        keep = X != 0
        rp = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int64)
        ds = ctx.parallelize_csr(np.zeros(n), rp, np.nonzero(keep)[1].astype(np.int32), X[keep], d, store="f64")
        Xs = X
    else:
        ds = ctx.parallelize(np.zeros(n), X, store="f32")
        Xs, _ = _stored_dense(ds, "f32")
    try:
        whole = agd.Statistics.colStats(ds)
        parts = ds.randomSplit([0.5, 0.3, 0.2], seed=3)
        sts = [agd.Statistics.colStats(p) for p in parts]
        assert sum(s.count for s in sts) == whole.count == n
        mag = np.abs(Xs).sum(0)
        assert np.all(np.abs(sum(s.sum for s in sts) - whole.sum) <= (n + 2) * U * mag)
        assert np.array_equal(sum(s.numNonzeros for s in sts), whole.numNonzeros)
        assert np.array_equal(np.fmax.reduce([s.max for s in sts]), whole.max)
        for p, s in zip(parts, sts):
            m = p.row_mask(0, 0, n)
            check_summary(s, dense_cols(Xs[m]), int(m.sum()))
        for tr, va in agd.MLUtils.kFold(ds, 3, seed=5):
            mt, mv = tr.row_mask(0, 0, n), va.row_mask(0, 0, n)
            check_summary(agd.Statistics.colStats(tr), dense_cols(Xs[mt]), int(mt.sum()))
            check_summary(agd.Statistics.colStats(va), dense_cols(Xs[mv]), int(mv.sum()))
        with pytest.raises(ValueError, match="Nothing has been added"):
            agd.Statistics.colStats(ds.sample(False, 0.0))
        again = agd.Statistics.colStats(ds)                    # the view's filter was cleared after each call
        assert again.count == n
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "csr"])
def test_collectives_keep_their_bits(agd, ctx, store):
    """smooth and evaluate give the same bits before and after a colStats call on the same handle."""
    rng = np.random.default_rng(23)
    n, d = 5000, 128
    X = rng.standard_normal((n, d))
    y = (rng.random(n) > 0.5).astype(np.float64)
    w = rng.standard_normal(d) * 0.1
    if store == "csr":
        X[rng.random((n, d)) < 0.8] = 0.0
        keep = X != 0
        rp = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int64)
        ds = ctx.parallelize_csr(y, rp, np.nonzero(keep)[1].astype(np.int32), X[keep], d, store="f64")
    else:
        ds = ctx.parallelize(y, X, store=store)
    try:
        g = agd.LogisticGradient()
        e1 = ds.evaluate(g, w, 0.25, 0.5)
        l1, g1, c1 = ds.smooth(g, w)
        agd.Statistics.colStats(ds)
        agd.Statistics.colStats(ds.sample(False, 0.3))
        e2 = ds.evaluate(g, w, 0.25, 0.5)
        l2, g2, c2 = ds.smooth(g, w)
        assert list(e1.__dict__.values()) == list(e2.__dict__.values())
        assert c1 == c2
        if store != "csr":                                     # the CSR gradient kernel scatters: equal to rounding
            assert l1 == l2 and np.array_equal(bits(g1), bits(g2))
        else:
            assert abs(l1 - l2) <= 1e-13 * abs(l1) and np.allclose(g1, g2, rtol=1e-12, atol=1e-15)
    finally:
        ds.close()


def _device_count():
    try:
        cuda = C.CDLL("libcuda.so.1")
        n = C.c_int()
        return n.value if cuda.cuInit(0) == 0 and cuda.cuDeviceGetCount(C.byref(n)) == 0 else 0
    except OSError:
        return 0


@pytest.mark.gpu
@pytest.mark.skipif(_device_count() < 2, reason="needs two GPUs in one process")
@pytest.mark.parametrize("store", ["f32", "csr"])
def test_two_gpus_one_process(agd, store):
    """Two local GPUs are a world of two: the sums and maxima travel through the peer-memory exchange in several epochs."""
    rng = np.random.default_rng(29)
    n, d = 3001, 300
    X = _matrix(rng, n, d)
    c2 = agd.Context(devices=[0, 1])
    if store == "csr":
        keep = X != 0
        rp = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int64)
        ds = c2.parallelize_csr(np.zeros(n), rp, np.nonzero(keep)[1].astype(np.int32), X[keep], d, store="f64")
        Xs = X
    else:
        ds = c2.parallelize(np.zeros(n), X, store="f32")
        Xs = np.concatenate([_stored_dense_dev(ds, i) for i in range(2)])
    try:
        st = agd.Statistics.colStats(ds)
        check_summary(st, dense_cols(Xs), n)
        v = ds.sample(False, 0.4, seed=2)
        m = np.concatenate([v.row_mask(i, 0, ds.local_rows(i)) for i in range(2)])
        check_summary(agd.Statistics.colStats(v), dense_cols(Xs[m]), int(m.sum()))
    finally:
        ds.close()


def _stored_dense_dev(ds, dev):
    X, _ = ds.get_rows(dev, 0, ds.local_rows(dev), dtype=np.float32)
    return X.astype(np.float64)
