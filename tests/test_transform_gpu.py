"""Feature transforms on the GPU (agd_set_feature_transform, StandardScaler / MLUtils.appendBias views): every gradient kernel
on appendBias(s o x) against the reference on the materialised fp64 x', under views, with +-inf / NaN in skipped rows, the
two-point sweeps against separate sweeps, whole AGD / GD runs against the oracle, GLM training against the host path, and
LIBSVM -> randomSplit -> scaler -> appendBias -> train -> evaluate."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import k1_reference as R  # noqa: E402
from view_reference import view_mask  # noqa: E402

pytestmark = pytest.mark.gpu

INF, NAN = np.inf, np.nan

# name: (storage, d, options)
KERNELS = {
    "ring-f32-1024": ("f32", 1024, {"k1_variant": "ring"}),
    "ring-f32-100": ("f32", 100, {"k1_variant": "ring"}),
    "ring-f64-512": ("f64", 512, {"k1_variant": "ring"}),
    "generic-f32-1024": ("f32", 1024, {"k1_variant": "generic"}),
    "wgmma-1024": ("bf16", 1024, {"k1_variant": "tc"}),
    "csr-f32": ("csr-f32", 1024, {}),
    "csr-f64": ("csr-f64", 1024, {}),
}
LOSSES = ["logistic", "least_squares", "hinge", "least_squares_half"]
FORMS = ["bias", "scale", "both"]


def gradient(agd, kind):
    return {"logistic": agd.LogisticGradient(), "least_squares": agd.LeastSquaresGradient(),
            "hinge": agd.HingeGradient(), "least_squares_half": agd.LeastSquaresGradient(half=True)}[kind]


def make(name, n=3001, seed=0):
    """(X as loaded, X as stored (fp64 values), y, csr as stored or None, std of a pinned StandardScalerModel, with zeros)."""
    store, d, _ = KERNELS[name]
    rng = np.random.default_rng(seed + d)
    X = rng.standard_normal((n, d)).astype(np.float32) * 2.0
    if store == "bf16":
        X = R.bf16_to_f32(R.f32_to_bf16_bits(X))
    wt = rng.standard_normal(d) / np.sqrt(d)
    y = (X.astype(np.float64) @ wt + 0.3 + rng.logistic(size=n) > 0).astype(np.float64)
    Xs = X.astype(np.float64)
    csr = None
    if store.startswith("csr"):
        keep = rng.random(X.shape) < 0.05
        rowptr = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
        csr = (rowptr, np.nonzero(keep)[1].astype(np.int32), Xs[keep])
        Xs = np.where(keep, Xs, 0.0)
    std = np.abs(rng.standard_normal(d)) + 0.25
    std[::7] = 0.0
    return X, Xs, y, csr, std


def load(ctx, name, X, y, csr):
    store, d, opts = KERNELS[name]
    ds = ctx.parallelize_csr(y, *csr, d, store=store[4:]) if csr is not None else ctx.parallelize(y, X, store=store)
    for k, v in opts.items():
        ds.set_option(k, v)
    return ds


def transformed(agd, ds, std, form):
    """(the view, its scale factors s)"""
    v, model = ds, agd.StandardScalerModel(std)
    if form in ("scale", "both"):
        v = model.transform(v)
    if form in ("bias", "both"):
        v = agd.MLUtils.appendBias(v)
    return v, model.factor


def materialise(Xs, s, form, csr=None):
    """x' = appendBias(s o x) in fp64 (dense), and its CSR form when the shard is CSR (explicit entries kept, bias last)."""
    Xp = Xs * s if form in ("scale", "both") else Xs.copy()
    if form in ("bias", "both"):
        Xp = np.concatenate([Xp, np.ones((Xs.shape[0], 1))], axis=1)
    if csr is None:
        return Xp, None
    rowptr, idx, val = csr
    sv = val * s[idx] if form in ("scale", "both") else val.copy()
    if form not in ("bias", "both"):
        return Xp, (rowptr, idx, sv)
    n, d = len(rowptr) - 1, Xs.shape[1]
    cnt = np.diff(rowptr) + 1
    rp = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    ni, nv = np.empty(rp[-1], np.int32), np.empty(rp[-1])
    for r in range(n):
        a, b = rowptr[r], rowptr[r + 1]
        ni[rp[r]:rp[r + 1] - 1], nv[rp[r]:rp[r + 1] - 1] = idx[a:b], sv[a:b]
        ni[rp[r + 1] - 1], nv[rp[r + 1] - 1] = d, 1.0
    return Xp, (rp, ni, nv)


def point(rng, d, form):
    w = rng.standard_normal(d + (1 if form in ("bias", "both") else 0)) / np.sqrt(d)
    if form in ("bias", "both"):
        w[-1] = 0.7
    return w


def check(name, got, kind, Xp, cp, y, w, mask=None):
    loss, g, cnt = got
    mask = np.ones(len(y), bool) if mask is None else mask
    if cp is not None:
        lref, cref, gref = R.fold_shard(kind, y[mask], w, csr=compact_csr(cp, mask))
    else:
        lref, cref, gref = R.fold_shard(kind, y[mask], w, X=Xp[mask])
    assert cnt == cref
    if name.startswith("wgmma"):
        gb, lb, _ = R.dense_bounds(kind, Xp[mask], y[mask], w)
        assert np.all(np.abs(g - gref / cref) <= gb)
        assert abs(loss - lref / cref) <= lb
        return
    gr = gref / cref
    np.testing.assert_allclose(g, gr, rtol=0, atol=1e-12 * max(np.max(np.abs(gr)), 1e-300))
    assert abs(loss - lref / cref) <= 1e-12 * abs(lref / cref) + 1e-300


def compact_csr(csr, mask):
    rowptr, idx, val = csr
    rows = np.nonzero(mask)[0]
    sel = np.concatenate([np.arange(rowptr[r], rowptr[r + 1]) for r in rows]) if rows.size else np.zeros(0, np.int64)
    rp = np.concatenate([[0], np.cumsum(rowptr[rows + 1] - rowptr[rows])]).astype(np.int64)
    return rp, idx[sel], val[sel]


# ---------------------------------------------------------------- one sweep, every kernel, every loss, every form
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", list(KERNELS))
def test_smooth_transformed(agd, ctx, name, form):
    X, Xs, y, csr, std = make(name, seed=1)
    ds = load(ctx, name, X, y, csr)
    v, s = transformed(agd, ds, std, form)
    Xp, cp = materialise(Xs, s, form, csr)
    rng = np.random.default_rng(2)
    assert v.d == Xp.shape[1]
    base = ds.smooth(agd.LogisticGradient(), rng.standard_normal(ds.d) * 0.01)
    for kind in LOSSES:
        w = point(rng, ds.d, form)
        got = v.smooth(gradient(agd, kind), w)
        check(name, got, kind, Xp, cp, y, w)
        # a view of the transformed view: both apply
        part = v.randomSplit([0.6, 0.4], seed=9)[1]
        check(name, part.smooth(gradient(agd, kind), w), kind, Xp, cp, y, w, view_mask(part._preds, 0, len(y)))
        if name in ("ring-f32-1024", "ring-f64-512", "wgmma-1024") and kind in ("logistic", "hinge"):
            w2 = point(rng, ds.d, form)
            one, two = v.smooth(gradient(agd, kind), w), v.smooth(gradient(agd, kind), w2)
            l, g, c, l2 = v.smooth_pair(gradient(agd, kind), w, w2)
            assert (l, c, l2) == (one[0], one[2], two[0]) and np.array_equal(g, one[1])
            l, g, c, l2, g2 = v.smooth_two(gradient(agd, kind), w, w2)
            assert (l, c, l2) == (one[0], one[2], two[0]) and np.array_equal(g, one[1]) and np.array_equal(g2, two[1])
    again = ds.smooth(                                  # the parent after the view calls: no transform left behind
        agd.LogisticGradient(), np.random.default_rng(2).standard_normal(ds.d) * 0.01)
    if csr is None:
        assert again[0] == base[0] and np.array_equal(again[1], base[1])
    else:
        np.testing.assert_allclose(again[1], base[1], rtol=0, atol=1e-13 * np.max(np.abs(base[1])))
    ds.close()


# ---------------------------------------------------------------- skipped rows with +-inf / NaN
@pytest.mark.parametrize("name", list(KERNELS))
def test_skipped_rows_leave_no_trace(agd, ctx, name):
    X, Xs, y, csr, std = make(name, seed=3)
    n, d = X.shape
    keep = view_mask(((11, 0.0, 0.75, False),), 0, n)
    out = np.nonzero(~keep)[0]
    targets = sorted({int(out[np.argmin(np.abs(out - t))]) for t in (0, 15, 50, n // 2, n - 1)})
    Xq, Xsq = X.copy(), Xs.copy()
    for t, i in enumerate(targets):
        val = (INF, -INF, NAN)[t % 3]
        Xq[i, 1 + t % 5] = val
        Xsq[i, 1 + t % 5] = val
    c = None
    if csr is not None:
        nz = (np.random.default_rng(4).random(Xsq.shape) < 0.05) | ~np.isfinite(Xsq)
        rowptr = np.concatenate([[0], np.cumsum(nz.sum(axis=1))]).astype(np.int64)
        c = (rowptr, np.nonzero(nz)[1].astype(np.int32), Xsq[nz])
        Xsq = np.where(nz, Xsq, 0.0)
    ds = load(ctx, name, Xq, y, c)
    v, s = transformed(agd, ds.sample(False, 0.75, seed=11), std, "scale")
    v = agd.MLUtils.appendBias(v)
    Xp, cp = materialise(Xsq, s, "both", c)
    rng = np.random.default_rng(5)
    for kind in ("logistic", "hinge"):
        w = point(rng, d, "both")
        got = v.smooth(gradient(agd, kind), w)
        assert np.all(np.isfinite(got[1])) and np.isfinite(got[0])
        check(name, got, kind, Xp, cp, y, w, keep)
    ds.close()


# ---------------------------------------------------------------- whole runs against the oracle on x'
@pytest.mark.parametrize("name", ["ring-f32-1024", "ring-f64-512", "generic-f32-1024", "wgmma-1024", "csr-f32"])
def test_runs_on_transformed_view(agd, ctx, oracle, name):
    X, Xs, y, csr, std = make(name, seed=4)
    ds = load(ctx, name, X, y, csr)
    d = KERNELS[name][1]
    both, s = transformed(agd, ds, std, "both")
    train = agd.MLUtils.kFold(both, 3, seed=17)[1][0]
    mask = view_mask(train._preds, 0, len(y))
    Xp, cp = materialise(Xs, s, "both", csr)
    w0 = np.zeros(d + 1)
    w0[-1] = 1.0
    wf, hf, sf = agd.run_with_stats(train, agd.LogisticGradient(), agd.SquaredL2Updater(), 0.0, 6, 0.05, w0)
    wm, hm, _ = agd.run_with_stats(train, agd.LogisticGradient(), agd.SquaredL2Updater(), 0.0, 6, 0.05, w0, memoize=True)
    if csr is None:
        assert np.array_equal(wf, wm) and np.array_equal(hf, hm)
    D = oracle.Data(y[mask], csr=compact_csr(cp, mask), d=d + 1) if csr is not None else oracle.Data(y[mask], X=Xp[mask])
    ref = oracle.agd_run(D, "logistic", "squared_l2", w0, convergence_tol=0.0, num_iterations=6, reg_param=0.05, partitions=1)
    tol = 1e-6 if name.startswith("wgmma") else 1e-9
    np.testing.assert_allclose(hf, ref.loss_history, rtol=tol)
    assert np.linalg.norm(wf - ref.weights) <= tol * np.linalg.norm(ref.weights)
    assert (sf.passes, sf.backtracks, sf.restarts) == (ref.passes, ref.backtracks, ref.restarts)
    # mini-batch SGD: a row must pass the view and the iteration's mask
    wg, _ = agd.GradientDescent.runMiniBatchSGD(train, agd.LeastSquaresGradient(), agd.SquaredL2Updater(), 0.1, 4, 0.01,
                                                0.5, w0)
    w_h = w0.copy()
    thresh = int(np.ldexp(0.5, 64))
    for i in range(1, 5):
        sel = R.row_selected(42 + i, thresh, np.arange(len(y))) & mask
        if cp is not None:
            _, cnt, g = R.fold_shard("least_squares", y[sel], w_h, csr=compact_csr(cp, sel))
        else:
            _, cnt, g = R.fold_shard("least_squares", y[sel], w_h, X=Xp[sel])
        step = 0.1 / np.sqrt(i)
        w_h = w_h * (1.0 - step * 0.01) - step * (g / cnt)
    assert np.linalg.norm(wg - w_h) <= tol * np.linalg.norm(w_h)
    ds.close()


# ---------------------------------------------------------------- GLM: the view route against the host route
def test_glm_pinned_scaler_matches_host_path(agd, ctx):
    rng = np.random.default_rng(6)
    n, d = 4000, 40
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 20.0, d) + rng.uniform(-3, 3, d)
    X[:, 5] = 2.0                                         # a constant column: s = 0
    y = (X @ (rng.standard_normal(d) / 20.0) + 1.0 + rng.logistic(size=n) > 0).astype(np.float64)
    w0 = rng.standard_normal(d) * 0.01
    host = agd.LogisticRegressionWithAGD(numIterations=15, regParam=0.01).setIntercept(True).setFeatureScaling(True)
    mh = host.run(ctx, y, X, initialWeights=w0)
    data = ctx.parallelize(y, X, store="f64")
    scaler = agd.StandardScalerModel(agd.column_std(X))          # pinned: the host path's own std
    view = agd.MLUtils.appendBias(scaler.transform(data))
    fitted = agd.StandardScaler().fit(data)
    np.testing.assert_allclose(fitted.std, scaler.std, rtol=1e-12)
    s = scaler.factor
    # the host path starts from appendBias(w0) in the scaled space: w0 is already the scaled-space weights there
    mv = agd.LogisticRegressionWithAGD(numIterations=15, regParam=0.01).run(view, initialWeights=np.append(w0, 1.0))
    assert mv.weights.shape == (d + 1,) and mv.intercept == 0.0
    np.testing.assert_allclose(mv.weights[:d] * s, mh.weights, rtol=1e-8, atol=1e-10)
    assert mv.weights[d] == pytest.approx(mh.intercept, rel=1e-8)
    ev_view, ev_host = mv.evaluate(view), mh.evaluate(data)
    assert ev_view.count == ev_host.count == n
    assert ev_view.mean_loss == pytest.approx(ev_host.mean_loss, rel=1e-8)
    np.testing.assert_allclose(mv.predict(view), mh.predict(data))
    # colStats of the view: the transformed columns, bias last
    st = agd.Statistics.colStats(view)
    np.testing.assert_allclose(st.variance[:d], np.where(s != 0, 1.0, 0.0), rtol=1e-10, atol=1e-12)
    assert st.mean[d] == 1.0 and st.variance[d] == 0.0 and st.count == n
    data.close()


def test_learned_intercept_recovers_offset(agd, ctx):
    rng = np.random.default_rng(7)
    n, d = 20000, 64
    X = rng.standard_normal((n, d)).astype(np.float32)
    wt = rng.standard_normal(d)
    y = X.astype(np.float64) @ wt + 3.0 + 0.01 * rng.standard_normal(n)
    data = ctx.parallelize(y, X, store="f32")
    m = agd.LinearRegressionWithAGD(numIterations=200, convergenceTol=1e-12).run(agd.MLUtils.appendBias(data))
    assert m.weights[-1] == pytest.approx(3.0, abs=1e-2)
    np.testing.assert_allclose(m.weights[:d], wt, atol=1e-2)
    data.close()


def test_transform_install_hygiene(agd, ctx):
    X, Xs, y, _, _ = make("ring-f32-1024", seed=8)
    ds = load(ctx, "ring-f32-1024", X, y, None)
    grad = agd.LogisticGradient()
    w = np.random.default_rng(1).standard_normal(1024) * 0.01
    base = ds.smooth(grad, w)
    L = agd._native.lib()
    bad = np.ones(1024)
    bad[3] = np.nan
    assert L.agd_set_feature_transform(ds.h, bad.ctypes.data_as(C.c_void_p), 0) != 0
    assert L.agd_set_feature_transform(ds.h, None, 2) != 0
    after = ds.smooth(grad, w)                                  # a failed install leaves no transform
    assert after[0] == base[0] and np.array_equal(after[1], base[1])
    ones = np.ones(1024)
    assert L.agd_set_feature_transform(ds.h, ones.ctypes.data_as(C.c_void_p), 0) == 0   # s = 1: the same model
    same = ds.smooth(grad, w)
    assert same[2] == base[2]
    np.testing.assert_allclose(same[1], base[1], rtol=0, atol=1e-15 * np.max(np.abs(base[1])))
    assert L.agd_set_feature_transform(ds.h, None, 0) == 0
    view = agd.MLUtils.appendBias(ds)
    with pytest.raises(RuntimeError):
        with view._filtered():                                 # an error inside a view call clears the transform too
            raise RuntimeError("failed inside a view call")
    again = ds.smooth(grad, w)
    assert again[0] == base[0] and np.array_equal(again[1], base[1])
    ds.close()


# ---------------------------------------------------------------- end to end
def _libsvm(tmp_path, n=3000, d=60, seed=0):
    rng = np.random.default_rng(seed)
    wt = rng.standard_normal(d)
    scale = rng.uniform(0.1, 30.0, d)
    lines = []
    for _ in range(n):
        cols = np.sort(rng.choice(d, size=8, replace=False))
        vals = rng.standard_normal(8) * scale[cols] + 2.0
        y = 1.0 if (vals / scale[cols]) @ wt[cols] + 0.5 + 0.3 * rng.standard_normal() > 0 else 0.0
        lines.append(f"{y:g} " + " ".join(f"{c + 1}:{float(v)!r}" for c, v in zip(cols, vals)))
    p = tmp_path / "data.libsvm"
    p.write_text("\n".join(lines) + "\n")
    return str(p)


def test_libsvm_split_scale_bias_train_evaluate(agd, ctx, tmp_path):
    path = _libsvm(tmp_path)
    labels, rowptr, idx, val, d = agd.MLUtils.parseLibSVMFile(path)
    data = agd.MLUtils.loadLibSVMFile(ctx, path)
    train, test = data.randomSplit([0.8, 0.2], seed=13)
    scaler = agd.StandardScaler().fit(train)
    tr, te = (agd.MLUtils.appendBias(scaler.transform(v)) for v in (train, test))
    model = agd.LogisticRegressionWithAGD(numIterations=30, regParam=0.01).run(tr)
    ev = model.evaluate(te)
    svm = agd.SVMWithAGD(numIterations=30, regParam=0.01).run(tr)     # the README's pipeline
    assert svm.evaluate(te).accuracy > 0.7
    # the same pipeline on parsed host arrays
    X = np.zeros((len(labels), d))
    for r in range(len(labels)):
        X[r, idx[rowptr[r]:rowptr[r + 1]]] = val[rowptr[r]:rowptr[r + 1]]
    mtr, mte = view_mask(train._preds, 0, len(labels)), view_mask(test._preds, 0, len(labels))
    hs = agd.StandardScaler().fit(X[mtr])
    np.testing.assert_allclose(scaler.std, hs.std, rtol=1e-12)
    Xtr, Xte = (agd.MLUtils.appendBias(hs.transform(X[m])) for m in (mtr, mte))
    host = ctx.parallelize(labels[mtr], Xtr, store="f64")
    hm = agd.LogisticRegressionWithAGD(numIterations=30, regParam=0.01).run(host)
    assert np.linalg.norm(model.weights - hm.weights) <= 1e-7 * np.linalg.norm(hm.weights)
    m = Xte @ hm.weights
    yt = labels[mte]
    pos = m > 0.0
    assert ev.count == mte.sum()
    assert abs(ev.accuracy - (pos == (yt == 1)).mean()) <= 2.0 / mte.sum()
    assert ev.accuracy > 0.7
    host.close()
    data.close()
