"""Scoring the resident shards: agd_margins / agd_evaluate (csrc/score.cu) and the GLM layer on top of them.

Margins are held to the bound of a correctly rounded reference, |dm| <= (d + 2) 2^-53 (sum_j |x_ij w_j| + |b|), where the
reference is math.fsum of the fp64 products plus b over the rows as stored (read back with agd_get_rows /
agd_get_csr_rows).  Evaluation sums are held to 1e-12 of the sum of their terms' magnitudes, counts exactly."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from k1_reference import row_terms  # noqa: E402

U = 2.0 ** -53
KINDS = {"logistic": 0, "least_squares": 1, "hinge": 2, "least_squares_half": 3}


def _grad(agd, kind):
    return {"logistic": agd.LogisticGradient(), "least_squares": agd.LeastSquaresGradient(),
            "hinge": agd.HingeGradient(), "least_squares_half": agd.LeastSquaresGradient(half=True)}[kind]


def _stored_dense(ds, store):
    """The rows as stored on device 0, widened exactly to fp64."""
    dt = {"f32": np.float32, "f64": np.float64, "bf16": np.uint16}[store]
    X, y = ds.get_rows(0, 0, ds.local_rows(0), dtype=dt)
    if store == "bf16":
        X = (X.astype(np.uint32) << 16).view(np.float32)
    return X.astype(np.float64), y


def _stored_csr(ds, store, dev=0):
    n = ds.local_rows(dev)
    rp, ix, va, y = ds.get_csr_rows(dev, 0, n, 1 << 24, dtype=np.float32 if store == "f32" else np.float64)
    return rp, ix, va.astype(np.float64), y


def _ref_row(prods, b):
    """fsum of the fp64 products plus b, and the bound's scale; IEEE classes for non-finite rows."""
    if not np.all(np.isfinite(prods)):
        return float(np.sum(prods) + b), float("inf")
    return math.fsum(list(prods) + [b]), float(np.sum(np.abs(prods)) + abs(b))


def check_dense(m, X, w, b):
    d = X.shape[1]
    assert m.shape == (X.shape[0],)
    for i in range(X.shape[0]):
        ref, scale = _ref_row(X[i] * w, b)
        _check_one(m[i], ref, scale, d, i)


def check_csr(m, rp, ix, va, w, b, d):
    assert m.shape == (rp.shape[0] - 1,)
    for i in range(rp.shape[0] - 1):
        a, e = rp[i], rp[i + 1]
        ref, scale = _ref_row(va[a:e] * w[ix[a:e]], b)
        _check_one(m[i], ref, scale, d, i)


def _check_one(got, ref, scale, d, i):
    if math.isnan(ref) or math.isinf(ref):
        assert (math.isnan(got) and math.isnan(ref)) or got == ref, (i, got, ref)
        return
    assert abs(got - ref) <= (d + 2) * U * scale, (i, got, ref, scale)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


DS = [1, 3, 100, 1001, 1024, 4096, 20000]


def _rows_for(d):
    return (1, 37) if d >= 4096 else (5, 203)


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64", "bf16"])
@pytest.mark.parametrize("d", DS)
def test_dense_margins(agd, ctx, store, d):
    rng = np.random.default_rng(d * 7 + len(store))
    n1, n2 = _rows_for(d)
    X = rng.standard_normal((n1 + n2, d)) * np.exp(rng.uniform(-3, 3, (n1 + n2, 1)))
    y = (rng.random(n1 + n2) > 0.5).astype(np.float64)
    w = rng.standard_normal(d)
    b = -0.8125
    ds = ctx.parallelize(y[:n1], X[:n1], store=store)
    try:
        # a one-row (or few-row) shard, then an appended partition
        Xs, _ = _stored_dense(ds, store)
        check_dense(ds.margins(w, b), Xs, w, b)
        ds.load_dense(y[n1:], X[n1:], store=store)
        Xs, _ = _stored_dense(ds, store)
        m = ds.margins(w, b)
        check_dense(m, Xs, w, b)
        n = n1 + n2
        # a sub-range equals the same rows of the full-range call, bit for bit
        for r0, r in ((0, 1), (n - 1, 1), (n // 3, n - n // 3 - 1), (1, n - 2)):
            assert np.array_equal(bits(ds.margins_rows(0, r0, r, w, b)), bits(m[r0:r0 + r])), (r0, r)
        assert ds.margins_rows(0, n, 0, w, b).shape == (0,)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
@pytest.mark.parametrize("d", [1, 3, 100, 1001, 20000])
def test_csr_margins(agd, ctx, store, d):
    rng = np.random.default_rng(d + 5)
    n = 301
    nnz = rng.integers(0, min(d, 40) + 1, size=n)
    nnz[[0, 7, n - 1]] = 0                                          # empty rows, the last one included
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate([np.sort(rng.choice(d, k, replace=False)) for k in nnz]).astype(np.int32)
    va = rng.standard_normal(rp[-1])
    va[::9] = 0.0                                                   # explicitly stored zeros
    y = (rng.random(n) > 0.5).astype(np.float64)
    w = rng.standard_normal(d)
    b = 0.4375
    h = 120
    ds = ctx.parallelize_csr(y[:h], rp[:h + 1], ix[:rp[h]], va[:rp[h]], d, store=store)
    try:
        ds.load_csr(y[h:], rp[h:] - rp[h], ix[rp[h]:], va[rp[h]:], d, store=store)   # appended partition
        rps, ixs, vas, _ = _stored_csr(ds, store)
        m = ds.margins(w, b)
        check_csr(m, rps, ixs, vas, w, b, d)
        assert m[0] == b and m[7] == b and m[n - 1] == b            # an empty row's margin is the intercept
        for r0, r in ((0, 1), (n - 1, 1), (50, 200)):
            assert np.array_equal(bits(ds.margins_rows(0, r0, r, w, b)), bits(m[r0:r0 + r]))
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store,d", [("f32", 1024), ("bf16", 4096), ("f64", 1001), ("f32", 3), ("bf16", 20000)])
def test_generated_dense_margins(agd, ctx, store, d):
    ds = ctx.synthetic(3001, d, agd.LogisticGradient(), seed=5, store=store)
    try:
        w = np.random.default_rng(1).standard_normal(d) / np.sqrt(d)
        Xs, _ = _stored_dense(ds, store)
        m = ds.margins(w, 0.3)
        check_dense(m[:400], Xs[:400], w, 0.3)
        check_dense(m[-50:], Xs[-50:], w, 0.3)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_generated_csr_margins(agd, ctx, store):
    d = 100000
    ds = ctx.synthetic_csr(5000, d, 64, agd.HingeGradient(), seed=3, store=store)
    try:
        w = np.random.default_rng(2).standard_normal(d)
        rps, ixs, vas, _ = _stored_csr(ds, store)
        check_csr(ds.margins(w, -1.5), rps, ixs, vas, w, -1.5, d)
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "bf16", "f64", "csr_f32"])
def test_nonfinite_features_follow_ieee(agd, ctx, store):
    """An inf feature under a zero weight gives a NaN margin (0 * inf), as ddot and numpy give; nothing is skipped."""
    rng = np.random.default_rng(9)
    n, d = 64, 1024
    X = rng.standard_normal((n, d))
    w = rng.standard_normal(d)
    w[[5, 700]] = 0.0
    X[3, 5] = np.inf
    X[10, 700] = -np.inf
    X[20, 6] = np.inf                                               # nonzero weight: +-inf margin
    X[30, 9] = np.nan
    y = np.zeros(n)
    if store == "csr_f32":
        ds = ctx.parallelize_csr(y, np.arange(n + 1, dtype=np.int64) * d, np.tile(np.arange(d, dtype=np.int32), n),
                                 X.ravel(), d, store="f32")
        Xs = X.astype(np.float32).astype(np.float64)
    else:
        ds = ctx.parallelize(y, X, store=store)
        Xs, _ = _stored_dense(ds, store)
    try:
        m = ds.margins(w, 0.25)
        with np.errstate(invalid="ignore"):
            ref = Xs @ w + 0.25
        np.testing.assert_array_equal(np.isnan(m), np.isnan(ref))
        assert np.isnan(m[[3, 10, 30]]).all() and np.isinf(m[20]) and np.sign(m[20]) == np.sign(ref[20])
        fin = np.isfinite(ref)
        assert np.all(np.isfinite(m[fin]))
    finally:
        ds.close()


@pytest.mark.gpu
def test_margins_argument_errors(agd, ctx):
    L = agd._native.lib()
    ds = ctx.parallelize(np.zeros(10), np.ones((10, 4)), store="f32")
    try:
        w = np.ones(4)
        out = np.empty(10)
        wp, op = w.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)
        with pytest.raises(agd.NativeError, match="bad local device"):
            ds.margins_rows(3, 0, 1, w)
        with pytest.raises(agd.NativeError, match="outside"):
            ds.margins_rows(0, 5, 6, w)
        with pytest.raises(agd.NativeError, match="outside"):
            ds.margins_rows(0, -1, 2, w)
        with pytest.raises(agd.NativeError, match="outside"):
            ds.margins_rows(0, 0, -1, w)
        assert L.agd_margins(ds.h, 0, None, 0.0, 0, 10, op) != 0 and b"NULL" in L.agd_last_error(ds.h)
        assert L.agd_margins(ds.h, 0, wp, 0.0, 0, 10, None) != 0 and b"NULL" in L.agd_last_error(ds.h)
        assert L.agd_margins(ds.h, 0, wp, 0.0, 10, 0, op) == 0                  # rows = 0 succeeds
        sums = np.empty(agd._native.EVAL_N)
        assert L.agd_evaluate(ds.h, 7, wp, 0.0, 0.5, sums.ctypes.data_as(C.c_void_p)) != 0
        assert b"unknown gradient" in L.agd_last_error(ds.h)
        assert L.agd_evaluate(ds.h, 0, wp, 0.0, 0.5, None) != 0 and b"NULL" in L.agd_last_error(ds.h)
        with pytest.raises(ValueError):
            ds.margins(np.ones(5))
    finally:
        ds.close()
    empty = agd.DeviceDataset(ctx)
    try:
        with pytest.raises(agd.NativeError, match="no shard"):
            empty.margins_rows(0, 0, 0, np.ones(0))
    finally:
        empty.close()


# ---------------------------------------------------------------- evaluation
def eval_reference(kind, m, y, t):
    """numpy restatement of the AGD_EVAL_* sums: (value, sum of the terms' magnitudes) per entry."""
    _, loss = row_terms(kind, m, y)
    e = m - y
    binary = (y == 0.0) | (y == 1.0)
    if kind == "logistic":
        pos = 1.0 / (1.0 + np.exp(-m)) > t
    else:
        pos = m > t
    counted = binary if kind in ("logistic", "hinge") else np.zeros_like(binary)
    one = y == 1.0
    terms = [np.ones_like(m), loss, counted & pos & one, counted & pos & ~one, counted & ~pos & ~one, counted & ~pos & one,
             e, e * e, np.abs(e), y, y * y]
    return [(math.fsum(np.asarray(tm, dtype=np.float64)), float(np.sum(np.abs(np.asarray(tm, dtype=np.float64)))))
            for tm in terms]


def _eval_data(rng, n, d):
    X = rng.standard_normal((n, d))
    w = rng.standard_normal(d) / np.sqrt(d) * 2.0
    y = (rng.random(n) > 0.5).astype(np.float64)
    y[::23] = 0.5                                               # rows outside the confusion counts
    y[::31] = 2.0
    return X, w, y


EVAL_CASES = [("f32", 100), ("bf16", 1024), ("f64", 3), ("csr_f64", 300), ("csr_f32", 1)]


def _load(ctx, store, X, y):
    n, d = X.shape
    if store.startswith("csr"):
        rng = np.random.default_rng(d)
        keep = rng.random(X.shape) < (0.3 if d > 1 else 0.8)
        rp = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
        ix = np.nonzero(keep)[1].astype(np.int32)
        return ctx.parallelize_csr(y, rp, ix, X[keep], d, store=store[4:])
    return ctx.parallelize(y, X, store=store)


def _host_rows(ds, store):
    """Exact margins of the stored rows (fsum), for the host restatement."""
    if store.startswith("csr"):
        rp, ix, va, y = _stored_csr(ds, store[4:])
        return lambda w, b: np.array([math.fsum(list(va[rp[i]:rp[i + 1]] * w[ix[rp[i]:rp[i + 1]]]) + [b])
                                      for i in range(len(y))]), y
    X, y = _stored_dense(ds, store)
    return lambda w, b: np.array([math.fsum(list(X[i] * w) + [b]) for i in range(X.shape[0])]), y


@pytest.mark.gpu
@pytest.mark.parametrize("store,d", EVAL_CASES)
@pytest.mark.parametrize("kind", list(KINDS))
def test_evaluate_sums(agd, ctx, store, d, kind):
    rng = np.random.default_rng(d * 3 + KINDS[kind])
    n = 4099
    X, w, y = _eval_data(rng, n, d)
    ds = _load(ctx, store, X, y)
    try:
        margins_of, ys = _host_rows(ds, store)
        b = 0.125
        t = {"logistic": 0.3, "hinge": 0.25}.get(kind, 0.5)
        m = margins_of(w, b)
        # no score within a few ulp of the threshold: the confusion counts are then exact
        score = 1.0 / (1.0 + np.exp(-m)) if kind == "logistic" else m
        assert np.min(np.abs(score - t)) > 1e-12
        ev = ds.evaluate(_grad(agd, kind), w, b, t)
        got = [ev.count, ev.loss_sum, ev.tp, ev.fp, ev.tn, ev.fn, ev.sum_err, ev.sum_err2, ev.sum_abs_err, ev.sum_y, ev.sum_y2]
        ref = eval_reference(kind, m, ys, t)
        for k, (g, (r, mag)) in enumerate(zip(got, ref)):
            if k in (0, 2, 3, 4, 5):
                assert g == r, (k, g, r)
            else:
                assert abs(g - r) <= 1e-12 * mag, (k, g, r, mag)
        assert ev.count == n
        if kind in ("logistic", "hinge"):
            assert ev.tp + ev.fp + ev.tn + ev.fn == np.sum((ys == 0) | (ys == 1)) and ev.tp > 0 and ev.tn > 0
        else:
            assert ev.tp == ev.fp == ev.tn == ev.fn == 0
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store,d", [("f32", 1024), ("bf16", 4096), ("f64", 20000), ("csr_f32", 300), ("csr_f64", 1)])
def test_evaluate_matches_smooth_loss_and_is_reproducible(agd, ctx, store, d):
    rng = np.random.default_rng(d + 11)
    n = 30011 if d <= 1024 else 2003
    X, w, y = _eval_data(rng, n, d)
    y[y > 1] = 1.0
    ds = _load(ctx, store, X, y)
    if store == "bf16":
        ds.set_option("k1_variant", "ring")        # fp64 margins in smooth (the wgmma kernel forms them in fp32)
    try:
        for kind in KINDS:
            g = _grad(agd, kind)
            loss, _, cnt = ds.smooth(g, w)
            ev = ds.evaluate(g, w, 0.0, 0.5)
            assert ev.count == cnt == n
            assert abs(ev.mean_loss - loss) <= 1e-13 * abs(loss), (kind, ev.mean_loss, loss)
            ev2 = ds.evaluate(g, w, 0.0, 0.5)
            assert np.array_equal(bits(list(ev.__dict__.values())), bits(list(ev2.__dict__.values()))), kind
    finally:
        ds.close()


# ---------------------------------------------------------------- the GLM layer
@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f64", "f32"])
def test_glm_predict_on_device_matches_host(agd, ctx, store):
    rng = np.random.default_rng(4)
    n, d = 2000, 50
    X = rng.standard_normal((n, d))
    ds = ctx.parallelize(np.zeros(n), X, store=store)
    try:
        Xh = _stored_dense(ds, store)[0]
        w = rng.standard_normal(d) * 0.3
        for model in (agd.LogisticRegressionModel(w, 0.2), agd.SVMModel(w, -0.1), agd.LinearRegressionModel(w, 0.7)):
            raw = model.predict(Xh)
            dev = model.predict(ds)
            if isinstance(model, agd.LinearRegressionModel):
                np.testing.assert_allclose(dev, raw, rtol=1e-12, atol=1e-12)
                continue
            np.testing.assert_array_equal(dev, raw)                        # the class default threshold
            model.setThreshold(0.6 if isinstance(model, agd.LogisticRegressionModel) else 0.3)
            np.testing.assert_array_equal(model.predict(ds), model.predict(Xh))
            model.clearThreshold()
            assert model.getThreshold() is None
            np.testing.assert_allclose(model.predict(ds), model.predict(Xh), rtol=1e-12, atol=1e-15)
    finally:
        ds.close()


LIBSVM_ROWS = 3000


def _write_libsvm(path, rng, d=40):
    lines = []
    w_true = rng.standard_normal(d)
    for _ in range(LIBSVM_ROWS):
        k = rng.integers(1, 12)
        cols = np.sort(rng.choice(d, k, replace=False))
        vals = rng.standard_normal(k)
        y = 1 if vals @ w_true[cols] + 0.2 * rng.standard_normal() > 0 else 0
        lines.append(f"{y} " + " ".join(f"{c + 1}:{float(v)!r}" for c, v in zip(cols, vals)))
    path.write_text("\n".join(lines) + "\n")


@pytest.mark.gpu
def test_libsvm_train_then_evaluate_on_device(agd, ctx, tmp_path):
    p = tmp_path / "train.libsvm"
    _write_libsvm(p, np.random.default_rng(8))
    data = agd.MLUtils.loadLibSVMFile(ctx, str(p))
    try:
        model = agd.SVMWithAGD(numIterations=30, regParam=0.01).run(data)
        assert isinstance(model, agd.SVMModel) and model.intercept == 0.0
        ev = model.evaluate(data)
        y, rp, ix, va, d = agd.MLUtils.parseLibSVMFile(str(p))
        X = np.zeros((len(y), d))
        for i in range(len(y)):
            X[i, ix[rp[i]:rp[i + 1]]] = va[rp[i]:rp[i + 1]]
        m = X @ model.weights
        assert np.min(np.abs(m)) > 1e-9
        pred = (m > 0.0).astype(np.float64)
        assert ev.count == len(y)
        assert ev.accuracy == np.mean(pred == y) and ev.accuracy > 0.7
        assert ev.tp == np.sum((pred == 1) & (y == 1)) and ev.fn == np.sum((pred == 0) & (y == 1))
        np.testing.assert_array_equal(model.predict(data), pred)
        hinge = np.maximum(0.0, 1.0 - (2 * y - 1) * m)
        assert abs(ev.mean_loss - hinge.mean()) <= 1e-12 * max(hinge.mean(), 1e-300)
        # the model as trained from explicit initial weights, too (run(data, initialWeights))
        m2 = agd.SVMWithAGD(numIterations=2, regParam=0.01).run(data, np.full(d, 0.01))
        assert m2.weights.shape == (d,)
    finally:
        data.close()


@pytest.mark.gpu
def test_run_on_device_rejects_intercept_and_scaling(agd, ctx):
    ds = ctx.parallelize(np.array([0.0, 1.0, 1.0]), np.eye(3), store="f64")
    try:
        with pytest.raises(ValueError, match="intercept"):
            agd.LogisticRegressionWithAGD(numIterations=2).setIntercept(True).run(ds)
        with pytest.raises(ValueError, match="scal"):
            agd.LogisticRegressionWithAGD(numIterations=2).setFeatureScaling(True).run(ds)
        model = agd.LogisticRegressionWithAGD(numIterations=2).run(ds)
        assert model.weights.shape == (3,)
    finally:
        ds.close()


# w sits in shared memory beside the evaluation form's static reduction array up to d = 6056 (48 KB without an opt-in);
# these widths straddle that limit, on the vector (d * elem % 16 == 0) and scalar instantiations
@pytest.mark.gpu
@pytest.mark.parametrize("store,d", [("f64", 6056), ("f32", 6057), ("f32", 6100), ("f32", 6144), ("bf16", 6144),
                                     ("bf16", 6060), ("f64", 6144)])
def test_scoring_across_the_shared_memory_limit(agd, ctx, store, d):
    rng = np.random.default_rng(d + len(store))
    n = 301
    X, w, y = _eval_data(rng, n, d)
    ds = _load(ctx, store, X, y)
    try:
        margins_of, ys = _host_rows(ds, store)
        Xs, _ = _stored_dense(ds, store)
        b = -0.375
        m = ds.margins(w, b)
        check_dense(m, Xs, w, b)
        mref = margins_of(w, b)
        for kind, t in (("logistic", 0.45), ("hinge", 0.1), ("least_squares", 0.5)):
            score = 1.0 / (1.0 + np.exp(-mref)) if kind == "logistic" else mref
            assert np.min(np.abs(score - t)) > 1e-12
            ev = ds.evaluate(_grad(agd, kind), w, b, t)
            got = [ev.count, ev.loss_sum, ev.tp, ev.fp, ev.tn, ev.fn, ev.sum_err, ev.sum_err2, ev.sum_abs_err, ev.sum_y,
                   ev.sum_y2]
            for k, (g, (r, mag)) in enumerate(zip(got, eval_reference(kind, mref, ys, t))):
                if k in (0, 2, 3, 4, 5):
                    assert g == r, (kind, k, g, r)
                else:
                    assert abs(g - r) <= 1e-12 * mag, (kind, k, g, r, mag)
    finally:
        ds.close()
