"""Views of the resident shards on the GPU: the device mask against the Python restatement, splits that partition the rows,
every gradient kernel on a view against the reference on the host-compacted rows, whole runs on views, excluded rows with
+-inf / NaN features, filter hygiene, and LIBSVM -> randomSplit -> train -> evaluate."""
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
    "ring-f64-1024": ("f64", 1024, {"k1_variant": "ring"}),
    "ring-bf16-1024": ("bf16", 1024, {"k1_variant": "ring"}),
    "generic-f32-1024": ("f32", 1024, {"k1_variant": "generic"}),
    "generic-f32-20000": ("f32", 20000, {}),
    "wgmma-1024": ("bf16", 1024, {"k1_variant": "tc"}),
    "wgmma-4096": ("bf16", 4096, {"k1_variant": "tc"}),
    "csr-f32-pipelined": ("csr-f32", 1024, {"ring_rows": 0}),
    "csr-f32-simple": ("csr-f32", 1024, {"ring_rows": 1}),
    "csr-f64-pipelined": ("csr-f64", 1024, {"ring_rows": 0}),
    "csr-f64-simple": ("csr-f64", 1024, {"ring_rows": 1}),
}
LOSSES = ["logistic", "least_squares", "hinge", "least_squares_half"]


def gradient(agd, kind):
    return {"logistic": agd.LogisticGradient(), "least_squares": agd.LeastSquaresGradient(),
            "hinge": agd.HingeGradient(), "least_squares_half": agd.LeastSquaresGradient(half=True)}[kind]


def make(name, n=None, seed=0):
    """(X as loaded, X as stored, y, w, csr as loaded / stored or None)."""
    store, d, _ = KERNELS[name]
    n = n or (400 if d > 4096 else 6007)
    rng = np.random.default_rng(seed + d)
    X = rng.standard_normal((n, d)).astype(np.float32)
    if store == "bf16":
        X = R.bf16_to_f32(R.f32_to_bf16_bits(X))
    w = rng.standard_normal(d) / np.sqrt(d)
    y = (X.astype(np.float64) @ w + rng.logistic(size=n) > 0).astype(np.float64)
    Xs = X.astype(np.float64) if store.endswith("f64") else X
    csr = None
    if store.startswith("csr"):
        keep = rng.random(X.shape) < 0.05
        rowptr = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
        csr = (rowptr, np.nonzero(keep)[1].astype(np.int32), Xs[keep])
    return X, Xs, y, w, csr


def load(ctx, name, X, y, csr):
    store, d, opts = KERNELS[name]
    ds = ctx.parallelize_csr(y, *csr, d, store=store[4:]) if csr is not None else ctx.parallelize(y, X, store=store)
    for k, v in opts.items():
        ds.set_option(k, v)
    return ds


def compact_csr(csr, mask):
    rowptr, idx, val = csr
    rows = np.nonzero(mask)[0]
    sel = np.concatenate([np.arange(rowptr[r], rowptr[r + 1]) for r in rows]) if rows.size else np.zeros(0, np.int64)
    rp = np.concatenate([[0], np.cumsum(rowptr[rows + 1] - rowptr[rows])]).astype(np.int64)
    return rp, idx[sel], val[sel]


def reference(kind, y, w, Xs, csr, mask):
    if csr is not None:
        return R.fold_shard(kind, y[mask], w, csr=compact_csr(csr, mask))
    return R.fold_shard(kind, y[mask], w, X=Xs[mask])


def check(name, got, ref, kind, Xs, y, w, mask):
    loss, g, cnt = got
    lref, cref, gref = ref
    assert cnt == cref
    if name.startswith("wgmma"):
        gb, lb, _ = R.dense_bounds(kind, Xs[mask], y[mask], w)
        assert np.all(np.abs(g - gref / cref) <= gb)
        assert abs(loss - lref / cref) <= lb
        return
    gr = gref / cref
    np.testing.assert_allclose(g, gr, rtol=0, atol=1e-12 * max(np.max(np.abs(gr)), 1e-300))
    assert abs(loss - lref / cref) <= 1e-12 * abs(lref / cref) + 1e-300


# ---------------------------------------------------------------- the mask
@pytest.mark.parametrize("first_rank,world", [(0, 1), (2, 3), (5, 7)])
def test_mask_matches_restatement_loaded(agd, first_rank, world):
    """Loaded shards number their rows rank << 40: the device mask equals the Python restatement at every row_base."""
    ctx = agd.Context(devices=[0], world_size=world, first_rank=first_rank,
                      handle_exchange=(lambda b: b) if world > 1 else None, transport="ipc" if world > 1 else None)
    n = 3001
    ds = ctx.parallelize(np.zeros(n), np.ones((n, 4), np.float32), store="f32")
    base = first_rank << 40
    for view in (ds.sample(False, 0.3, seed=7), ds.randomSplit([0.5, 0.25, 0.25], seed=1 << 40)[1],
                 agd.MLUtils.kFold(ds.sample(False, 0.9, seed=3), 4, seed=0xFFFFFFFFFFFFFFFF)[2][0]):
        ref = view_mask(view._preds, base, n)
        assert np.array_equal(view.row_mask(0, 0, n), ref)
        assert np.array_equal(view.row_mask(0, 1000, 77), ref[1000:1077])
    assert np.all(ds.row_mask(0, 0, n))             # no view: every row
    ds.close()


@pytest.mark.parametrize("total,world,rank", [(5000, 1, 0), (5000, 3, 2), (7001, 4, 1)])
def test_mask_matches_restatement_generated(agd, total, world, rank):
    """Generated shards number their rows globally: the mask is the restatement at the shard's first global row."""
    ctx = agd.Context(devices=[0], world_size=world, first_rank=rank,
                      handle_exchange=(lambda b: b) if world > 1 else None, transport="ipc" if world > 1 else None)
    ds = ctx.synthetic(total, 16, agd.LogisticGradient(), store="f32")
    lo, hi = rank * total // world, (rank + 1) * total // world
    v = ds.sample(False, 0.6, seed=99)
    assert np.array_equal(v.row_mask(0, 0, hi - lo), view_mask(v._preds, lo, hi - lo))
    ds.close()


def test_filter_arguments_refused(agd, ctx):
    import ctypes as C
    ds = ctx.parallelize(np.zeros(10), np.ones((10, 4), np.float32), store="f32")
    L = agd._native.lib()

    def setf(n, seeds, lo, hi, comp):
        a = [np.asarray(x, dtype=t) for x, t in ((seeds, np.uint64), (lo, np.float64), (hi, np.float64), (comp, np.int32))]
        return L.agd_set_row_filter(ds.h, n, *(x.ctypes.data_as(C.c_void_p) for x in a))

    for bad in [(5, [1] * 5, [0] * 5, [1] * 5, [0] * 5), (-1, [1], [0], [1], [0]), (1, [1], [0.5], [0.4], [0]),
                (1, [1], [-0.1], [0.5], [0]), (1, [1], [0.0], [1.5], [0]), (1, [1], [NAN], [0.5], [0]),
                (1, [1], [0.0], [0.5], [2])]:
        assert setf(*bad) != 0
        assert L.agd_last_error(ds.h)
    assert L.agd_row_filter_mask(ds.h, 0, 5, 6, None) != 0        # outside the shard
    assert setf(4, [1] * 4, [0] * 4, [1] * 4, [0] * 4) == 0
    assert L.agd_set_row_filter(ds.h, 0, None, None, None, None) == 0
    ds.close()


# ---------------------------------------------------------------- splits partition the rows
@pytest.mark.parametrize("name", ["ring-f32-1024", "csr-f64-pipelined"])
def test_random_split_partitions(agd, ctx, name):
    X, Xs, y, w, csr = make(name)
    ds = load(ctx, name, X, y, csr)
    parts = ds.randomSplit([0.6, 0.3, 0.1], seed=2024)
    masks = [p.row_mask(0, 0, len(y)) for p in parts]
    assert np.array_equal(np.sum(masks, axis=0), np.ones(len(y)))     # disjoint and covering, exactly
    counts = [p.count() for p in parts]
    assert counts == [int(m.sum()) for m in masks] and sum(counts) == ds.count() == len(y)
    grad = agd.LogisticGradient()
    lw, gw, cw = ds.smooth(grad, w)
    ls = [p.smooth(grad, w) for p in parts]
    assert sum(c for _, _, c in ls) == cw
    np.testing.assert_allclose(sum(l * c for l, _, c in ls), lw * cw, rtol=1e-12)
    np.testing.assert_allclose(sum(g * c for _, g, c in ls), gw * cw, rtol=0, atol=1e-12 * np.max(np.abs(gw * cw)))
    ev = ds.evaluate(grad, w)
    evs = [p.evaluate(grad, w) for p in parts]
    assert sum(e.count for e in evs) == ev.count and sum(e.tp + e.fp + e.tn + e.fn for e in evs) == ev.count
    np.testing.assert_allclose(sum(e.loss_sum for e in evs), ev.loss_sum, rtol=1e-12)
    # margins of a view are its own rows, in load order
    m = ds.margins(w)
    for p, mk in zip(parts, masks):
        assert np.array_equal(p.margins(w), m[mk])
    ds.close()


# ---------------------------------------------------------------- every kernel on a view
@pytest.mark.parametrize("kind", LOSSES)
@pytest.mark.parametrize("name", list(KERNELS))
def test_smooth_on_view(agd, ctx, name, kind):
    X, Xs, y, w, csr = make(name, seed=1)
    ds = load(ctx, name, X, y, csr)
    v = ds.randomSplit([0.7, 0.3], seed=5)[0].sample(False, 0.8, seed=6)     # two predicates
    mask = view_mask(v._preds, 0, len(y))
    ref = reference(kind, y, w, Xs, csr, mask)
    check(name, v.smooth(gradient(agd, kind), w), ref, kind, Xs, y, w, mask)
    before = ds.smooth(gradient(agd, kind), w)
    if name in ("ring-f32-1024", "ring-f64-1024", "wgmma-1024") and kind in ("logistic", "hinge"):
        l, g, c, l2 = v.smooth_pair(gradient(agd, kind), w, 0.5 * w)        # one filter for both points
        assert (l, c) == v.smooth(gradient(agd, kind), w)[::2] and np.array_equal(g, v.smooth(gradient(agd, kind), w)[1])
        assert l2 == v.smooth(gradient(agd, kind), 0.5 * w)[0]
        l, g, c, l2, g2 = v.smooth_two(gradient(agd, kind), w, 0.5 * w)
        s2 = v.smooth(gradient(agd, kind), 0.5 * w)
        assert l2 == s2[0] and np.array_equal(g2, s2[1])
    after = ds.smooth(gradient(agd, kind), w)                                # the parent never sees the view's filter
    assert before[2] == after[2] == len(y)
    if csr is None:
        assert before[0] == after[0] and np.array_equal(before[1], after[1])
    else:   # the CSR gradient is summed with atomics: reproducible to fp64 rounding, not to the bit
        assert abs(before[0] - after[0]) <= 1e-13 * abs(before[0])
        np.testing.assert_allclose(after[1], before[1], rtol=0, atol=1e-13 * np.max(np.abs(before[1])))
    ds.close()


# ---------------------------------------------------------------- excluded rows with +-inf / NaN
@pytest.mark.parametrize("name", list(KERNELS))
def test_excluded_rows_leave_no_trace(agd, ctx, name):
    X, Xs, y, w, csr = make(name, seed=2)
    n, d = X.shape
    keep = view_mask(((11, 0.0, 0.75, False),), 0, n)
    out = np.nonzero(~keep)[0]
    T = 16
    targets = sorted({int(out[np.argmin(np.abs(out - t))]) for t in (0, T - 1, 3 * T + 2, n // 2, n - 1, 132 * T + 5)})
    Xp, Xsp = X.copy(), np.array(Xs, copy=True)
    for t, i in enumerate(targets):
        v = (INF, -INF, NAN)[t % 3]
        Xp[i, 1 + t % 7] = v
        Xsp[i, 1 + t % 7] = v
    c = None
    if csr is not None:
        nz = (np.random.default_rng(4).random(Xsp.shape) < 0.05) | ~np.isfinite(Xsp)
        rowptr = np.concatenate([[0], np.cumsum(nz.sum(axis=1))]).astype(np.int64)
        c = (rowptr, np.nonzero(nz)[1].astype(np.int32), Xsp[nz])
    ds = load(ctx, name, Xp, y, c)
    v = ds.sample(False, 0.75, seed=11)
    assert np.array_equal(v.row_mask(0, 0, n), keep)
    for kind in ("logistic", "hinge"):
        got = v.smooth(gradient(agd, kind), w)
        assert np.all(np.isfinite(got[1])) and np.isfinite(got[0])
        check(name, got, reference(kind, y, w, Xsp, c, keep), kind, Xsp, y, w, keep)
        ev = v.evaluate(gradient(agd, kind), w)
        assert all(np.isfinite(list(ev.__dict__.values())))
        assert ev.count == keep.sum()
    ds.close()


# ---------------------------------------------------------------- whole runs on views
@pytest.mark.parametrize("name", ["ring-f32-1024", "ring-f64-1024", "generic-f32-1024", "wgmma-1024", "csr-f32-pipelined"])
def test_agd_run_on_view(agd, ctx, oracle, name):
    X, Xs, y, w, csr = make(name, seed=3)
    ds = load(ctx, name, X, y, csr)
    d = KERNELS[name][1]
    train = agd.MLUtils.kFold(ds, 3, seed=17)[1][0]
    mask = view_mask(train._preds, 0, len(y))
    args = (train, agd.LogisticGradient(), agd.SquaredL2Updater(), 0.0, 6, 0.05, np.zeros(d))
    wf, hf, sf = agd.run_with_stats(*args)
    wu, hu, su = agd.run_with_stats(*args, fuse=False)
    wm, hm, sm = agd.run_with_stats(*args, memoize=True)
    if csr is None:
        assert np.array_equal(wf, wu) and np.array_equal(hf, hu)
        assert np.array_equal(wf, wm) and np.array_equal(hf, hm)
    D = oracle.Data(y[mask], csr=compact_csr(csr, mask), d=d) if csr is not None else oracle.Data(y[mask], X=Xs[mask])
    ref = oracle.agd_run(D, "logistic", "squared_l2", np.zeros(d), convergence_tol=0.0, num_iterations=6, reg_param=0.05,
                         partitions=1)
    tol = 1e-6 if name.startswith("wgmma") else 1e-9
    np.testing.assert_allclose(hf, ref.loss_history, rtol=tol)
    assert np.linalg.norm(wf - ref.weights) <= tol * np.linalg.norm(ref.weights)
    assert (su.passes, su.backtracks, su.restarts) == (ref.passes, ref.backtracks, ref.restarts)
    # mini-batch SGD on the view: a row must pass the view and the mini-batch mask
    wg, hg = agd.GradientDescent.runMiniBatchSGD(train, agd.LeastSquaresGradient(), agd.SquaredL2Updater(), 0.1, 4, 0.01,
                                                  0.5, np.zeros(d))
    # a row of the run must pass the view and the mini-batch mask of its iteration (the oracle numbers the compacted rows
    # afresh, so the host restatement folds the rows both masks keep, by their global ids)
    w_h = np.zeros(d)
    ids = np.arange(len(y))
    thresh = int(np.ldexp(0.5, 64))
    for i in range(1, 5):
        sel = R.row_selected(42 + i, thresh, ids) & mask
        if csr is not None:
            l, cnt, g = R.fold_shard("least_squares", y[sel], w_h, csr=compact_csr(csr, sel))
        else:
            l, cnt, g = R.fold_shard("least_squares", y[sel], w_h, X=Xs[sel])
        step = 0.1 / np.sqrt(i)
        w_h = w_h * (1.0 - step * 0.01) - step * (g / cnt)
    tolg = 1e-6 if name.startswith("wgmma") else 1e-9
    assert np.linalg.norm(wg - w_h) <= tolg * np.linalg.norm(w_h)
    ds.close()


# ---------------------------------------------------------------- filter hygiene
def test_filter_hygiene(agd, ctx):
    import ctypes as C
    X, Xs, y, w, _ = make("ring-f32-1024", seed=4)
    ds = ctx.parallelize(y, X, store="f32")
    grad = agd.LogisticGradient()
    base = ds.smooth(grad, w)
    base_ev = ds.evaluate(grad, w)
    whole = ds.sample(False, 1.0, seed=3)                           # [0, 1): every row, the same bits as no filter
    s = whole.smooth(grad, w)
    assert s[0] == base[0] and s[2] == base[2] and np.array_equal(s[1], base[1])
    assert whole.evaluate(grad, w) == base_ev
    L = agd._native.lib()
    seeds, lo, hi, comp = (np.array([1], np.uint64), np.array([0.2]), np.array([0.4]), np.array([0], np.int32))
    assert L.agd_set_row_filter(ds.h, 1, *(a.ctypes.data_as(C.c_void_p) for a in (seeds, lo, hi, comp))) == 0
    assert L.agd_set_row_filter(ds.h, 0, None, None, None, None) == 0     # n = 0: as if there never was a filter
    s = ds.smooth(grad, w)
    assert s[0] == base[0] and np.array_equal(s[1], base[1])
    wb, hb, _ = agd.run_with_stats(ds, grad, agd.SquaredL2Updater(), 0.0, 4, 0.05, np.zeros(1024))
    part = ds.sample(False, 0.3, seed=8)
    part.smooth(grad, w)
    agd.run_with_stats(part, grad, agd.SquaredL2Updater(), 0.0, 4, 0.05, np.zeros(1024))
    with pytest.raises(RuntimeError):
        with part._filtered():                                         # an error inside a view call clears the filter too
            raise RuntimeError("failed inside a view call")
    wa, ha, _ = agd.run_with_stats(ds, grad, agd.SquaredL2Updater(), 0.0, 4, 0.05, np.zeros(1024))
    assert np.array_equal(wa, wb) and np.array_equal(ha, hb)           # the parent after view calls: the same bits
    assert ds.evaluate(grad, w) == base_ev
    part.close()                                                       # frees nothing
    assert ds.count() == len(y)
    empty = ds.sample(False, 0.0)                                      # behaves as an empty RDD
    assert empty.count() == 0
    l, g, c = empty.smooth(grad, w)
    assert c == 0 and np.isnan(l)
    _, hist, st = agd.run_with_stats(empty, grad, agd.SquaredL2Updater(), 0.0, 4, 0.05, np.zeros(1024))
    assert st.nonterminating
    ds.close()


# ---------------------------------------------------------------- end to end
def _libsvm(tmp_path, n=3000, d=60, seed=0):
    rng = np.random.default_rng(seed)
    wt = rng.standard_normal(d)
    lines, rows = [], []
    for _ in range(n):
        cols = np.sort(rng.choice(d, size=8, replace=False))
        vals = rng.standard_normal(8)
        y = 1.0 if vals @ wt[cols] + 0.3 * rng.standard_normal() > 0 else 0.0
        lines.append(f"{y:g} " + " ".join(f"{c + 1}:{float(v)!r}" for c, v in zip(cols, vals)))
    p = tmp_path / "data.libsvm"
    p.write_text("\n".join(lines) + "\n")
    return str(p)


def test_libsvm_split_train_evaluate(agd, ctx, tmp_path):
    path = _libsvm(tmp_path)
    labels, rowptr, idx, val, d = agd.MLUtils.parseLibSVMFile(path)
    data = agd.MLUtils.loadLibSVMFile(ctx, path)
    train, test = data.randomSplit([0.8, 0.2], seed=13)
    model = agd.SVMWithAGD(numIterations=20, regParam=0.01).run(train)
    ev = model.evaluate(test)
    X = np.zeros((len(labels), d))
    for r in range(len(labels)):
        X[r, idx[rowptr[r]:rowptr[r + 1]]] = val[rowptr[r]:rowptr[r + 1]]
    mask = view_mask(test._preds, 0, len(labels))
    m = X[mask] @ model.weights
    yt = labels[mask]
    pos = m > 0.0
    assert (ev.tp, ev.fp, ev.tn, ev.fn) == ((pos & (yt == 1)).sum(), (pos & (yt == 0)).sum(), (~pos & (yt == 0)).sum(),
                                            (~pos & (yt == 1)).sum())
    assert ev.accuracy == (pos == (yt == 1)).mean() and ev.count == mask.sum()
    np.testing.assert_allclose(model.predict(test), pos.astype(np.float64))
    accs = []
    for tr, va in agd.MLUtils.kFold(data, 3, seed=21):
        mdl = agd.LogisticRegressionWithAGD(numIterations=15).run(tr)
        e = mdl.evaluate(va)
        vm = view_mask(va._preds, 0, len(labels))
        assert e.count == vm.sum() and tr.count() == len(labels) - vm.sum()
        p = 1.0 / (1.0 + np.exp(-(X[vm] @ mdl.weights))) > 0.5
        assert e.tp == (p & (labels[vm] == 1)).sum() and e.tn == (~p & (labels[vm] == 0)).sum()
        accs.append(e.accuracy)
    assert min(accs) > 0.7
    data.close()


@pytest.mark.parametrize("name", ["ring-f32-1024", "wgmma-1024"])
def test_view_follows_appended_rows_and_filter_changes(agd, ctx, name):
    """The ring and wgmma kernels read the view as a bitmap of the shard's rows: it must follow rows appended after a view
    call and a change of view between calls on the same shard."""
    X, Xs, y, w, _ = make(name, seed=6)
    half = len(y) // 2
    ds = load(ctx, name, X[:half], y[:half], None)
    grad = agd.LogisticGradient()
    a, b = ds.sample(False, 0.5, seed=1), ds.sample(False, 0.5, seed=2)
    for v in (a, b, a):
        m = view_mask(v._preds, 0, half)
        check(name, v.smooth(grad, w), reference("logistic", y[:half], w, Xs[:half], None, m), "logistic", Xs[:half],
              y[:half], w, m)
    ds.load_dense(y[half:], X[half:], store=KERNELS[name][0])
    m = view_mask(a._preds, 0, len(y))
    check(name, a.smooth(grad, w), reference("logistic", y, w, Xs, None, m), "logistic", Xs, y, w, m)
    ds.close()
