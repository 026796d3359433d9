"""A second, independent restatement of the reference's whole path in pure Python (explicit loops, Python floats = IEEE fp64, no
FMA): AcceleratedGradientDescent.run (AGD.scala:177-338) on top of the [mllib-1.3.0] Gradient / Updater formulas, with the
same evaluation order the C oracle documents (sequential dot / axpy per row, ParallelCollectionRDD slices folded in partition
order).  The C oracle must reproduce it BIT FOR BIT on small problems, including every branch count -- two independent
readings of the Scala agreeing to the last bit is the strongest pin available without a JVM."""
import math

import numpy as np
import pytest

INF = float("inf")


def log1p_exp(x):                                   # MLUtils.log1pExp [mllib-1.3.0]
    return x + math.log1p(math.exp(-x)) if x > 0 else math.log1p(math.exp(x))


def axpy(a, x, cum):                                # dense BLAS.axpy: netlib DAXPY, which starts with IF (DA.EQ.0) RETURN
    if a == 0.0:
        return
    for j in range(len(x)):
        cum[j] += a * x[j]


def gradient_compute(kind, x, label, w, cum):       # Gradient.compute(data, label, weights, cumGradient): Double
    dot = 0.0
    for j in range(len(x)):
        dot += x[j] * w[j]
    if kind == "logistic":
        margin = -1.0 * dot
        mult = (1.0 / (1.0 + math.exp(margin))) - label
        axpy(mult, x, cum)
        return log1p_exp(margin) if label > 0 else log1p_exp(margin) - margin
    if kind == "least_squares":
        diff = dot - label
        axpy(2.0 * diff, x, cum)
        return diff * diff
    s = 2 * label - 1.0                             # hinge
    if 1.0 > s * dot:
        axpy(-s, x, cum)
        return 1.0 - s * dot
    return 0.0


def updater_compute(kind, w, g, step, reg):         # Updater.compute(weightsOld, gradient, stepSize, iter = 1, regParam)
    if kind == "simple":
        return [w[j] + (-step) * g[j] for j in range(len(w))], 0.0
    if kind == "squared_l2":
        scale = 1.0 - step * reg
        out = [w[j] * scale for j in range(len(w))]
        for j in range(len(w)):
            out[j] += (-step) * g[j]
        nrm = math.sqrt(sum_seq(v * v for v in out))
        return out, 0.5 * reg * nrm * nrm
    out = [w[j] + (-step) * g[j] for j in range(len(w))]          # L1
    shrink = reg * step
    out = [math.copysign(1.0, v) * max(0.0, abs(v) - shrink) if v != 0.0 else 0.0 for v in out]
    return out, sum_seq(abs(v) for v in out) * reg


def sum_seq(it):
    s = 0.0
    for v in it:
        s += v
    return s


def vdot(a, b):
    return sum_seq(a[j] * b[j] for j in range(len(a)))


def vnorm(a):
    return math.sqrt(sum_seq(v * v for v in a))


def py_agd_run(X, y, grad, upd, w0, tol, iters, reg, L0=1.0, Lexact=INF, beta=0.5, alpha=0.9, may_restart=True, parts=2):
    n, d = len(X), len(w0)
    stats = dict(passes=0, backtracks=0, restarts=0)

    def apply_smooth(w):                            # AGD.scala:192-208
        stats["passes"] += 1
        partials = []
        for p in range(parts):                      # ParallelCollectionRDD.slice
            lo, hi = (p * n) // parts, ((p + 1) * n) // parts
            loss, g, cnt = 0.0, [0.0] * d, 0
            for i in range(lo, hi):
                loss = loss + gradient_compute(grad, X[i], y[i], w, g)
                cnt += 1
            partials.append((loss, g, cnt))
        loss, g, cnt = partials[0]
        for l2, g2, c2 in partials[1:]:             # combOp, folded in partition order
            loss, g, cnt = loss + l2, [g[j] + g2[j] for j in range(d)], cnt + c2
        return loss / cnt, [v / float(cnt) for v in g]

    x, z, theta, hist = list(w0), list(w0), INF, []
    f_y, g_y, L, simple = 0.0, [0.0] * d, L0, True
    for n_iter in range(1, iters + 1):
        x_old, z_old, L_old = x, z, L
        L = L * alpha
        theta_old = theta
        while True:
            theta = 2.0 / (1.0 + math.sqrt(1.0 + 4.0 * (L / L_old) / (theta_old * theta_old)))
            yv = [x_old[j] * (1.0 - theta) + z_old[j] * theta for j in range(d)]
            f_y, g_y = apply_smooth(yv)
            step = 1.0 / (theta * L)
            z, _ = updater_compute(upd, z_old, g_y, step, reg)
            x = [x_old[j] * (1.0 - theta) + z[j] * theta for j in range(d)]
            if beta >= 1.0:
                break
            xy = [x[j] - yv[j] for j in range(d)]
            nxy = vnorm(xy)
            xy_sq = nxy * nxy
            if xy_sq == 0:
                break
            f_x, g_x = apply_smooth(x)
            if simple:
                q_x = f_y + vdot(xy, g_y) + 0.5 * L * xy_sq
                local_l = L + 2.0 * max(f_x - q_x, 0.0) / xy_sq
                simple = abs(f_y - f_x) >= 1e-10 * max(abs(f_x), abs(f_y))
            else:
                local_l = 2.0 * vdot(xy, [g_x[j] - g_y[j] for j in range(d)]) / xy_sq
            if local_l <= L or L >= Lexact:
                break
            if not math.isinf(local_l):
                L = min(Lexact, local_l)
            else:
                local_l = L
            L = min(Lexact, max(local_l, L / beta))
            stats["backtracks"] += 1
        f_x, g_x = apply_smooth(x)
        _, c_x = updater_compute(upd, x, g_x, 0.0, reg)
        hist.append(f_x + c_x)
        if math.isnan(f_y) or math.isinf(f_y):
            break
        norm_x, norm_dx = vnorm(x), vnorm([x[j] - x_old[j] for j in range(d)])
        if norm_dx == 0.0 and n_iter > 1:
            break
        if norm_dx < tol * max(norm_x, 1):
            break
        if may_restart and vdot(g_y, [x[j] - x_old[j] for j in range(d)]) > 0.0:
            z, theta, simple = x, INF, True
            stats["restarts"] += 1
    return x, hist, stats


def make(rng, n, d, grad):
    X = rng.standard_normal((n, d))
    wt = rng.standard_normal(d)
    m = X @ wt
    y = m + 0.3 * rng.standard_normal(n) if grad == "least_squares" else (m + rng.logistic(size=n) > 0).astype(float)
    return X, y


CASES = [("logistic", "simple", 0.0, {}), ("logistic", "squared_l2", 0.1, {}), ("logistic", "l1", 0.02, {}),
         ("least_squares", "simple", 0.0, {"L0": 1e-3}), ("least_squares", "squared_l2", 0.05, {"may_restart": False}),
         ("least_squares", "l1", 0.05, {"L0": 0.01, "Lexact": 4.0}), ("hinge", "squared_l2", 0.1, {}),
         ("hinge", "simple", 0.0, {"beta": 1.0, "L0": 2.0, "Lexact": 2.0}), ("logistic", "simple", 0.0, {"tol": 1e-3, "parts": 3})]


@pytest.mark.parametrize("grad,upd,reg,kw", CASES, ids=[f"{c[0]}-{c[1]}-{i}" for i, c in enumerate(CASES)])
def test_c_oracle_equals_python_restatement_bit_for_bit(oracle, grad, upd, reg, kw):
    rng = np.random.default_rng(len(grad) * 31 + len(upd))
    n, d, iters = 120, 5, 25
    X, y = make(rng, n, d, grad)
    w0 = [0.0] * d
    parts = kw.get("parts", 2)
    w, hist, st = py_agd_run(X.tolist(), y.tolist(), grad, upd, w0, kw.get("tol", 0.0), iters, reg, kw.get("L0", 1.0),
                             kw.get("Lexact", INF), kw.get("beta", 0.5), kw.get("alpha", 0.9), kw.get("may_restart", True), parts)
    ref = oracle.agd_run(oracle.Data(y, X=X), grad, upd, np.zeros(d), convergence_tol=kw.get("tol", 0.0), num_iterations=iters,
                         reg_param=reg, L0=kw.get("L0", 1.0), Lexact=kw.get("Lexact", INF), beta=kw.get("beta", 0.5),
                         alpha=kw.get("alpha", 0.9), may_restart=kw.get("may_restart", True), partitions=parts)
    assert len(hist) == ref.iterations == len(ref.loss_history)
    assert (st["passes"], st["backtracks"], st["restarts"]) == (ref.passes, ref.backtracks, ref.restarts)
    assert np.array_equal(np.array(hist), ref.loss_history)
    assert np.array_equal(np.array(w), ref.weights)


def py_gd_run(X, y, grad, upd, w0, step_size, iters, reg, parts=2):
    """GradientDescent.runMiniBatchSGD [mllib-1.3.0] with miniBatchFraction = 1.0 (the comparator of Suite.scala:78,118,225)."""
    n, d = len(X), len(w0)
    w = list(w0)
    _, reg_val = updater_compute(upd, w, [0.0] * d, 0.0, reg)
    hist = []
    for i in range(1, iters + 1):
        partials = []
        for p in range(parts):
            lo, hi = (p * n) // parts, ((p + 1) * n) // parts
            loss, g, cnt = 0.0, [0.0] * d, 0
            for r in range(lo, hi):
                loss = loss + gradient_compute(grad, X[r], y[r], w, g)
                cnt += 1
            partials.append((loss, g, cnt))
        loss, g, cnt = partials[0]
        for l2, g2, c2 in partials[1:]:
            loss, g, cnt = loss + l2, [g[j] + g2[j] for j in range(d)], cnt + c2
        hist.append(loss / cnt + reg_val)
        w, reg_val = updater_compute(upd, w, [v / float(cnt) for v in g], step_size / math.sqrt(i), reg)
    return w, hist


@pytest.mark.parametrize("grad,upd,reg", [("logistic", "simple", 0.0), ("logistic", "squared_l2", 0.2), ("least_squares", "l1", 0.05),
                                          ("hinge", "squared_l2", 0.1)])
def test_c_oracle_gd_equals_python_restatement_bit_for_bit(oracle, grad, upd, reg):
    rng = np.random.default_rng(len(grad) + 7 * len(upd))
    X, y = make(rng, 90, 4, grad)
    w, hist = py_gd_run(X.tolist(), y.tolist(), grad, upd, [0.1, -0.2, 0.0, 0.3], 0.5, 30, reg)
    rw, rhist = oracle.gd_run(oracle.Data(y, X=X), grad, upd, np.array([0.1, -0.2, 0.0, 0.3]), step_size=0.5, num_iterations=30,
                              reg_param=reg, partitions=2)
    assert np.array_equal(np.array(hist), rhist) and np.array_equal(np.array(w), rw)


def test_c_oracle_sparse_rows_equal_python_on_the_densified_matrix(oracle):
    """SparseVector rows take the sparse branches of BLAS.dot / BLAS.axpy [mllib-1.3.0] (stored entries only, index order).
    Skipped zeros contribute exact zeros, so the CSR oracle must match the dense Python restatement bit for bit."""
    rng = np.random.default_rng(99)
    n, d, k = 80, 12, 4
    idx = np.sort(np.stack([rng.choice(d, k, replace=False) for _ in range(n)]), axis=1).astype(np.int32)
    val = rng.standard_normal((n, k))
    rowptr = np.arange(n + 1, dtype=np.int64) * k
    Xd = np.zeros((n, d))
    for i in range(n):
        Xd[i, idx[i]] = val[i]
    y = (Xd @ rng.standard_normal(d) > 0).astype(float)
    for grad, upd, reg in (("hinge", "squared_l2", 0.1), ("logistic", "l1", 0.01)):
        w, hist, st = py_agd_run(Xd.tolist(), y.tolist(), grad, upd, [0.0] * d, 0.0, 20, reg)
        ref = oracle.agd_run(oracle.Data(y, csr=(rowptr, idx.ravel(), val.ravel()), d=d), grad, upd, np.zeros(d),
                             convergence_tol=0.0, num_iterations=20, reg_param=reg, partitions=2)
        assert (st["passes"], st["backtracks"], st["restarts"]) == (ref.passes, ref.backtracks, ref.restarts)
        assert np.array_equal(np.array(hist), ref.loss_history) and np.array_equal(np.array(w), ref.weights)
