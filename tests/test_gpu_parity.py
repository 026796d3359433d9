"""Parity of the CUDA path (through the C-ABI) against the CPU oracle on identical inputs.

Tolerances: the element-wise vector arithmetic is bit-faithful; reductions differ only in fp64
summation order, so losses agree to ~1e-13 relative and trajectories (weights after equal
iterations) to <= 1e-9 relative -- far inside north_star's 1e-5 bound, which is also asserted."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import k1_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

GRADS = ["logistic", "least_squares", "hinge"]
UPDS = ["simple", "squared_l2", "l1"]


def G(agd, name):
    return {"logistic": agd.LogisticGradient(), "least_squares": agd.LeastSquaresGradient(),
            "hinge": agd.HingeGradient(), "least_squares_half": agd.LeastSquaresGradient(half=True)}[name]


def U(agd, name):
    return {"simple": agd.SimpleUpdater(), "squared_l2": agd.SquaredL2Updater(), "l1": agd.L1Updater()}[name]


def make_data(rng, n, d, grad, dtype):
    X = rng.standard_normal((n, d)).astype(dtype)
    wt = rng.standard_normal(d) / np.sqrt(d)
    m = X.astype(np.float64) @ wt
    if grad == "least_squares" or grad == "least_squares_half":
        y = m + 0.1 * rng.standard_normal(n)
    else:
        y = (m + rng.logistic(size=n) > 0).astype(np.float64)
    return X, y


def rel_err(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


# ------------------------------------------------------------------ applySmooth (K1 + reduce)
SHAPES = [(1000, 100), (10000, 2), (3001, 1024), (2000, 512), (515, 256), (260, 128), (777, 2048), (300, 4096),
          (129, 1100), (10, 20000), (37, 36), (1, 1024), (7, 1024), (501, 1001), (300, 37), (64, 4095), (90, 3)]


@pytest.mark.parametrize("grad", GRADS + ["least_squares_half"])
@pytest.mark.parametrize("store", ["f32", "f64"])
@pytest.mark.parametrize("shape", SHAPES)
def test_smooth_matches_oracle(agd, ctx, oracle, grad, store, shape):
    n, d = shape
    rng = np.random.default_rng(1000 + n + d)
    X, y = make_data(rng, n, d, grad, np.float32 if store == "f32" else np.float64)
    w = rng.standard_normal(d) * 0.3 / np.sqrt(d) * 4
    ds = ctx.parallelize(y, X, store=store)
    loss, g, cnt = ds.smooth(G(agd, grad), w)
    ref_loss, ref_g, ref_cnt = oracle.smooth(oracle.Data(y, X=X), grad, w, partitions=2)
    assert cnt == ref_cnt == n
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12)
    assert rel_err(g, ref_g) < 1e-12
    np.testing.assert_allclose(g, ref_g, rtol=1e-9, atol=1e-13 * np.abs(ref_g).max())
    ds.close()


@pytest.mark.parametrize("variant", ["ring", "generic"])
def test_kernel_variants_agree(agd, ctx, oracle, variant):
    rng = np.random.default_rng(5)
    X, y = make_data(rng, 4099, 1024, "logistic", np.float32)
    w = rng.standard_normal(1024) * 0.05
    ds = ctx.parallelize(y, X, store="f32")
    ds.set_option("k1_variant", variant)
    loss, g, _ = ds.smooth(agd.LogisticGradient(), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=X), "logistic", w)
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12)
    assert rel_err(g, ref_g) < 1e-12
    ds.close()


@pytest.mark.parametrize("grad", ["logistic", "hinge"])
@pytest.mark.parametrize("store", ["f32", "f64"])
@pytest.mark.parametrize("shape", [(3001, 1024), (2000, 512), (515, 256), (260, 128), (777, 2048), (300, 4096), (129, 1100),
                                   (1, 1024), (7, 1024), (20011, 1024), (40000, 64)])
def test_ring_kernel_shape_families(agd, ctx, oracle, grad, store, shape):
    """The ring K1 forced onto every shape family it supports (row groups, wide threads, padded rows, 1-row shards)."""
    n, d = shape
    rng = np.random.default_rng(2000 + n + d)
    X, y = make_data(rng, n, d, grad, np.float32 if store == "f32" else np.float64)
    w = rng.standard_normal(d) * 0.3 / np.sqrt(d) * 4
    ds = ctx.parallelize(y, X, store=store)
    if not (store == "f64" and d > 2048):
        ds.set_option("k1_variant", "ring")
    loss, g, cnt = ds.smooth(G(agd, grad), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=X), grad, w, partitions=4, threads=4)
    assert cnt == n
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12)
    assert rel_err(g, ref_g) < 1e-12
    a = ds.smooth(G(agd, grad), w)
    assert a[0] == loss and np.array_equal(a[1], g)      # deterministic
    ds.close()


@pytest.mark.parametrize("rows,ctas,stages", [(8, 2, 0), (8, 1, 0), (4, 2, 0), (4, 3, 0), (8, 2, 1), (8, 2, 2), (4, 4, 0), (4, 5, 0)])
def test_ring_tuning_variants(agd, ctx, oracle, rows, ctas, stages):
    rng = np.random.default_rng(6)
    X, y = make_data(rng, 70001, 1024, "logistic", np.float32)
    w = rng.standard_normal(1024) * 0.05
    ds = ctx.parallelize(y, X, store="f32")
    ds.set_option("ring_rows", rows)
    ds.set_option("ring_ctas", ctas)
    ds.set_option("ring_stages", stages)
    loss, g, _ = ds.smooth(agd.LogisticGradient(), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=X), "logistic", w, partitions=8, threads=8)
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12)
    assert rel_err(g, ref_g) < 1e-12
    ds.close()


def test_smooth_is_deterministic(agd, ctx):
    rng = np.random.default_rng(8)
    X, y = make_data(rng, 50000, 1024, "logistic", np.float32)
    w = rng.standard_normal(1024) * 0.05
    ds = ctx.parallelize(y, X, store="f32")
    a = ds.smooth(agd.LogisticGradient(), w)
    b = ds.smooth(agd.LogisticGradient(), w)
    assert a[0] == b[0] and np.array_equal(a[1], b[1])
    ds.close()


def test_appended_loads_equal_single_load(agd, ctx):
    """Spark hands partitions over one at a time: agd_load_dense appends (with growth)."""
    rng = np.random.default_rng(9)
    X, y = make_data(rng, 1500, 64, "logistic", np.float64)
    w = rng.standard_normal(64) * 0.1
    one = ctx.parallelize(y, X)
    many = agd.DeviceDataset(ctx)
    for lo, hi in [(0, 100), (100, 101), (101, 900), (900, 1500)]:
        many.load_dense(y[lo:hi], X[lo:hi])
    a, b = one.smooth(agd.LogisticGradient(), w), many.smooth(agd.LogisticGradient(), w)
    assert a[2] == b[2] == 1500 and a[0] == b[0] and np.array_equal(a[1], b[1])
    one.close(); many.close()


def test_strided_and_converted_load(agd, ctx, oracle):
    """fp64 source rows with a leading dimension > d, stored as fp32 in HBM."""
    rng = np.random.default_rng(10)
    big = rng.standard_normal((400, 160))
    X = big[:, :128]                      # ld = 160
    y = (rng.random(400) > 0.5).astype(np.float64)
    w = rng.standard_normal(128) * 0.1
    ds = agd.DeviceDataset(ctx)
    import ctypes as C
    N = agd._native
    N.check(N.lib().agd_load_dense(ds.h, 0, big.ctypes.data_as(C.c_void_p), N.F64, y.ctypes.data_as(C.c_void_p),
                                   400, 128, 160, N.F32), ds.h)
    loss, g, _ = ds.smooth(agd.LogisticGradient(), w)
    X32 = np.ascontiguousarray(X.astype(np.float32))
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=X32), "logistic", w)
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12)
    assert rel_err(g, ref_g) < 1e-12
    ds.close()


@pytest.mark.parametrize("scale", [1e-8, 1.0, 30.0, 300.0, 700.0, 2000.0])
@pytest.mark.parametrize("d", [1, 4])
def test_logistic_extreme_margins(agd, ctx, oracle, scale, d):
    """The device sigmoid/softplus (k1_device.cuh: table exp + shared reciprocal + fdlibm-style log)
    against libm through the oracle, from vanishing to saturating margins (exp under/overflow)."""
    rng = np.random.default_rng(77)
    n = 8192
    X = np.zeros((n, d))
    X[:, 0] = np.linspace(-1.0, 1.0, n)
    y = (rng.random(n) > 0.5).astype(np.float64)
    w = np.zeros(d); w[0] = scale
    ds = ctx.parallelize(y, X)
    loss, g, _ = ds.smooth(agd.LogisticGradient(), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=X), "logistic", w)
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-13)
    np.testing.assert_allclose(g[0], ref_g[0], rtol=1e-12)
    ds.close()


# ------------------------------------------------------------------ bf16 storage
def f32_to_bf16_bits(x):
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)       # round to nearest even


def tc_shape(d):
    return d % 128 == 0 and d <= 4096


def assert_within_tc_bounds(record_property, grad, Xs, y, w, f32_margins, loss, g, ref_loss, ref_g):
    """The wgmma kernel's element-wise contract (tests/k1_reference.py): every gradient entry and the loss within the bound
    that the margin error (fp32 margins: 2^-20 sum |x w|) and the bf16 x 3 split with fp32 tile sums (2^-20 sum |x r|) allow."""
    gb, lb, _ = R.dense_bounds(grad, Xs, y, w, f32_margins=f32_margins)
    eg, el = float(np.max(np.abs(g - ref_g) / gb)), abs(loss - ref_loss) / lb
    record_property("grad_normwise", rel_err(g, ref_g))
    record_property("loss_rel", abs(loss - ref_loss) / abs(ref_loss))
    record_property("grad_elementwise_of_bound", eg)
    record_property("loss_of_bound", el)
    assert eg <= 1.0 and el <= 1.0, (eg, el)


@pytest.mark.parametrize("variant", ["auto", "auto-f64", "ring"])
@pytest.mark.parametrize("grad", ["logistic", "least_squares", "hinge"])
@pytest.mark.parametrize("shape", [(3001, 1024), (2000, 512), (515, 256), (777, 2048), (300, 4096), (129, 1104),
                                   (37, 40), (10, 20000), (64, 8192), (5, 3), (4099, 128), (33, 3072), (517, 768),
                                   (260, 640)])
def test_bf16_storage_matches_oracle(agd, ctx, oracle, record_property, grad, shape, variant):
    """X stored as bf16 in HBM (rounded to nearest-even at load).  `ring`/generic: fp64 CUDA-core path, same
    tolerances as fp32 storage.  `auto` on d % 128 == 0, d <= 4096 is the wgmma kernel: X^T r on the tensor cores with r
    split into three bf16 pieces and fp32 partial sums over 16 rows -> gradient to 3e-7 norm-wise and within the
    element-wise bound of tests/k1_reference.py; margins on the CUDA cores, by default in fp32 (w rounded to fp32, packed
    FMAs over at most 8 terms, then fp64) -> loss to 1.5e-7, or fp64-exact with option tc_margins=f64 (`auto-f64`) -> loss
    to 1e-12.  Off the tensor path `auto-f64` checks that the option changes
    nothing, and `ring` forces the generic CUDA-core kernel (auto takes the ring wherever the ring fits)."""
    n, d = shape
    rng = np.random.default_rng(3000 + n + d)
    X, y = make_data(rng, n, d, grad, np.float32)
    w = rng.standard_normal(d) * 0.3 / np.sqrt(d) * 4
    ds = ctx.parallelize(y, X, store="bf16")
    if variant == "ring":
        ds.set_option("k1_variant", "ring" if tc_shape(d) else "generic")
    if variant == "auto-f64":
        ds.set_option("tc_margins", "f64")
    raw, yb = ds.get_rows(0, 0, n, dtype=np.uint16)
    assert np.array_equal(raw, f32_to_bf16_bits(X)) and np.array_equal(yb, y)
    Xs = agd.bf16_to_f32(raw)
    loss, g, cnt = ds.smooth(G(agd, grad), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=Xs), grad, w, partitions=2)
    assert cnt == n
    tensor_path = variant != "ring" and tc_shape(d)
    np.testing.assert_allclose(loss, ref_loss, rtol=1.5e-7 if (tensor_path and variant == "auto") else 1e-12)
    assert rel_err(g, ref_g) < (3e-7 if tensor_path else 1e-12)
    if tensor_path:
        assert_within_tc_bounds(record_property, grad, Xs, y, w, variant == "auto", loss, g, ref_loss, ref_g)
    a = ds.smooth(G(agd, grad), w)
    assert a[0] == loss and np.array_equal(a[1], g)      # deterministic either way
    ds.close()


@pytest.mark.parametrize("rows_opt,copy_opt", [(0, 0), (0, 2), (1, 0), (1, 2), (4, 0), (4, 2)])
@pytest.mark.parametrize("shape,grad", [((3001, 1024), "logistic"), ((300, 4096), "least_squares"), ((515, 256), "hinge"),
                                        ((1000, 128), "logistic"), ((130, 3072), "least_squares"), ((517, 768), "hinge")])
def test_tc_kernel_forms(agd, ctx, oracle, record_property, shape, grad, rows_opt, copy_opt):
    """The wgmma kernel's consumer mappings (ring_rows: 0 = default, two rows per thread of the column-slice mapping; 4 = four
    rows per thread; 1 = row per lane with broadcast w reads) and its two TMA forms (default: one 3-D copy per ring group;
    ring_ctas=2: one 2-D copy per 64-feature block) all meet the tolerances of the tensor path."""
    n, d = shape
    rng = np.random.default_rng(4000 + n + d)
    X, y = make_data(rng, n, d, grad, np.float32)
    w = rng.standard_normal(d) * 0.3 / np.sqrt(d) * 4
    ds = ctx.parallelize(y, X, store="bf16")
    ds.set_option("k1_variant", "tc")
    ds.set_option("ring_rows", rows_opt)
    ds.set_option("ring_ctas", copy_opt)
    raw, _ = ds.get_rows(0, 0, n, dtype=np.uint16)
    loss, g, cnt = ds.smooth(G(agd, grad), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, X=agd.bf16_to_f32(raw)), grad, w, partitions=2)
    assert cnt == n
    np.testing.assert_allclose(loss, ref_loss, rtol=1.5e-7 if rows_opt == 0 else 1e-12)   # default mapping: fp32 margins
    assert rel_err(g, ref_g) < 3e-7
    assert_within_tc_bounds(record_property, grad, agd.bf16_to_f32(raw), y, w, rows_opt == 0, loss, g, ref_loss, ref_g)
    ds.close()


@pytest.mark.parametrize("variant", ["tc", "ring"])
def test_bf16_run_and_generator(agd, ctx, oracle, variant):
    n, d = 20000, 1024
    ds = ctx.synthetic(n, d, agd.LeastSquaresGradient(), seed=7, store="bf16")
    ds.set_option("k1_variant", variant)
    raw, y = ds.get_rows(0, 0, n, dtype=np.uint16)
    assert np.array_equal(raw, f32_to_bf16_bits(oracle.synth_dense_f32(7, 0, n, d)))   # spec value, rounded once
    Xs = agd.bf16_to_f32(raw)
    w0 = np.zeros(d)
    # branch-free configuration for the tensor path (SURVEY.md section 7): beta = 1 skips backtracking
    kw = dict(L0=8.0, Lexact=8.0, beta=1.0, may_restart=False) if variant == "tc" else {}
    w, hist, st = agd.run_with_stats(ds, agd.LeastSquaresGradient(), agd.SquaredL2Updater(), 0.0, 10, 0.01, w0,
                                     kw.get("L0", 1.0), kw.get("Lexact", float("inf")), kw.get("beta", 0.5), 0.9,
                                     kw.get("may_restart", True))
    ref = oracle.agd_run(oracle.Data(y, X=Xs), "least_squares", "squared_l2", w0, convergence_tol=0.0,
                         num_iterations=10, reg_param=0.01, partitions=4, threads=4, L0=kw.get("L0", 1.0),
                         Lexact=kw.get("Lexact", float("inf")), beta=kw.get("beta", 0.5),
                         may_restart=kw.get("may_restart", True))
    if variant == "tc":
        np.testing.assert_allclose(hist, ref.loss_history, rtol=1e-6)
        assert rel_err(w, ref.weights) < 1e-5          # north_star's bound
    else:
        np.testing.assert_allclose(hist, ref.loss_history, rtol=1e-11)
        assert rel_err(w, ref.weights) < 1e-9
    assert st.passes == ref.passes
    ds.close()


# ------------------------------------------------------------------ CSR rows (SparseVector)
@pytest.mark.parametrize("grad", GRADS)
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_csr_smooth_matches_oracle(agd, ctx, oracle, grad, store):
    rng = np.random.default_rng(11)
    n, d = 3000, 5000
    nnz_row = rng.integers(0, 40, size=n)
    nnz_row[5] = 0
    nnz_row[7], nnz_row[8], nnz_row[9], nnz_row[n - 1] = 64, 65, 200, 33      # around the two-entries-per-lane fast path
    rowptr = np.concatenate([[0], np.cumsum(nnz_row)]).astype(np.int64)
    idx = np.concatenate([np.sort(rng.choice(d, size=k, replace=False)) for k in nnz_row]).astype(np.int32)
    val = rng.standard_normal(rowptr[-1]).astype(np.float32 if store == "f32" else np.float64)
    y = (rng.random(n) > 0.5).astype(np.float64)
    w = rng.standard_normal(d) * 0.2
    ds = ctx.parallelize_csr(y, rowptr, idx, val, d, store=store)
    loss, g, cnt = ds.smooth(G(agd, grad), w)
    ref_loss, ref_g, _ = oracle.smooth(oracle.Data(y, csr=(rowptr, idx, val), d=d), grad, w)
    assert cnt == n
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12)
    assert rel_err(g, ref_g) < 1e-12
    ds.set_option("ring_rows", 1)                     # the simple (unpipelined) row loop
    loss1, g1, _ = ds.smooth(G(agd, grad), w)
    np.testing.assert_allclose(loss1, loss, rtol=1e-14)   # same per-row arithmetic; only the order of the atomic sums differs
    assert rel_err(g1, g) < 1e-14
    ds.close()


def test_csr_appended_partitions_and_generator(agd, ctx, oracle):
    """Several SparseVector partitions appended to one GPU == one load; the on-device CSR generator ==
    its CPU twin; a whole hinge + L2 run on CSR rows == the oracle (BASELINE configs[2] in miniature)."""
    n, d, k, seed = 6000, 4096, 16, 11
    rp, ix, va = oracle.synth_csr_f32(seed, 0, n, d, k)
    gen = ctx.synthetic_csr(n, d, k, agd.HingeGradient(), seed=seed, store="f32")
    grp, gix, gva, y = gen.get_csr_rows(0, 0, n, n * k)
    assert np.array_equal(grp, rp) and np.array_equal(gix, ix) and np.array_equal(gva, va)
    assert np.all(np.diff(ix.reshape(n, k), axis=1) > 0)            # strictly increasing column ids per row
    many = agd.DeviceDataset(ctx)
    for lo, hi in [(0, 1000), (1000, 1001), (1001, 4000), (4000, 6000)]:
        many.load_csr(y[lo:hi], rp[lo:hi + 1] - rp[lo], ix[rp[lo]:rp[hi]], va[rp[lo]:rp[hi]], d, store="f32")
    w = np.random.default_rng(1).standard_normal(d) * 0.1
    a, b = gen.smooth(agd.HingeGradient(), w), many.smooth(agd.HingeGradient(), w)
    assert a[2] == b[2] == n
    np.testing.assert_allclose(a[0], b[0], rtol=1e-14)
    assert rel_err(a[1], b[1]) < 1e-13                               # RED.ADD order differs run to run
    w0 = np.zeros(d)
    wg, hist, st = agd.run_with_stats(many, agd.HingeGradient(), agd.SquaredL2Updater(), 0.0, 8, 0.1, w0)
    ref = oracle.agd_run(oracle.Data(y, csr=(rp, ix, va), d=d), "hinge", "squared_l2", w0, convergence_tol=0.0,
                         num_iterations=8, reg_param=0.1)
    np.testing.assert_allclose(hist, ref.loss_history, rtol=1e-10)
    assert rel_err(wg, ref.weights) < 1e-8
    gen.close(); many.close()


# ------------------------------------------------------------------ applyProjector (K3 prox)
@pytest.mark.parametrize("upd", UPDS)
@pytest.mark.parametrize("d", [2, 100, 1024, 70001])
def test_prox_matches_oracle(agd, ctx, oracle, upd, d):
    rng = np.random.default_rng(12 + d)
    w, g = rng.standard_normal(d), rng.standard_normal(d)
    w[:: 7] *= 1e-3
    ds = ctx.parallelize(np.zeros(1), np.zeros((1, 2)))
    for step, reg in [(0.37, 0.21), (0.0, 0.5), (1.5, 0.0)]:
        rv, wn = ds.prox(U(agd, upd), w, g, step, reg)
        ref_rv, ref_w = oracle.prox(upd, w, g, step, reg)
        assert np.array_equal(wn, ref_w)              # element-wise arithmetic is bit-faithful
        np.testing.assert_allclose(rv, ref_rv, rtol=1e-13)
    ds.close()


# ------------------------------------------------------------------ the reference's own suite, on the GPU path
def rel_close(a, b, eps):
    return abs(a - b) < eps * min(abs(a), abs(b))


def test_suite_T1_T2_T4_on_gpu(agd, ctx, oracle, fixture_gd_input):
    y, X = fixture_gd_input
    data = ctx.parallelize(y, X).cache()                                          # Suite.scala:51
    gradient, simple, l2 = agd.LogisticGradient(), agd.SimpleUpdater(), agd.SquaredL2Updater()
    # T1 Suite.scala:53-91
    w, loss_agd = agd.AcceleratedGradientDescent.run(data, gradient, simple, 1e-12, 10, 0.0, [1.0, -1.0], 1.0,
                                                     float("inf"), 0.5, 0.9, True)
    _, loss_gd = agd.GradientDescent.runMiniBatchSGD(data, gradient, simple, 1.0, 50, 0.0, 1.0, [1.0, -1.0])
    assert rel_close(loss_agd[-1], loss_gd[-1], 0.02)
    D = oracle.Data(y, X=X)
    ref = oracle.agd_run(D, "logistic", "simple", [1.0, -1.0], convergence_tol=1e-12, num_iterations=10)
    np.testing.assert_allclose(loss_agd, ref.loss_history, rtol=1e-12)
    assert rel_err(w, ref.weights) < 1e-10
    _, ref_gd = oracle.gd_run(D, "logistic", "simple", [1.0, -1.0], step_size=1.0, num_iterations=50)
    np.testing.assert_allclose(loss_gd, ref_gd, rtol=1e-12)
    # T2 Suite.scala:93-136
    w2, loss2 = agd.AcceleratedGradientDescent.run(data, gradient, l2, 1e-12, 10, 0.2, [0.3, 0.12], 1.0,
                                                   float("inf"), 0.5, 0.9, True)
    wgd, lgd = agd.GradientDescent.runMiniBatchSGD(data, gradient, l2, 1.0, 50, 0.2, 1.0, [0.3, 0.12])
    assert rel_close(loss2[-1], lgd[-1], 0.02)
    assert rel_close(w2[0], wgd[0], 0.02) and rel_close(w2[1], wgd[1], 0.02)
    ref2 = oracle.agd_run(D, "logistic", "squared_l2", [0.3, 0.12], convergence_tol=1e-12, num_iterations=10, reg_param=0.2)
    np.testing.assert_allclose(loss2, ref2.loss_history, rtol=1e-12)
    ref_wgd, ref_lgd = oracle.gd_run(D, "logistic", "squared_l2", [0.3, 0.12], step_size=1.0, num_iterations=50, reg_param=0.2)
    np.testing.assert_allclose(lgd, ref_lgd, rtol=1e-12)
    assert rel_err(wgd, ref_wgd) < 1e-11
    # T4 Suite.scala:209-239: the class API with its defaults
    opt = agd.AcceleratedGradientDescent(gradient, l2).setConvergenceTol(1e-12).setNumIterations(10).setRegParam(0.2)
    w4 = opt.optimize(data, [1.0, -1.0])
    wgd4, _ = agd.GradientDescent.runMiniBatchSGD(data, gradient, l2, 1.0, 50, 0.2, 1.0, [1.0, -1.0])
    assert rel_close(w4[0], wgd4[0], 0.02) and rel_close(w4[1], wgd4[1], 0.02)
    data.close()


@pytest.mark.parametrize("shape,store,variant", [((20000, 1024), "f32", "auto"), ((5000, 100), "f64", "auto"),
                                                 ((9000, 512), "f32", "ring"), ((3000, 30), "f64", "auto"),
                                                 ((3001, 1024), "bf16", "tc"), ((3001, 1024), "bf16", "ring"),
                                                 ((3000, 1024), "f64", "generic"), ((3000, 700), "csr-f32", "auto"),
                                                 ((3000, 700), "csr-f64", "auto")])
@pytest.mark.parametrize("fraction", [0.25, 0.9])
def test_minibatch_gd_matches_oracle(agd, ctx, oracle, shape, store, variant, fraction):
    """SURVEY.md 8(f).1: GradientDescent.runMiniBatchSGD with miniBatchFraction < 1 on every gradient kernel (row mask +
    selected-row count through the slabs: wgmma, ring, generic, CSR), against the oracle's restatement with the same
    counter-based mask.  The wgmma kernel is held to its own accuracy (fp32 margins, bf16 x 3 split)."""
    n, d = shape
    rng = np.random.default_rng(500 + n + d)
    X, y = make_data(rng, n, d, "logistic", np.float64 if store == "f64" or store == "csr-f64" else np.float32)
    w0 = rng.standard_normal(d) * 0.01
    if store.startswith("csr"):
        keep = np.abs(X) > 1.0                                      # about a third of the entries
        rowptr = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
        idx = np.nonzero(keep)[1].astype(np.int32)
        D = oracle.Data(y, csr=(rowptr, idx, X[keep]), d=d)
        data = ctx.parallelize_csr(y, rowptr, idx, X[keep], d, store=store[4:])
    else:
        if store == "bf16":
            X = R.bf16_to_f32(R.f32_to_bf16_bits(X))
        D = oracle.Data(y, X=X)
        data = ctx.parallelize(y, X, store=store)
    if variant != "auto":
        data.set_option("k1_variant", variant)
    w, hist = agd.GradientDescent.runMiniBatchSGD(data, agd.LogisticGradient(), agd.SquaredL2Updater(), 0.5, 12, 0.01,
                                                  fraction, w0)
    rw, rh = oracle.gd_run(D, "logistic", "squared_l2", w0, step_size=0.5, num_iterations=12,
                           reg_param=0.01, mini_batch_fraction=fraction)
    assert len(hist) == len(rh) == 12
    tc = variant == "tc"
    np.testing.assert_allclose(hist, rh, rtol=1e-7 if tc else 1e-11)
    assert rel_err(w, rw) < (1e-6 if tc else 1e-10)
    full = agd.GradientDescent.runMiniBatchSGD(data, agd.LogisticGradient(), agd.SquaredL2Updater(), 0.5, 12, 0.01, 1.0, w0)
    assert not np.allclose(full[1], hist)          # the mask really drops rows
    data.close()


def test_suite_T3_convergence_tol_on_gpu(agd, ctx, fixture_gd_input):             # Suite.scala:138-207
    y, X = fixture_gd_input
    data = ctx.parallelize(y, X).cache()
    gradient, l2 = agd.LogisticGradient(), agd.SquaredL2Updater()
    run = agd.AcceleratedGradientDescent.run
    w1, loss1 = run(data, gradient, l2, 0.1, 1000, 0.0, [0.0, 0.0], 1.0, float("inf"), 0.5, 0.9, True)
    w2, loss2 = run(data, gradient, l2, 0.0, len(loss1) - 1, 0.0, [0.0, 0.0], 1.0, float("inf"), 0.5, 0.9, True)
    assert len(loss2) == len(loss1) - 1
    assert np.linalg.norm(w1 - w2) / np.linalg.norm(w1) < 0.1
    _, loss3 = run(data, gradient, l2, 0.01, 100, 0.0, [0.0, 0.0], 1.0, float("inf"), 0.5, 0.9, True)
    assert len(loss3) > len(loss1)
    assert (len(loss1), len(loss2), len(loss3)) == (8, 7, 12)   # what the oracle gives (BASELINE.md section 2)
    data.close()


def test_suite_T5_wide_rows(agd, ctx, oracle):                                    # Suite.scala:244-259
    m, n = 10, 200000
    X = np.concatenate([oracle.jrandom_doubles(idx, (m // 2) * n).reshape(m // 2, n) for idx in (0, 1)], axis=0)
    y = np.ones(m)
    w0 = oracle.jrandom_doubles(0, n)
    data = ctx.parallelize(y, X)
    opt = agd.AcceleratedGradientDescent(agd.LogisticGradient(), agd.SquaredL2Updater()) \
        .setConvergenceTol(1e-12).setNumIterations(1).setRegParam(1.0)
    w = opt.optimize(data, w0)
    ref = oracle.agd_run(oracle.Data(y, X=X), "logistic", "squared_l2", w0, convergence_tol=1e-12, num_iterations=1,
                         reg_param=1.0)
    assert rel_err(w, ref.weights) < 1e-12
    data.close()



# ------------------------------------------------------------------ pass fusion (SURVEY 8(f).2): two points, one sweep
PAIR_SHAPES = [((3001, 1024), "f32", "auto"), ((2000, 512), "f32", "auto"), ((501, 1001), "f32", "auto"),
               ((777, 2048), "f32", "auto"), ((300, 4096), "f32", "auto"), ((1500, 512), "f64", "auto"),
               ((400, 2048), "f64", "auto"), ((10, 20000), "f32", "auto"), ((700, 300), "f64", "generic"),
               ((2000, 1024), "bf16", "ring"), ((900, 2048), "bf16", "ring"), ((600, 4096), "bf16", "ring"),
               ((2000, 1024), "bf16", "tc"), ((517, 4096), "bf16", "tc"), ((300, 128), "bf16", "tc")]


@pytest.mark.parametrize("grad", GRADS)
@pytest.mark.parametrize("shape,store,variant", PAIR_SHAPES)
def test_smooth_pair_equals_two_sweeps_bit_for_bit(agd, ctx, grad, shape, store, variant):
    """agd_smooth_pair (applySmooth at w + the loss at w2 from one read of X) returns exactly the bits of two agd_smooth calls."""
    n, d = shape
    rng = np.random.default_rng(77 + n + d)
    X, y = make_data(rng, n, d, grad, np.float64 if store == "f64" else np.float32)
    w = rng.standard_normal(d) * 0.7 / np.sqrt(d)
    w2 = w + rng.standard_normal(d) * 0.2 / np.sqrt(d)
    ds = ctx.parallelize(y, X, store=store)
    ds.set_option("k1_variant", variant)
    a = ds.smooth(G(agd, grad), w)
    b = ds.smooth(G(agd, grad), w2)
    loss, g, cnt, loss2 = ds.smooth_pair(G(agd, grad), w, w2)
    assert cnt == a[2] == n
    assert loss == a[0] and np.array_equal(g, a[1])
    assert loss2 == b[0]
    ds.close()


TWO_SHAPES = [((3001, 1024), "f32"), ((2000, 512), "f32"), ((501, 1001), "f32"), ((1500, 512), "f64"), ((700, 300), "f64"),
              ((16, 1024), "f32"), ((9, 640), "f32"), ((1200, 1024), "f64"), ((900, 2048), "f32"), ((333, 1500), "f32"),
              ((2000, 1024), "bf16"), ((517, 4096), "bf16"), ((300, 128), "bf16"), ((700, 768), "bf16"), ((260, 640), "bf16")]     # wgmma: r at w2 rides in B columns of its own


@pytest.mark.parametrize("grad", GRADS)
@pytest.mark.parametrize("shape,store", TWO_SHAPES)
def test_smooth_two_equals_two_sweeps_bit_for_bit(agd, ctx, grad, shape, store):
    """agd_smooth_two (two complete applySmooth evaluations from one read of X -- the speculative sweep of the memoised pass
    structure) returns exactly the bits of two agd_smooth calls, and of the loss-only pair form."""
    n, d = shape
    rng = np.random.default_rng(177 + n + d)
    X, y = make_data(rng, n, d, grad, np.float64 if store == "f64" else np.float32)
    w = rng.standard_normal(d) * 0.7 / np.sqrt(d)
    w2 = w + rng.standard_normal(d) * 0.2 / np.sqrt(d)
    ds = ctx.parallelize(y, X, store=store)
    a = ds.smooth(G(agd, grad), w)
    b = ds.smooth(G(agd, grad), w2)
    loss, g, cnt, loss2, g2 = ds.smooth_two(G(agd, grad), w, w2)
    assert cnt == a[2] == n
    assert loss == a[0] and np.array_equal(g, a[1])
    assert loss2 == b[0] and np.array_equal(g2, b[1])
    p = ds.smooth_pair(G(agd, grad), w, w2)
    assert p[0] == loss and p[3] == loss2 and np.array_equal(p[1], g)
    ds.close()


def test_smooth_two_unsupported_shards_refuse(agd, ctx):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((300, 4096)).astype(np.float32)
    y = (rng.random(300) > 0.5).astype(np.float64)
    for store, dd in (("f32", 4096), ("bf16", 1024)):        # four vectors per thread / wgmma with fp64 margins: no two-gradient form
        ds = ctx.parallelize(y, X[:, :dd].copy(), store=store)
        if store == "bf16":
            ds.set_option("tc_margins", "f64")
        with pytest.raises(agd.NativeError, match="two-(gradient|point)"):
            ds.smooth_two(agd.LogisticGradient(), np.zeros(dd), np.zeros(dd))
        # the memoised run simply does not speculate there
        w_, h_, st = agd.run_with_stats(ds, agd.LogisticGradient(), agd.SimpleUpdater(), 0.0, 4, 0.0, np.zeros(dd), memoize=True)
        assert st.iterations == 4
        ds.close()


SPEC_CASES = [(20000, 1024, "logistic", "simple", 0.0, "f32", 12, {}),
              (6000, 1001, "logistic", "l1", 0.002, "f32", 12, {}),
              (5000, 512, "hinge", "squared_l2", 0.1, "f32", 15, {}),
              (4000, 256, "least_squares", "simple", 0.0, "f64", 25, {"L0": 1e-3}),                 # L-increase: guesses rejected
              (1000, 100, "least_squares", "squared_l2", 0.1, "f64", 30, {}),                       # restarts: (f_x, g_x) reused
              (1000, 512, "least_squares", "simple", 0.0, "f64", 60, {"tol": 1e-6}),               # leaves through :322-324
              (5000, 1024, "logistic", "simple", 0.0, "bf16", 8, {}),                               # wgmma kernel, two-gradient form
              (3000, 4096, "least_squares", "squared_l2", 0.01, "bf16", 8, {})]


@pytest.mark.parametrize("case", SPEC_CASES, ids=[f"{c[0]}x{c[1]}-{c[2]}-{c[3]}-{i}" for i, c in enumerate(SPEC_CASES)])
def test_speculative_memoised_run_is_bit_identical(agd, ctx, case):
    """AGD_FLAG_MEMOIZE_FX on a shard with a two-gradient kernel: applySmooth(x) (AGD.scala:269) shares its sweep with the
    guessed applySmooth(y) of the next iteration.  Same weights, history and branch counts as every other pass structure,
    bit for bit; one sweep per accepted iteration."""
    n, d, grad, upd, reg, store, iters, kw = case
    rng = np.random.default_rng(n + d + iters + 19)
    X, y = make_data(rng, n, d, grad, np.float64 if store == "f64" else np.float32)
    data = ctx.parallelize(y, X, store=store)
    args = (data, G(agd, grad), U(agd, upd), kw.get("tol", 0.0), iters, reg, np.zeros(d), kw.get("L0", 1.0),
            kw.get("Lexact", float("inf")), kw.get("beta", 0.5), kw.get("alpha", 0.9), kw.get("may_restart", True))
    w0, h0, s0 = agd.run_with_stats(*args, fuse=False)
    wm, hm, sm = agd.run_with_stats(*args, memoize=True)
    assert np.array_equal(wm, w0) and np.array_equal(hm, h0)
    assert (sm.iterations, sm.backtracks, sm.restarts, sm.converged) == (s0.iterations, s0.backtracks, s0.restarts, s0.converged)
    # sweeps: one per backtracking round for applySmooth(x) plus one for applySmooth(y) -- unless y was guessed in the previous
    # round's sweep (fused_passes) or the iteration follows a restart (y = x: nothing to evaluate)
    rounds = sm.iterations + sm.backtracks
    assert sm.k1_launches < s0.k1_launches
    assert sm.k1_launches <= 2 * rounds - sm.fused_passes - max(0, sm.restarts - 1)
    row_bytes = d * {"f32": 4, "f64": 8, "bf16": 2}[store]
    if store == "bf16" or 1024 < row_bytes <= 8192:                # shapes with a two-gradient kernel
        assert sm.fused_passes > 0
    wn, hn, sn = agd.run_with_stats(*args, memoize=True, fuse=False)    # AGD_FLAG_NO_FUSE switches the speculation off as well
    assert np.array_equal(wn, w0) and np.array_equal(hn, h0) and sn.fused_passes == 0
    data.close()


def test_smooth_pair_csr_and_unsupported_kernels(agd, ctx, oracle):
    rng = np.random.default_rng(5)
    n, d, k = 3000, 5000, 24
    idx = np.sort(np.stack([rng.choice(d, k, replace=False) for _ in range(n)]), axis=1).astype(np.int32)
    val = rng.standard_normal((n, k)).astype(np.float32)
    rowptr = np.arange(n + 1, dtype=np.int64) * k
    y = (rng.random(n) > 0.5).astype(np.float64)
    w, w2 = rng.standard_normal(d) * 0.1, rng.standard_normal(d) * 0.1
    ds = ctx.parallelize_csr(y, rowptr, idx.ravel(), val.ravel(), d, store="f32")
    a, b = ds.smooth(agd.HingeGradient(), w), ds.smooth(agd.HingeGradient(), w2)
    loss, g, cnt, loss2 = ds.smooth_pair(agd.HingeGradient(), w, w2)
    assert cnt == n
    np.testing.assert_allclose(loss, a[0], rtol=1e-13)          # CSR sums are atomics: equal to rounding only
    np.testing.assert_allclose(loss2, b[0], rtol=1e-13)
    assert rel_err(g, a[1]) < 1e-13
    ds.close()
    # kernels without a two-point form refuse (agd_run then simply does not fuse)
    X = rng.standard_normal((300, 1024)).astype(np.float32)
    yd = (rng.random(300) > 0.5).astype(np.float64)
    ds = ctx.parallelize(yd, X, store="bf16")                   # wgmma path: only its default (fp32-margin) mapping has one
    ds.set_option("tc_margins", "f64")
    with pytest.raises(agd.NativeError, match="two-point"):
        ds.smooth_pair(agd.LogisticGradient(), np.zeros(1024), np.zeros(1024))
    ds.close()
    ds = ctx.parallelize(yd[:100], X[:100, :36].copy(), store="f32")   # 32-row tiles
    with pytest.raises(agd.NativeError, match="two-point"):
        ds.smooth_pair(agd.LogisticGradient(), np.zeros(36), np.zeros(36))
    w_, h_, st = agd.run_with_stats(ds, agd.LogisticGradient(), agd.SimpleUpdater(), 0.0, 5, 0.0, np.zeros(36))
    assert st.fused_passes == 0 and st.k1_launches == st.passes + st.wasted_passes
    ds.close()


FUSE_CASES = [(20000, 1024, "logistic", "simple", 0.0, "f32", 12, {}),
              (6000, 1001, "logistic", "l1", 0.002, "f32", 12, {}),
              (5000, 512, "hinge", "squared_l2", 0.1, "f32", 15, {}),
              (4000, 2048, "least_squares", "simple", 0.0, "f64", 25, {"L0": 1e-3}),          # L-increase branch
              (4000, 300, "logistic", "simple", 0.0, "f64", 20, {"beta": 1.0, "L0": 0.25, "Lexact": 0.25, "may_restart": False}),
              (3000, 20000, "logistic", "squared_l2", 0.01, "f32", 8, {}),                    # generic kernel
              (1000, 512, "least_squares", "simple", 0.0, "f64", 60, {"tol": 1e-6}),          # leaves through :322-324
              (6000, 1024, "least_squares", "squared_l2", 0.01, "bf16", 10,                     # wgmma kernel, branch-free config
               {"beta": 1.0, "L0": 8.0, "Lexact": 8.0, "may_restart": False}),
              (5000, 4096, "logistic", "simple", 0.0, "bf16", 8, {})]                           # wgmma kernel, defaults


@pytest.mark.parametrize("case", FUSE_CASES, ids=[f"{c[0]}x{c[1]}-{c[2]}-{c[3]}-{i}" for i, c in enumerate(FUSE_CASES)])
def test_fused_run_is_bit_identical_to_unfused(agd, ctx, case):
    """Default agd_run lets applySmooth(x) of AGD.scala:304 ride along with the next iteration's applySmooth(y) (:250):
    same evaluations, same weights and loss history bit for bit, one sweep over X fewer per iteration."""
    n, d, grad, upd, reg, store, iters, kw = case
    rng = np.random.default_rng(n + d + iters + 9)
    X, y = make_data(rng, n, d, grad, np.float64 if store == "f64" else np.float32)
    data = ctx.parallelize(y, X, store=store)
    args = (data, G(agd, grad), U(agd, upd), kw.get("tol", 0.0), iters, reg, np.zeros(d), kw.get("L0", 1.0),
            kw.get("Lexact", float("inf")), kw.get("beta", 0.5), kw.get("alpha", 0.9), kw.get("may_restart", True))
    w1, h1, s1 = agd.run_with_stats(*args, fuse=True)
    w0, h0, s0 = agd.run_with_stats(*args, fuse=False)
    assert np.array_equal(w1, w0) and np.array_equal(h1, h0)
    assert (s1.iterations, s1.passes, s1.backtracks, s1.restarts, s1.converged) == \
           (s0.iterations, s0.passes, s0.backtracks, s0.restarts, s0.converged)
    assert s0.fused_passes == 0 and s0.k1_launches == s0.passes + s0.wasted_passes
    assert s1.fused_passes == s1.iterations - 1            # every history evaluation but the last shared a sweep
    assert s1.k1_launches == s1.passes + s1.wasted_passes - s1.fused_passes
    wm, hm, sm = agd.run_with_stats(*args, memoize=True)   # memoisation leaves nothing to fuse unless x moved
    assert np.array_equal(wm, w0) and np.array_equal(hm, h0)
    data.close()

# ------------------------------------------------------------------ whole-loop parity (agd_run)
CASES = [
    # (n, d, grad, upd, reg, store, iters, kwargs)
    (1000, 100, "least_squares", "simple", 0.0, "f64", 30, {}),                    # BASELINE config 1
    (1000, 100, "least_squares", "simple", 0.0, "f64", 12, {}),                    # same, before convergence noise
    (1000, 100, "least_squares", "squared_l2", 0.1, "f64", 12, {}),
    (1000, 100, "least_squares", "squared_l2", 0.1, "f64", 30, {}),
    (1000, 100, "least_squares", "l1", 0.05, "f64", 30, {}),
    (20000, 1024, "logistic", "simple", 0.0, "f32", 10, {}),                       # config 2's shape, small n
    (20000, 1024, "logistic", "squared_l2", 0.01, "f32", 12, {}),
    (5000, 512, "hinge", "squared_l2", 0.1, "f32", 15, {}),
    (5000, 256, "logistic", "l1", 0.001, "f64", 15, {}),
    (4000, 64, "logistic", "simple", 0.0, "f64", 20, {"beta": 1.0, "L0": 0.25, "Lexact": 0.25, "may_restart": False}),
    (4000, 64, "logistic", "simple", 0.0, "f64", 20, {"may_restart": False}),
    (4000, 64, "least_squares", "simple", 0.0, "f64", 25, {"L0": 1e-3}),           # forces the L-increase branch
    (4000, 64, "least_squares", "simple", 0.0, "f64", 25, {"L0": 1e-3, "Lexact": 8.0}),
    (6000, 1001, "logistic", "l1", 0.002, "f32", 12, {}),       # odd d: rows padded with zero columns at load
    (3000, 37, "hinge", "squared_l2", 0.05, "f64", 12, {}),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}x{c[1]}-{c[2]}-{c[3]}-{i}" for i, c in enumerate(CASES)])
@pytest.mark.parametrize("memoize", [False, True])
def test_run_matches_oracle(agd, ctx, oracle, case, memoize):
    n, d, grad, upd, reg, store, iters, kw = case
    rng = np.random.default_rng(n + d + iters)
    X, y = make_data(rng, n, d, grad, np.float32 if store == "f32" else np.float64)
    w0 = np.zeros(d)
    data = ctx.parallelize(y, X, store=store)
    w, hist, st = agd.run_with_stats(data, G(agd, grad), U(agd, upd), 0.0, iters, reg, w0,
                                     kw.get("L0", 1.0), kw.get("Lexact", float("inf")), kw.get("beta", 0.5),
                                     kw.get("alpha", 0.9), kw.get("may_restart", True), memoize=memoize)
    ref = oracle.agd_run(oracle.Data(y, X=X), grad, upd, w0, convergence_tol=0.0, num_iterations=iters,
                         reg_param=reg, L0=kw.get("L0", 1.0), Lexact=kw.get("Lexact", float("inf")),
                         beta=kw.get("beta", 0.5), alpha=kw.get("alpha", 0.9),
                         may_restart=kw.get("may_restart", True), partitions=2)
    # The reference's trajectory is itself a function of Spark's partition count once f_x - q_x
    # (AGD.scala:273-274) is rounding noise: re-run the oracle with other partitionings and demand
    # identical branch decisions from the GPU only where the reference agrees with itself.
    alts = [oracle.agd_run(oracle.Data(y, X=X), grad, upd, w0, convergence_tol=0.0, num_iterations=iters,
                           reg_param=reg, L0=kw.get("L0", 1.0), Lexact=kw.get("Lexact", float("inf")),
                           beta=kw.get("beta", 0.5), alpha=kw.get("alpha", 0.9),
                           may_restart=kw.get("may_restart", True), partitions=P) for P in (1, 3, 8)]
    sig = lambda r: (r.iterations, r.passes, r.backtracks, r.restarts)
    stable = all(sig(a) == sig(ref) for a in alts)
    assert st.iterations == len(hist)
    if stable:
        assert st.iterations == ref.iterations == len(ref.loss_history)
        assert st.backtracks == ref.backtracks and st.restarts == ref.restarts
        if not memoize:
            assert st.passes == ref.passes
        else:
            assert st.passes <= ref.passes
        np.testing.assert_allclose(hist, ref.loss_history, rtol=1e-11)
        assert rel_err(w, ref.weights) < 1e-9
    else:
        spread = max(rel_err(a.weights, ref.weights) for a in alts)
        k = min(len(hist), len(ref.loss_history))
        assert k >= iters // 2          # exact stationarity (norm_dx == 0, AGD.scala:317) is itself a rounding event
        np.testing.assert_allclose(hist[:k], ref.loss_history[:k], rtol=1e-8)
        assert rel_err(w, ref.weights) < max(10 * spread, 1e-9)
    assert rel_err(w, ref.weights) < 1e-5          # north_star's stated tolerance
    data.close()


def test_empty_dataset_stops_like_the_flagged_reference(agd, ctx, oracle):
    data = ctx.parallelize(np.zeros(0), np.zeros((0, 4)))
    w, hist, st = agd.run_with_stats(data, agd.LogisticGradient(), agd.SimpleUpdater(), 1e-4, 5, 0.0,
                                     [0.1, 0.2, 0.3, 0.4])
    assert st.stopped_nan and st.nonterminating and len(hist) == 1 and np.isnan(hist[0])
    data.close()


def test_zero_iterations_returns_initial_weights(agd, ctx):
    data = ctx.parallelize(np.ones(4), np.eye(4))
    w, hist, st = agd.run_with_stats(data, agd.LogisticGradient(), agd.SimpleUpdater(), 1e-4, 0, 0.0, [1, 2, 3, 4.0])
    assert len(hist) == 0 and np.array_equal(w, [1, 2, 3, 4.0])
    data.close()


def test_padded_rows_are_invisible(agd, ctx, oracle):
    """d = 1001 fp32 rows are stored as 1004 columns (whole 16-byte vectors, zero padding) so that the TMA-ring kernel
    applies; the caller still sees d = 1001 everywhere and the ring and generic kernels agree."""
    rng = np.random.default_rng(41)
    X, y = make_data(rng, 2500, 1001, "logistic", np.float32)
    w = rng.standard_normal(1001) * 0.05
    ds = ctx.parallelize(y, X, store="f32")
    assert ds.d == 1001
    Xb, yb = ds.get_rows(0, 100, 50)
    assert Xb.shape == (50, 1001) and np.array_equal(Xb, X[100:150]) and np.array_equal(yb, y[100:150])
    a = ds.smooth(agd.LogisticGradient(), w)
    ds.set_option("k1_variant", "generic")
    b = ds.smooth(agd.LogisticGradient(), w)
    assert a[1].shape == (1001,) and a[2] == b[2] == 2500
    np.testing.assert_allclose(a[0], b[0], rtol=1e-13)
    assert rel_err(a[1], b[1]) < 1e-13
    ds.set_option("k1_variant", "ring")          # would have been rejected before: 1001 * 4 bytes is not a multiple of 16
    c = ds.smooth(agd.LogisticGradient(), w)
    assert c[0] == a[0] and np.array_equal(c[1], a[1])
    ds.close()


def test_argument_errors(agd, ctx):
    data = ctx.parallelize(np.ones(4), np.eye(4))
    with pytest.raises(ValueError):
        agd.AcceleratedGradientDescent(agd.LogisticGradient(), agd.SimpleUpdater()).optimize(data, [1.0, 2.0])
    with pytest.raises(agd.NativeError, match="dimension mismatch"):
        data.load_dense(np.ones(2), np.ones((2, 5)))
    with pytest.raises(ValueError):          # the native side reads / writes agd_dim doubles through these buffers
        agd.GradientDescent.runMiniBatchSGD(data, agd.LogisticGradient(), agd.SimpleUpdater(), 1.0, 2, 0.0, 1.0, [1.0, 2.0])
    data.close()


def test_bad_csr_partitions_are_rejected_at_load(agd, ctx):
    """The gradient kernel gathers w[idx] and scatters into g[idx]: a column id outside [0, d), or a SparseVector whose size
    differs from the weights', must fail at load -- not corrupt neighbouring device allocations (ADVICE r1)."""
    y = np.array([1.0, 0.0, 1.0])
    good = (np.array([0, 2, 3, 5]), np.array([0, 4, 2, 1, 3], dtype=np.int32), np.ones(5))
    ds = ctx.parallelize_csr(y, *good, d=5)
    l0, g0, c0 = ds.smooth(agd.HingeGradient(), np.zeros(5))
    for rowptr, idx, msg in [
        (np.array([0, 2, 3, 5]), np.array([0, 5, 2, 1, 3], dtype=np.int32), "column index"),      # idx == d
        (np.array([0, 2, 3, 5]), np.array([0, -1, 2, 1, 3], dtype=np.int32), "column index"),     # negative
        (np.array([0, 3, 2, 5]), np.array([0, 4, 2, 1, 3], dtype=np.int32), "rowptr"),            # not monotone
    ]:
        with pytest.raises(agd.NativeError, match=msg):
            ds.load_csr(y, rowptr, idx, np.ones(5), 5)
    # nothing of the rejected partitions became part of the shard
    assert ds.local_rows(0) == 3
    l1, g1, c1 = ds.smooth(agd.HingeGradient(), np.zeros(5))
    assert (l1, c1) == (l0, c0) and np.array_equal(g0, g1)
    ds.close()


# ------------------------------------------------------------------ synthetic generator vs its CPU twin
@pytest.mark.parametrize("grad", GRADS)
def test_synthetic_generator_matches_cpu_twin(agd, ctx, oracle, grad):
    n, d, seed = 5000, 1024, 42
    ds = ctx.synthetic(n, d, G(agd, grad), seed=seed, store="f32")
    Xg, yg = ds.get_rows(0, 0, n)
    Xc = oracle.synth_dense_f32(seed, 0, n, d)
    assert np.array_equal(Xg, Xc)                      # integer construction: bit-exact
    wt = oracle.synth_wtrue(seed, d)
    yc = oracle.synth_labels(seed, grad, 0, Xc, wt)
    if grad == "least_squares":
        np.testing.assert_allclose(yg, yc, rtol=1e-12, atol=1e-13)
    else:
        assert np.array_equal(yg, yc)
    assert abs(Xg.mean()) < 0.01 and abs(Xg.std() - 1.0) < 0.01
    ds.close()


# ------------------------------------------------------------------ full-size properties (BASELINE config 2)
def test_full_size_properties(agd, ctx, oracle):
    """10M x 1024 fp32 logistic is too big for the oracle; check size-independent properties and a
    sampled comparison instead."""
    n, d = 10_000_000, 1024
    ds = ctx.synthetic(n, d, agd.LogisticGradient(), seed=42, store="f32")
    assert ds.local_rows(0) == n
    w0 = np.zeros(d)
    loss0, g0, cnt = ds.smooth(agd.LogisticGradient(), w0)
    assert cnt == n
    np.testing.assert_allclose(loss0, np.log(2.0), rtol=1e-14)   # every row contributes log1p(exp(0))
    # least-squares gradient is affine in w: g(a+b) - g(0) = (g(a) - g(0)) + (g(b) - g(0))
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal(d) * 0.03, rng.standard_normal(d) * 0.03
    ls = agd.LeastSquaresGradient()
    gz, ga, gb, gab = (ds.smooth(ls, v)[1] for v in (w0, a, b, a + b))
    assert rel_err(gab - gz, (ga - gz) + (gb - gz)) < 1e-11
    # determinism
    l1, g1, _ = ds.smooth(agd.LogisticGradient(), a)
    l2, g2, _ = ds.smooth(agd.LogisticGradient(), a)
    assert l1 == l2 and np.array_equal(g1, g2)
    # a 3-iteration run: memoised and plain pass structures give bit-identical results
    w_a, h_a, st_a = agd.run_with_stats(ds, agd.LogisticGradient(), agd.SimpleUpdater(), 0.0, 3, 0.0, w0)
    w_b, h_b, st_b = agd.run_with_stats(ds, agd.LogisticGradient(), agd.SimpleUpdater(), 0.0, 3, 0.0, w0, memoize=True)
    assert np.array_equal(w_a, w_b) and np.array_equal(h_a, h_b) and st_b.passes < st_a.passes
    assert np.all(np.diff(h_a) < 0)                               # the loss decreases
    # sampled oracle comparison: first 20000 rows' statistics vs the same rows on the CPU
    Xs, ys = ds.get_rows(0, 0, 20000)
    sub = ctx.parallelize(ys, Xs, store="f32")
    ls_, gs_, _ = sub.smooth(agd.LogisticGradient(), a)
    rl, rg, _ = oracle.smooth(oracle.Data(ys, X=Xs), "logistic", a, partitions=8, threads=8)
    np.testing.assert_allclose(ls_, rl, rtol=1e-12)
    assert rel_err(gs_, rg) < 1e-12
    sub.close(); ds.close()


# ------------------------------------------------------------------ several GPUs in one process
def test_local_world_can_be_replaced_by_a_larger_one(agd):
    """agd_create makes the local GPUs a complete world; agd_comm_init on the same handle must be able to replace it with
    `first_rank .. first_rank + n_dev - 1 of a larger world` (include/agd_b200.h; ADVICE r1: it used to be rejected)."""
    import ctypes as C
    import torch
    N = agd._native
    L = N.lib()
    nd = min(torch.cuda.device_count(), 2)
    ids = (C.c_int32 * nd)(*range(nd))
    h = C.c_void_p()
    N.check(L.agd_create(ids, nd, C.byref(h)), None)
    buf = C.create_string_buffer(128)
    N.check(L.agd_comm_unique_id(buf), None)
    assert L.agd_comm_init(h, buf, nd, 0) == 0                      # replaces the default world (world == local GPUs here)
    assert L.agd_comm_init(h, buf, nd, 0) != 0                      # ... once
    assert b"already initialised" in L.agd_last_error(h)
    L.agd_destroy(h)
    h2 = C.c_void_p()
    N.check(L.agd_create(ids, nd, C.byref(h2)), None)
    assert L.agd_comm_init_ipc(h2, nd + 2, 1) == 0                  # ranks 1..nd of a world of nd + 2 processes' GPUs
    assert L.agd_comm_init_ipc(h2, nd, nd) != 0 and b"bad rank layout" in L.agd_last_error(h2)
    L.agd_destroy(h2)


@pytest.mark.parametrize("collective", ["p2p", "nccl"])
def test_two_local_gpus_match_one(agd, oracle, collective):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    rng = np.random.default_rng(21)
    X, y = make_data(rng, 30001, 1024, "logistic", np.float32)
    w0 = np.zeros(1024)
    two = agd.Context(devices=[0, 1]).parallelize(y, X, store="f32")
    two.set_option("collective", collective)
    w, hist, st = agd.run_with_stats(two, agd.LogisticGradient(), agd.SquaredL2Updater(), 0.0, 8, 0.01, w0)
    assert st.collective_kind == (1 if collective == "p2p" else 0)
    assert st.collective_calls == st.passes - st.fused_passes       # one all-reduce per sweep over X
    ref = oracle.agd_run(oracle.Data(y, X=X), "logistic", "squared_l2", w0, convergence_tol=0.0, num_iterations=8,
                         reg_param=0.01)
    np.testing.assert_allclose(hist, ref.loss_history, rtol=1e-11)
    assert rel_err(w, ref.weights) < 1e-9
    two.close()
