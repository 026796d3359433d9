"""Feature transforms on the host: the scale factors of StandardScaler, the transformed colStats algebra, the mapping of a
transformed model back to the stored features, the composition rules of transformed views, and a numpy restatement of the
decomposition the gradient kernels rely on (no materialised x')."""
import numpy as np
import pytest


def fake_dataset(agd, monkeypatch, d=3):
    """A DeviceDataset without a device: enough for the view bookkeeping, which never touches the handle."""
    monkeypatch.setattr(agd.DeviceDataset, "_phys_d", property(lambda self: d))
    ds = object.__new__(agd.DeviceDataset)
    ds.ctx, ds.h, ds.total_rows, ds._xchg_d = None, None, 0, 0
    ds._base, ds._preds, ds._scale, ds._bias = None, (), None, False
    return ds


# ---------------------------------------------------------------- scale factors
def test_scaler_factor_zero_sigma_and_fit(agd):
    X = np.array([[1.0, 5.0, 0.0], [3.0, 5.0, 2.0], [8.0, 5.0, 4.0]])
    m = agd.StandardScaler().fit(X)
    np.testing.assert_array_equal(m.std, np.sqrt(X.var(axis=0, ddof=1)))
    f = m.factor
    assert f[1] == 0.0                                   # a constant column is dropped, as MLlib does
    np.testing.assert_array_equal(f[[0, 2]], 1.0 / m.std[[0, 2]])
    np.testing.assert_array_equal(m.transform(X), X * f)
    np.testing.assert_array_equal(m.transform(X[0]), X[0] * f)


def test_scaler_fewer_than_two_rows(agd):
    m = agd.StandardScaler().fit(np.array([[1.0, -2.0]]))
    np.testing.assert_array_equal(m.std, [0.0, 0.0])
    np.testing.assert_array_equal(m.factor, [0.0, 0.0])


def test_scaler_options(agd):
    with pytest.raises(NotImplementedError):
        agd.StandardScaler(withMean=True)
    with pytest.raises(NotImplementedError):
        agd.StandardScalerModel([1.0], withMean=True)
    m = agd.StandardScalerModel([2.0, 0.0, 4.0], withStd=False)
    np.testing.assert_array_equal(m.factor, [1.0, 1.0, 1.0])
    pinned = agd.StandardScalerModel([2.0, 0.0, 4.0])
    np.testing.assert_array_equal(pinned.factor, [0.5, 0.0, 0.25])
    with pytest.raises(ValueError):
        pinned.transform(np.ones((2, 4)))


# ---------------------------------------------------------------- colStats of a transformed view
def summary_of(agd, X):
    n = X.shape[0]
    mu = X.sum(axis=0) / n
    sums = np.stack([X.sum(axis=0), (X * X).sum(axis=0), np.abs(X).sum(axis=0), (X != 0).sum(axis=0).astype(float),
                     (X - mu).sum(axis=0), ((X - mu) ** 2).sum(axis=0), X.max(axis=0), X.min(axis=0)])
    return agd.MultivariateStatisticalSummary.from_sums(n, sums)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("scaled", [False, True])
def test_transformed_summary_matches_materialised(agd, scaled, bias):
    rng = np.random.default_rng(3)
    X = rng.standard_normal((50, 4)) * [1.0, 3.0, 0.5, 2.0] + [0.0, 10.0, -1.0, 0.0]
    X[::3, 3] = 0.0
    s = np.array([0.5, 0.0, -2.0, 1.5]) if scaled else None
    Xt = X * s if scaled else X
    if bias:
        Xt = np.concatenate([Xt, np.ones((50, 1))], axis=1)
    got = summary_of(agd, X).transformed(s, bias)
    ref = summary_of(agd, Xt)
    assert got.count == ref.count == 50
    for name in ("mean", "variance", "max", "min", "normL1", "normL2", "numNonzeros"):
        np.testing.assert_allclose(getattr(got, name), getattr(ref, name), rtol=1e-13, atol=1e-13, err_msg=name)
    if scaled:
        assert got.numNonzeros[1] == 0.0                # s = 0: the column is all zeros
    if bias:
        assert got.mean[-1] == 1.0 and got.variance[-1] == 0.0 and got.max[-1] == got.min[-1] == 1.0
        assert got.normL1[-1] == 50.0 and got.normL2[-1] == np.sqrt(50.0)


# ---------------------------------------------------------------- weights of a transformed model on the stored features
def test_physical_model_mapping(agd):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((20, 3))
    s = np.array([2.0, 0.0, 0.25])
    w = rng.standard_normal(4)
    v, b = agd.physical_model(w, 0.5, s, True)
    np.testing.assert_array_equal(v, s * w[:3])
    assert b == 0.5 + w[3]
    Xt = np.concatenate([X * s, np.ones((20, 1))], axis=1)
    np.testing.assert_allclose(X @ v + b, Xt @ w + 0.5, rtol=1e-14, atol=1e-14)
    v2, b2 = agd.physical_model(w[:3], 0.0, None, False)
    np.testing.assert_array_equal(v2, w[:3])
    assert b2 == 0.0
    v3, b3 = agd.physical_model(w, 1.0, None, True)
    np.testing.assert_array_equal(v3, w[:3])
    assert b3 == 1.0 + w[3]


# ---------------------------------------------------------------- composition rules
def test_composition_rules(agd, monkeypatch):
    ds = fake_dataset(agd, monkeypatch)
    scaler = agd.StandardScalerModel([1.0, 2.0, 0.0])
    scaled = scaler.transform(ds)
    assert scaled.is_view and scaled._base is ds and scaled.h is ds.h
    np.testing.assert_array_equal(scaled._scale, [1.0, 0.5, 0.0])
    both = agd.MLUtils.appendBias(scaled)                # MLlib's order: scale, then appendBias
    assert both._bias and both.d == 4 and both._phys_d == 3
    np.testing.assert_array_equal(both._scale, scaled._scale)
    with pytest.raises(ValueError):
        agd.MLUtils.appendBias(both)                     # a second bias column
    with pytest.raises(ValueError):
        scaler.transform(agd.MLUtils.appendBias(ds))     # scaling after appendBias
    with pytest.raises(ValueError):
        scaler.transform(scaled)                         # one scaling per view
    with pytest.raises(ValueError):
        agd.StandardScalerModel([1.0, 2.0]).transform(ds)   # wrong width
    # row views keep the transform, in either order
    for train, test in (both.randomSplit([0.8, 0.2]),):
        assert train._bias and test._bias and train._preds != test._preds
        np.testing.assert_array_equal(train._scale, both._scale)
    split_first = agd.MLUtils.appendBias(scaler.transform(ds.randomSplit([0.5, 0.5])[0]))
    assert split_first._preds == ds.randomSplit([0.5, 0.5])[0]._preds and split_first._bias
    both.close()                                         # a view frees nothing
    assert ds.h is None and both._base is ds


def test_append_bias_host(agd):
    X = np.arange(6.0).reshape(2, 3)
    np.testing.assert_array_equal(agd.MLUtils.appendBias(X), [[0, 1, 2, 1], [3, 4, 5, 1]])
    np.testing.assert_array_equal(agd.MLUtils.appendBias(np.array([7.0, 8.0])), [7.0, 8.0, 1.0])


# ---------------------------------------------------------------- the decomposition the kernels compute
@pytest.mark.parametrize("kind", ["logistic", "least_squares", "hinge"])
def test_gradient_decomposition_restatement(kind):
    """x'.w' = x.(s o v) + b and grad' = (s o X^T r, sum r) equal the materialised x' = appendBias(s o x) within rounding."""
    rng = np.random.default_rng(11)
    n, d = 300, 7
    X = rng.standard_normal((n, d)) * 3.0
    y = (rng.random(n) < 0.5).astype(float)
    s = np.abs(rng.standard_normal(d)) + 0.1
    s[2] = 0.0
    w = rng.standard_normal(d + 1)
    v, b = w[:d], w[d]

    def mult(m):
        if kind == "logistic":
            return 1.0 / (1.0 + np.exp(-m)) - y
        if kind == "least_squares":
            return 2.0 * (m - y)
        sg = 2 * y - 1.0
        return np.where(1.0 > sg * m, -sg, 0.0)

    Xp = np.concatenate([X * s, np.ones((n, 1))], axis=1)
    m_ref = Xp @ w
    m = X @ (s * v) + b
    np.testing.assert_allclose(m, m_ref, rtol=1e-13, atol=1e-13)
    r = mult(m_ref)
    g_ref = Xp.T @ r
    g = np.concatenate([s * (X.T @ r), [r.sum()]])
    np.testing.assert_allclose(g, g_ref, rtol=1e-12, atol=1e-12 * np.max(np.abs(g_ref)))
    assert g[2] == 0.0
