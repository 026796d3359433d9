"""KMeans without a GPU: argument errors, LocalKMeans.kMeansPlusPlus against an independent restatement, the Lloyd loop's
convergence and empty-cluster rules driven by an exact host step, and the new C-ABI symbols in the header and the binding."""
import numpy as np
import pytest

from test_abi import declared_symbols


def test_argument_errors(agd):
    K = agd.KMeans
    with pytest.raises(ValueError, match="k must be"):
        K(k=0)
    with pytest.raises(ValueError, match="initialization mode"):
        K(initializationMode="kmeans++")
    with pytest.raises(ValueError, match="maxIterations"):
        K(maxIterations=-1)
    with pytest.raises(ValueError, match="runs"):
        K(runs=0)
    with pytest.raises(ValueError, match="initializationSteps"):
        K().setInitializationSteps(0)
    with pytest.raises(ValueError, match="centres, k is"):
        K(k=3).setInitialModel(agd.KMeansModel(np.zeros((2, 4))))
    with pytest.raises(ValueError, match="finite"):
        K(k=2).setInitialModel(agd.KMeansModel(np.array([[0.0, np.nan], [1.0, 1.0]])))
    with pytest.raises(ValueError, match="non-empty"):
        agd.KMeansModel(np.zeros((0, 3)))


def test_setters_and_getters(agd):
    km = agd.KMeans().setK(5).setMaxIterations(7).setRuns(2).setInitializationMode("random").setInitializationSteps(3)
    km.setEpsilon(0.5).setSeed(11)
    assert (km.getK(), km.getMaxIterations(), km.getRuns(), km.getInitializationMode(), km.getInitializationSteps(),
            km.getEpsilon(), km.getSeed()) == (5, 7, 2, "random", 3, 0.5, 11)
    d = agd.KMeans()
    assert (d.getK(), d.getMaxIterations(), d.getRuns(), d.getInitializationMode(), d.getInitializationSteps(),
            d.getEpsilon(), d.getSeed()) == (2, 20, 1, "k-means||", 5, 1e-4, None)


def _kpp_restated(seed, pts, w, k, iters):
    """LocalKMeans.kMeansPlusPlus written out element by element, independently of the library's vectorised form."""
    rng = np.random.default_rng(seed)
    n = len(pts)

    def dist(a, b):
        return sum((float(x) - float(y)) ** 2 for x, y in zip(a, b))

    def closest(cs, p):
        best, bi = float("inf"), 0
        for j, c in enumerate(cs):
            v = dist(p, c)
            if v < best:
                best, bi = v, j
        return bi, best

    r = rng.random() * sum(w)
    i, cur = 0, 0.0
    while i < n and cur < r:
        cur += w[i]
        i += 1
    centers = [list(pts[max(i - 1, 0)])]
    for _ in range(1, k):
        costs = [w[j] * closest(centers, pts[j])[1] for j in range(n)]
        r = rng.random() * sum(costs)
        cum, j = 0.0, 0
        while j < n and cum < r:
            cum += costs[j]
            j += 1
        centers.append(list(pts[0] if j == 0 else pts[j - 1]))
    old = [-1] * n
    it, moved = 0, True
    while moved and it < iters:
        moved = False
        sums = [[0.0] * len(pts[0]) for _ in range(k)]
        cnt = [0.0] * k
        for i in range(n):
            c = closest(centers, pts[i])[0]
            for l in range(len(pts[0])):
                sums[c][l] += w[i] * pts[i][l]
            cnt[c] += w[i]
            if c != old[i]:
                moved = True
                old[i] = c
        for j in range(k):
            if cnt[j] == 0.0:
                centers[j] = list(pts[rng.integers(n)])
            else:
                centers[j] = [s * (1.0 / cnt[j]) for s in sums[j]]
        it += 1
    return np.array(centers)


@pytest.mark.parametrize("k", [1, 3, 6])
def test_local_kmeans_pp(agd, k):
    rng = np.random.default_rng(3)
    pts = np.concatenate([rng.normal(m, 0.3, (8, 3)) for m in (-4.0, 0.0, 5.0)])
    w = rng.integers(1, 9, pts.shape[0]).astype(np.float64)
    w[[2, 9]] = 0.0
    got = agd.LocalKMeans.kMeansPlusPlus(17, pts, w, k, 30)
    np.testing.assert_allclose(got, _kpp_restated(17, pts.tolist(), w.tolist(), k, 30), rtol=1e-13, atol=1e-13)


def test_local_kmeans_pp_more_centres_than_points(agd):
    pts = np.array([[0.0, 0.0], [1.0, 1.0]])
    got = agd.LocalKMeans.kMeansPlusPlus(5, pts, np.array([1.0, 1.0]), 4, 30)
    np.testing.assert_array_equal(got, _kpp_restated(5, pts.tolist(), [1.0, 1.0], 4, 30))


class ExactStep:
    """step(centers) on host rows, exact: every row to its closest centre (lowest index), the sums, counts and cost."""

    def __init__(self, X):
        self.X, self.calls = np.asarray(X, dtype=np.float64), []

    def __call__(self, centers):
        from spark_agd_b200.clustering import closest
        self.calls.append(np.array(centers))
        idx = closest(self.X, centers)
        k = centers.shape[0]
        sums = np.zeros((k, self.X.shape[1]))
        np.add.at(sums, idx, self.X)
        counts = np.bincount(idx, minlength=k).astype(np.float64)
        return sums, counts, float(((self.X - centers[idx]) ** 2).sum())


def test_lloyd_converges_and_keeps_empty_centres(agd):
    from spark_agd_b200.clustering import lloyd
    X = np.array([[0.0], [1.0], [10.0], [11.0]])
    step = ExactStep(X)
    start = np.array([[0.0], [10.0], [100.0]])                 # the third centre wins no row: it keeps its value
    c, cost, it = lloyd(step, start, 20, 1e-4)
    np.testing.assert_array_equal(c, [[0.5], [10.5], [100.0]])
    assert it == 2                                              # the second step moves nothing: converged
    assert cost == 4 * 0.25                                     # the cost of the centres the last step started from
    np.testing.assert_array_equal(step.calls[1], c)


def test_lloyd_epsilon_and_iteration_cap(agd):
    from spark_agd_b200.clustering import lloyd
    X = np.array([[0.0], [2.0], [3.0]])
    # a move of exactly epsilon is not a move (MLlib: changed iff distance^2 > epsilon^2)
    c, _, it = lloyd(ExactStep(X), np.array([[0.0], [3.0]]), 20, 0.5)
    assert it == 1 and c[1, 0] == 2.5
    c, cost, it = lloyd(ExactStep(X), np.array([[0.0], [3.0]]), 0, 1e-4)
    assert it == 0 and cost == 1.0 and c[1, 0] == 3.0           # no step: the cost of the start
    _, _, it = lloyd(ExactStep(X), np.array([[0.0], [3.0]]), 1, 0.0)
    assert it == 1


def test_host_predict_and_cost(agd):
    m = agd.KMeansModel(np.array([[0.0, 0.0], [2.0, 0.0], [2.0, 0.0]]))
    assert m.k == 3
    assert m.predict([1.0, 0.0]) == 0                           # a tie goes to the lowest index
    assert m.predict([1.5, 0.0]) == 1                           # a duplicated centre: the lower copy
    np.testing.assert_array_equal(m.predict([[np.nan, 0.0], [3.0, 1.0]]), [0, 1])   # no centre wins a NaN row: 0
    assert m.computeCost(np.array([[1.0, 1.0], [3.0, 0.0]])) == 2.0 + 1.0


def test_header_and_binding_declare_kmeans(agd):
    names = declared_symbols()
    for n in ("agd_kmeans_step", "agd_kmeans_assign", "agd_kmeans_costs", "agd_kmeans_sample"):
        assert n in names and n in agd.exported_symbols()
