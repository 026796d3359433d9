"""The gradient kernels element by element against exact references (tests/k1_reference.py).

One-hot designs put a single product into every per-tile fp32 sum of the wgmma kernel, so its gradient can be predicted
almost to the bit: a dropped piece of r, a row landing on the wrong feature or a stale ring slot shows up as a wrong element.
Every form of the kernel runs on them, over widths where a tile holds many ring groups, shards of fewer than 16 rows, long
streams and the smallest ring; then tiles of extreme magnitude, the sigmoid row by row out to the underflow point, and a
zero-residual probe of the margins."""
import os
import sys
from decimal import Decimal, getcontext

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import k1_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu


def one_hot_shard(ctx, n, d, seed, tile_exp=None, **opts):
    rng = np.random.default_rng(seed)
    X, col = R.one_hot_design(n, d, rng)
    y = R.full_labels(n, rng)
    if tile_exp is not None:                      # largest |r| of tile t near 2^tile_exp[t]
        y = np.ldexp(y, np.repeat(np.asarray(tile_exp) - 20, 16)[:n])
    ds = ctx.parallelize(y, X, store="bf16")
    ds.set_option("k1_variant", "tc")
    for k, v in opts.items():
        ds.set_option(k, v)
    return ds, X[np.arange(n), col].astype(np.float64), col, y, rng


def assert_one_hot(g, x, col, r, cnt):
    e1, e2 = R.one_hot_check(g, x, col, r, cnt)
    assert e2 <= 1.0, f"gradient off the exact r by {e2:.3g} x 2^-22"
    assert e1 <= 1.0, f"gradient off sum x (hi + mid + lo) by {e1:.3g} x 2^-40"


FORMS = {"default": {}, "tc_margins=f64": {"tc_margins": "f64"}, "ring_rows=1": {"ring_rows": 1},
         "ring_rows=4": {"ring_rows": 4}, "ring_ctas=2": {"ring_ctas": 2}, "smooth_pair": {}, "smooth_two": {}}


@pytest.mark.parametrize("d", [640, 3200])
@pytest.mark.parametrize("at_zero", [True, False])
@pytest.mark.parametrize("form", list(FORMS))
def test_one_hot_every_form(agd, ctx, form, at_zero, d):
    """Least squares on one-hot designs.  At w = 0, r = -2y exactly; otherwise every margin is one product, in fp32 (x times
    w rounded to fp32) on the default mapping and its two-point forms, in fp64 on the others."""
    n = 2113
    ds, x, col, y, rng = one_hot_shard(ctx, n, d, 11 + d, **FORMS[form])
    f32 = form in ("default", "ring_ctas=2", "smooth_pair", "smooth_two")

    def r_at(w):
        wc = w[col]
        m = (x.astype(np.float32) * wc.astype(np.float32)).astype(np.float64) if f32 else x * wc
        return 2.0 * (m - y), np.sum((m - y) ** 2) / n

    w = np.zeros(d) if at_zero else rng.standard_normal(d) * 8.0
    w2 = rng.standard_normal(d) * 8.0
    if form == "smooth_two":
        loss, g, cnt, loss2, g2 = ds.smooth_two(agd.LeastSquaresGradient(), w, w2)
        r2, l2 = r_at(w2)
        assert_one_hot(g2, x, col, r2, cnt)
        assert loss2 == pytest.approx(l2, rel=1e-14)
    elif form == "smooth_pair":
        loss, g, cnt, loss2 = ds.smooth_pair(agd.LeastSquaresGradient(), w, w2)
        assert loss2 == pytest.approx(r_at(w2)[1], rel=1e-14)
    else:
        loss, g, cnt = ds.smooth(agd.LeastSquaresGradient(), w)
    r, l1 = r_at(w)
    assert cnt == n
    assert loss == pytest.approx(l1, rel=1e-14)
    assert_one_hot(g, x, col, r, cnt)
    ds.close()


@pytest.mark.parametrize("stages", [0, 1])            # 0: the default ring (16 groups or what fits); 1: the smallest, ngt + 1
@pytest.mark.parametrize("n", [1, 7, 15, 16, 17, 2111, 2112, 2113])      # 2112 = 16 rows x 132 SMs
@pytest.mark.parametrize("d", [128, 384, 640, 1152, 2176, 3200, 3968, 4096])
def test_one_hot_streams_and_rings(agd, ctx, d, n, stages):
    ds, x, col, y, _ = one_hot_shard(ctx, n, d, 100 + d + n, ring_stages=stages)
    loss, g, cnt = ds.smooth(agd.LeastSquaresGradient(), np.zeros(d))
    assert cnt == n and loss == pytest.approx(np.sum(y * y) / n, rel=1e-14)
    assert_one_hot(g, x, col, -2.0 * y, cnt)
    ds.close()


@pytest.mark.parametrize("stages", [0, 1])
def test_one_hot_long_stream(agd, ctx, stages):
    """31 tiles per CTA on 132 SMs: the ring and the B double buffer wrap many times."""
    n, d = 132 * 16 * 31 + 5, 1152
    ds, x, col, y, _ = one_hot_shard(ctx, n, d, 5, ring_stages=stages)
    loss, g, cnt = ds.smooth(agd.LeastSquaresGradient(), np.zeros(d))
    assert cnt == n
    assert_one_hot(g, x, col, -2.0 * y, cnt)
    ds.close()


@pytest.mark.parametrize("exps", [[-140], [-110], [100], [126], "mixed"], ids=["2^-140", "2^-110", "2^100", "2^126", "mixed"])
def test_tile_magnitude_edges(agd, ctx, exps):
    """Tiles whose largest |r| is far outside fp32's comfortable range: r is scaled by a power of two per tile before the
    split, so the gradient keeps the accuracy of in-range tiles (|x| <= 2^4 here; the contract is |x| <= 2^100)."""
    n, d = 2113, 640
    T = -(-n // 16)
    if exps == "mixed":
        exps = np.random.default_rng(1).choice([-140, -110, -20, 0, 60, 100, 126], T)
    else:
        exps = np.full(T, exps[0])
    ds, x, col, y, _ = one_hot_shard(ctx, n, d, 31, tile_exp=exps)
    loss, g, cnt = ds.smooth(agd.LeastSquaresGradient(), np.zeros(d))
    assert np.all(np.isfinite(g))
    assert_one_hot(g, x, col, -2.0 * y, cnt)
    ds.close()


def test_logistic_tiles_below_fp32_range(agd, ctx):
    """Logistic rows with y = 0 and margins near -97: r = sigmoid(m) ~ 2^-140, below every normal fp32 and bf16."""
    n = d = 2048
    rng = np.random.default_rng(4)
    w = (-97.0 + rng.random(d) * 4.0).astype(np.float32).astype(np.float64)
    X = np.eye(n, dtype=np.float32)
    ds = ctx.parallelize(np.zeros(n), X, store="bf16")
    ds.set_option("k1_variant", "tc")
    loss, g, cnt = ds.smooth(agd.LogisticGradient(), w)
    r = 1.0 / (1.0 + np.exp(-w))
    e1, e2 = R.one_hot_check(g, np.ones(n), np.arange(n), r, cnt)
    assert e2 <= 1.0
    ds.close()


# ------------------------------------------------------------------ the sigmoid, row by row
SPECIAL = [700.0, 708.4, 709.8, 745.1]


def _sigmoid_dec(m):
    getcontext().prec = 50
    return 1 / (1 + (-Decimal(float(m))).exp())


def _sigmoid_m1_dec(m):    # sigmoid(m) - 1 = -1 / (1 + e^m), without 1 - (1 - tiny) cancelling at 50 digits
    getcontext().prec = 50
    return -1 / (1 + Decimal(float(m)).exp())


def _softplus_dec(m):      # log(1 + e^m) = max(m, 0) + log1p(e^-|m|); log1p by its series where 1 + t would round to 1
    getcontext().prec = 50
    m = Decimal(float(m))
    t = (-abs(m)).exp()
    l1p = t - t * t / 2 + t * t * t / 3 if t < Decimal("1e-15") else (1 + t).ln()
    return max(m, Decimal(0)) + l1p


TAIL = [700.0, 708.4, 709.8, 720.0, 737.0, 745.1, 746.0, 750.0]


@pytest.mark.parametrize("store,d,variant", [("f64", 1024, "ring"), ("f64", 4096, "auto"), ("bf16", 4096, "tc")])
def test_logistic_per_row(agd, ctx, oracle, store, d, variant):
    """One-hot rows with x = n and w = m / n (both exact): each gradient entry is then one row's multiplier itself, with
    no division into the subnormals.  Margins are exact fp32 values over [-750, 750] through +-700, +-708.4, +-709.8 and
    +-745.1; half the rows have y = 0, half y = 1."""
    n = d
    half = n // 2
    # sorted, so a 16-row tile holds neighbouring margins: on the wgmma kernel a row whose |r| is below 2^-133 of its
    # tile's largest is lost to bf16's range (DESIGN.md section 4)
    grid = np.sort(np.concatenate([np.linspace(-750, 750, half - 8), SPECIAL, [-s for s in SPECIAL]]))
    m = np.float32(grid).astype(np.float64)
    w = np.concatenate([m, m]) / n
    y = np.concatenate([np.zeros(half), np.ones(half)])
    ds = ctx.parallelize(y, n * np.eye(n, dtype=np.float32), store=store)
    if variant != "auto":
        ds.set_option("k1_variant", variant)
    loss, g, cnt = ds.smooth(agd.LogisticGradient(), w)
    assert cnt == n
    sig = np.array([float(_sigmoid_dec(v)) for v in m])
    sigm1 = np.array([float(_sigmoid_m1_dec(v)) for v in m])
    # fp64 kernels: 4 ulp (4 x 2^-1074 among the subnormals) for y = 0, 2^-52 absolute for y = 1; the wgmma kernel carries
    # r to 24 bits (bf16 x 3), so there 2^-22 relative, with the same floors
    rel = 2.0 ** -22 if variant == "tc" else 0.0
    err0, tol0 = np.abs(g[:half] - sig), np.maximum(4 * np.spacing(np.abs(sig)), rel * np.abs(sig))
    assert np.all(err0 <= tol0), m[np.argmax(err0 / tol0)]
    err1, tol1 = np.abs(g[half:] - sigm1), np.maximum(2.0 ** -52, rel * np.abs(sigm1))
    assert np.all(err1 <= tol1), m[np.argmax(err1 / tol1)]
    # loss over two margin bands: rows outside the band sit at margins whose loss and multiplier are 0 in double
    for lo, hi in [(0, 30), (30, 700)]:
        band = (np.abs(m) >= lo) & (np.abs(m) < hi)
        band = np.concatenate([band, band])
        wb = np.where(band, w, np.where(y > 0, 800.0, -800.0) / n)
        lb, _, _ = ds.smooth(agd.LogisticGradient(), wb)
        ref = sum((_softplus_dec(-v) if yy > 0 else _softplus_dec(v)) for v, yy in zip(w[band] * n, y[band])) / n
        assert lb == pytest.approx(float(ref), rel=4e-15), (lo, hi)
    ds.close()
    # |m| >= 700, one row per shard (the loss is not divided by a count): y = 1 against the exact log(1 + e^-m), 4 ulp down
    # into the subnormals.  y = 0 with m < 0 is MLlib's log1pExp(-m) + m, which cancels to 0 instead of e^m: the host
    # restatement of Gradient.scala gives the same, and the device must match it
    dd = 128
    for v in np.float32(TAIL + [-t for t in TAIL]).astype(np.float64):
        for yy in (0.0, 1.0):
            X1 = np.zeros((1, dd), np.float32)
            X1[0, 0] = 1.0
            w1 = np.zeros(dd)
            w1[0] = v
            one = ctx.parallelize(np.array([yy]), X1, store=store)
            if variant != "auto":
                one.set_option("k1_variant", variant)
            l1, _, _ = one.smooth(agd.LogisticGradient(), w1)
            one.close()
            if yy > 0 or v > 0:
                ref = float(_softplus_dec(-v) if yy > 0 else _softplus_dec(v))
            else:
                ref = oracle.smooth(oracle.Data(np.array([yy]), X=X1.astype(np.float64)), "logistic", w1)[0]
            assert abs(l1 - ref) <= 4 * np.spacing(abs(ref)), (v, yy, l1, ref)


# ------------------------------------------------------------------ zero-residual least-squares probe of the margins
@pytest.mark.parametrize("store,variant", [("f64", "ring"), ("f64", "generic"), ("f32", "ring"), ("f32", "generic"),
                                           ("bf16", "ring"), ("bf16", "generic"), ("bf16", "tc-f64"), ("bf16", "tc")])
def test_zero_residual_probe(agd, ctx, store, variant):
    """y = the correctly rounded exact margin, so the loss is the mean squared margin error.  fp64 margins: below the fp64
    bound.  The default wgmma mapping (fp32 margins): within 1% of the phase-1 emulator, both ways -- the documented
    arithmetic is pinned, and accumulating whole rows in fp32 would give about 10 times the loss at this width."""
    n, d = 1000, (2048 if (store, variant) == ("f64", "ring") else 3200)     # the fp64 ring holds rows of up to 16 KB
    rng = np.random.default_rng(8)
    X = R.bf16_to_f32(R.f32_to_bf16_bits(rng.standard_normal((n, d)).astype(np.float32)))
    w = rng.standard_normal(d) / np.sqrt(d)
    y = R.exact_margins(X, w)
    ds = ctx.parallelize(y, X, store=store)
    ds.set_option("k1_variant", {"tc-f64": "tc"}.get(variant, variant))
    if variant == "tc-f64":
        ds.set_option("tc_margins", "f64")
    loss, _, cnt = ds.smooth(agd.LeastSquaresGradient(), w)
    assert cnt == n
    if variant == "tc":
        mse = np.mean((R.tc_margins_f32(X, w) - y) ** 2)
        assert abs(loss / mse - 1.0) < 0.01, (loss, mse)
    else:
        S = np.abs(X.astype(np.float64)) @ np.abs(w)
        bound = np.mean(((d + 4) * 2.0 ** -53 * S + 2.0 ** -53 * np.abs(y)) ** 2)
        assert loss <= bound, (loss, bound)
    ds.close()
