"""Scoring, colStats, the Gramian and ranking on shards long enough to reach the code that only runs on real shards, against
exact references.  On a few hundred rows every persistent-grid launch finishes in its first pass and the Gramian's ring never
wraps; here each launch loops at least three times, each ring wraps, the radix sort's scans take several rounds, and one shard
holds more than 2^31 elements.

Exact designs.  Every stored feature is a small integer (|x| <= 7, about 15 % zeros), exact in bf16, fp32 and fp64; weights are
integers with |w| <= 2, the intercept is -13/16 and labels are integers.  Every product and partial sum the kernels form is
then a multiple of 2^-8 far below 2^53, so no result depends on summation order and an fp64 BLAS reference is itself exact.
Margins, the least-squares and hinge AGD_EVAL_* sums, colStats' sums, counts, maxima and minima and the uncentered Gramian are
compared bit for bit; logistic losses are held to the bounds of test_score_gpu.

A dense shard is built from one base block [P; -P] + c (P random, c an integer per column) of 2H rows: rotated copies of it,
then a tail of T rows of P and their T mirrors.  Base row r appears cnt_r times, so every sum over the shard is cnt^T f(base),
and each column sums to exactly n c: mu = fl(sum / n) = c.  That makes colStats' pass-2 sums (dev = 0, dev2) and the centered
Gramian exact too.  On a view cnt comes from row_mask and mu is no longer an integer: the pass-2 sums are then held to
(n + n_base + 2) u times the sum of their terms' magnitudes (the device's n roundings plus the BLAS reference's n_base).

Geometry.  The row counts are derived below from the launch rules, with upper bounds on every grid (2048 / threads CTAs per SM,
and each launcher's own cap), so the regimes are reached whatever the occupancy; test_geometry_reaches_every_regime checks
that without a GPU.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import binmetrics_reference as R  # noqa: E402
from k1_reference import row_terms  # noqa: E402
from test_binmetrics_gpu import check as check_curve  # noqa: E402
from test_colstats_gpu import _Sub, check_summary, csr_cols  # noqa: E402
from test_score_gpu import _grad, _stored_csr, bits, eval_reference  # noqa: E402

U = 2.0 ** -53
B = -0.8125                      # the intercept: dyadic, so margins stay multiples of 2^-4
H100_SMS = 132                   # the SM count the CPU-only geometry test assumes

# ---------------------------------------------------------------- the launch rules, restated
# kernel                   source                          rows per CTA and step / ring / scans; grid upper bound
# score_dense_kernel       score.cu:174, 302-317, 380      8 warps x (32 / G) x 4 rows, G = pow2 >= d / EPV, <= 32;
#                                                          grid <= score_max_blocks = 8 SMs (= 2048 / 256 per SM)
# score_csr_kernel         score.cu:266, 329-337           8 warps x 4 rows; grid <= 8 SMs
# colstats_dense_kernel    colstats.cu:147, 340-363, 373   a chunk of rows per CTA, RL x 8 rows per step, RL = 256 / TU,
#                                                          TU = pow2 >= d / EPV, <= 256; gx <= min(8 SMs / y-tiles,
#                                                          colstats_max_blocks = 2 SMs), chunk = ceil(rows / gx)
# colstats_csr_kernel      colstats.cu:251, 396-410        8 warps x 4 rows; grid <= 8 SMs
# gramian_dense_kernel     gramian.cu:183-207, 319-346     splits = gramian_splits; chunk = ceil(rows / splits) rounded up
#                                                          to 16; a ring of 3 stages of 16 rows
# gramian_csr_kernel       gramian.cu:248, 348-361         one warp per row, 8 rows per CTA; grid <= 8 SMs
# rank.cu                  rank.cu:65-77, 96-115, 207-220, tiles of 2048 pairs; offsets and run scans take 256 tiles per
#                          329-342, 356-360                round; bin_hist8 grid <= 1024 CTAs of 256; the area reduce gives
#                                                          a thread ceil(blocks / 256) of ceil((K + 1) / 2048) blocks
PER_SM_MAX = 2048 // 256         # every kernel above runs 256 threads
EPV_SCORE = {"f32": 4, "f64": 2, "bf16": 8}
EPV_COLSTATS = {"f32": 4, "f64": 2, "bf16": 4}
ELEM = {"f32": 4, "f64": 8, "bf16": 2}
K_TILE, SCAN_TILES, HIST_GRID = 2048, 256, 1024


def _pow2(n, cap):
    g = 1
    while g < n and g < cap:
        g <<= 1
    return g


def _widths(store, d, epv):
    """Element units per row of each form a shard of user width d may take: rows padded to whole 16-byte vectors (the
    vector form) or left as they are (the scalar form, one element per unit)."""
    return [-(-d // epv), d]


def score_steps(rows, store, d, sms, csr=False):
    """Fewest grid-stride steps any warp of a scoring launch takes, over both forms (score.cu)."""
    out = []
    for nunit in ([1] if csr else _widths(store, d, EPV_SCORE[store])):
        per_cta = 8 * (4 if csr else (32 // _pow2(nunit, 32)) * 4)
        grid = max(1, min(PER_SM_MAX * sms, 8 * sms, -(-rows // per_cta)))
        out.append(rows // (grid * per_cta))
    return min(out)


def colstats_max_blocks(sms, d):
    return max(1, min(2 * sms, (32 << 20) // (6 * d + 1)))


def colstats_steps(rows, store, d, sms, csr=False):
    """Fewest row-loop steps of a full chunk in a colStats launch, over both forms (colstats.cu)."""
    if csr:
        return score_steps(rows, store, d, sms, csr=True)
    out = []
    for nunit in _widths(store, d, EPV_COLSTATS[store]):
        tu = _pow2(nunit, 256)
        step = (256 // tu) * 8
        ytiles = -(-nunit // tu)
        gx = max(1, PER_SM_MAX * sms // ytiles)
        gx = max(1, min(gx, colstats_max_blocks(sms, d), -(-rows // step)))
        chunk = -(-rows // gx)
        out.append(chunk // step)
    return min(out)


def gramian_splits(sms, d, rows):
    """gramian.cu:319-336."""
    nb = -(-d // 128)
    pairs = nb * (nb + 1) // 2
    packed = (d + 1) * (d + 2) // 2
    smax = max(1, min((1 << 27) // packed, rows // 128, 64))
    best, best_cost = 1, 1e300
    for s in range(1, smax + 1):
        cost = (-(-(pairs * s) // sms)) / s
        if cost < best_cost * (1.0 - 1e-12):
            best, best_cost = s, cost
    return best


def gramian_geometry(rows, d, sms):
    """(splits, fewest 16-row chunks of a split that has rows, splits that get no rows) of a dense Gramian launch."""
    s = gramian_splits(sms, d, rows)
    chunk = max(16, -(-(-(-rows // s)) // 16) * 16)
    per = [min(chunk, rows - k * chunk) for k in range(s)]
    live = [-(-r // 16) for r in per if r > 0]
    return s, min(live), sum(1 for r in per if r <= 0)


def gramian_csr_steps(rows, sms):
    grid = max(1, min(PER_SM_MAX * sms, -(-rows // 8)))
    return rows // (grid * 8)


def rank_geometry(n, k):
    """(tiles, rounds of the tile scans, rounds of bin_hist8, area blocks per thread of bin_area_final)."""
    tiles = -(-n // K_TILE)
    hist_grid = min(HIST_GRID, -(-n // 256))
    area_blocks = -(-(k + 1) // K_TILE)
    return tiles, -(-tiles // SCAN_TILES), -(-n // (hist_grid * 256)), -(-area_blocks // 256)


# ---------------------------------------------------------------- the cases
# dense shards for scoring, colStats, ranking and views: both sides of the scoring kernel's shared-memory limit for w (d = 6056)
# and the widest rows.  f64 at d = 20000 would need 16 GB for three grid steps; its global-w form is covered at d = 6144 by f32
# and at 20000 by f32 and bf16.
LONG_DENSE = [("f32", 3), ("f32", 100), ("f32", 1024), ("f32", 4096), ("f32", 6144), ("f32", 20000),
              ("f64", 3), ("f64", 100), ("f64", 1024), ("f64", 4096), ("f64", 6056),
              ("bf16", 3), ("bf16", 100), ("bf16", 1024), ("bf16", 4096), ("bf16", 20000)]
GRAMIAN_LONG_MAX_D = 4096        # the long shards' Gramian is checked up to here (the host reference grows as d^2)
MIN_STEPS = 3
TAIL = 997                       # rows of P (and as many mirrors) after the rotated blocks: the shard ends off every tile


def _half(d):
    return 4096 if d <= 1024 else (2048 if d <= 6144 else 1024)


def long_rows(store, d, sms):
    """The fewest rows that give every scoring and colStats launch MIN_STEPS steps: rotated blocks of 2H rows plus the tail."""
    need = 0
    while score_steps(need, store, d, sms) < MIN_STEPS or colstats_steps(need, store, d, sms) < MIN_STEPS:
        need = max(2 * need, 4096)
    lo, hi = need // 2, need
    while lo < hi:
        mid = (lo + hi) // 2
        if score_steps(mid, store, d, sms) >= MIN_STEPS and colstats_steps(mid, store, d, sms) >= MIN_STEPS:
            hi = mid
        else:
            lo = mid + 1
    h = _half(d)
    blocks = max(1, -(-(lo - 2 * TAIL) // (2 * h)))
    return blocks, h, blocks * 2 * h + 2 * TAIL


# dense Gramian cases (store, d, rows): 1, 11 and 64 splits; a last split with no rows (1410 rows at d = 1024: 10 x 144 >= 1410);
# the plain-load staging form (2051 f64, 4099 f32 / bf16); the documented limit d = 8192; many ring wraps per split
GRAMIAN_CASES = [("f32", 128, 20010), ("f64", 1001, 9000), ("f32", 1024, 1410), ("bf16", 1024, 45000), ("f64", 2051, 6006),
                 ("f32", 4096, 3002), ("f32", 4099, 2004), ("bf16", 4099, 2004), ("f64", 8192, 612)]
CSR_ROWS, CSR_D = 110_001, 1000
RANK_DISTINCT, RANK_TIED = 1_200_007, 700_001


def geometry_table(sms):
    """One row per case: what the case reaches under the restated launch rules."""
    rows = []
    for store, d in LONG_DENSE:
        _, _, n = long_rows(store, d, sms)
        g = gramian_geometry(n, d, sms) if d <= GRAMIAN_LONG_MAX_D else None
        rows.append(dict(case=f"dense {store} d={d}", rows=n, score_steps=score_steps(n, store, d, sms),
                         colstats_steps=colstats_steps(n, store, d, sms),
                         splits=g and g[0], chunks=g and g[1], empty_splits=g and g[2]))
    for store, d, n in GRAMIAN_CASES:
        s, c, e = gramian_geometry(n, d, sms)
        rows.append(dict(case=f"gramian {store} d={d}", rows=n, splits=s, chunks=c, empty_splits=e))
    rows.append(dict(case=f"csr d={CSR_D}", rows=CSR_ROWS, score_steps=score_steps(CSR_ROWS, "f32", CSR_D, sms, csr=True),
                     colstats_steps=colstats_steps(CSR_ROWS, "f32", CSR_D, sms, csr=True),
                     gramian_steps=gramian_csr_steps(CSR_ROWS, sms)))
    for name, n, k in (("rank distinct", RANK_DISTINCT, RANK_DISTINCT), ("rank tied", RANK_TIED, 121)):
        t, sc, hi, ar = rank_geometry(n, k)
        rows.append(dict(case=name, rows=n, tiles=t, scan_rounds=sc, hist_rounds=hi, area_blocks_per_thread=ar))
    return rows


def test_geometry_reaches_every_regime():
    """Without a GPU: every case reaches the regime it is there for, under the launch rules restated above."""
    table = geometry_table(H100_SMS)
    for r in table:
        print("  ".join(f"{k}={v}" for k, v in r.items() if v is not None))
    for r in table:
        for k in ("score_steps", "colstats_steps", "gramian_steps"):
            if r.get(k) is not None:
                assert r[k] >= MIN_STEPS, r
        if r.get("chunks") is not None:
            assert r["chunks"] > 2 * 3, r            # every stage of each split's 3-stage ring is refilled
    gm = {r["case"] + f" rows={r['rows']}": r for r in table if r.get("splits") is not None}
    assert {1, 11, 64} <= {r["splits"] for r in gm.values()}, gm
    assert any(r["empty_splits"] for r in gm.values()), gm
    assert any(r["chunks"] >= 12 * 3 and r["splits"] > 1 for r in gm.values()), gm     # a dozen wraps per split
    dist = next(r for r in table if r["case"] == "rank distinct")
    tied = next(r for r in table if r["case"] == "rank tied")
    assert dist["tiles"] > 2 * SCAN_TILES and dist["scan_rounds"] >= 3 and dist["hist_rounds"] >= 3
    assert dist["area_blocks_per_thread"] >= 2
    assert tied["tiles"] > SCAN_TILES and tied["scan_rounds"] >= 2
    # the launch rules restated here are the sources' own: a few fixed points of each
    assert gramian_splits(132, 1024, 1410) == 11 and gramian_splits(132, 128, 9000) == 64
    assert gramian_geometry(1410, 1024, 132)[2] == 1
    assert score_steps(3 * 1056 * 32, "f32", 1024, 132) == 3 and score_steps(3 * 1056 * 32 - 1, "f32", 1024, 132) == 2
    assert colstats_steps(2112, "f32", 1024, 132) == 1 and colstats_steps(2113, "f32", 1024, 132) == 1


# ---------------------------------------------------------------- exact designs
class Design:
    """A dense shard of 2H-row base blocks [P; -P] + c: `blocks` rotated copies, then rows 0..T-1 of P and their mirrors.
    idx[i] = the base row that shard row i is."""

    def __init__(self, d, h, blocks, tail, seed):
        rng = np.random.default_rng(seed)
        p = rng.integers(-4, 5, (h, d), dtype=np.int8)
        p[rng.random((h, d)) < 0.15] = 0
        self.c = rng.integers(-3, 4, d).astype(np.int8)
        if d > 2:
            p[:, 1] = 0
            self.c[1] = 0                                     # an all-zero column
        self.base = np.concatenate([p, -p]) + self.c           # |x| <= 7
        self.y = (rng.random(2 * h) < 0.45).astype(np.float64)
        self.y[rng.random(2 * h) < 0.03] = 2.0                 # rows outside the confusion counts
        self.w = rng.integers(-2, 3, d).astype(np.float64)
        shifts = (np.arange(blocks) * 7919) % (2 * h)
        self.parts = [(np.arange(2 * h) + s) % (2 * h) for s in shifts]
        if tail:
            self.parts.append(np.concatenate([np.arange(tail), h + np.arange(tail)]))
        self.idx = np.concatenate(self.parts)
        self.n = self.idx.shape[0]
        self.d = d
        self.xb = self.base.astype(np.float64)
        self.mb = self.xb @ self.w + B                         # exact: integer products and sums, one dyadic addition

    def counts(self, mask=None):
        sel = self.idx if mask is None else self.idx[mask]
        return np.bincount(sel, minlength=self.base.shape[0]).astype(np.float64)

    def load(self, agd, ctx, store):
        ds = resident(agd, ctx, store, self.d, self.n)
        src = np.float64 if store == "f64" else np.float32
        for part in self.parts:
            ds.load_dense(self.y[part], self.base[part].astype(src), store=store)
        assert ds.local_rows(0) == self.n
        return ds


def resident(agd, ctx, store, d, rows):
    """An empty dataset whose device 0 has room for `rows` rows, so appending blocks does not copy the shard each time."""
    from spark_agd_b200 import _native as N
    ds = agd.DeviceDataset(ctx)
    N.check(N.lib().agd_reserve(ds.h, 0, rows, d, {"f64": N.F64, "f32": N.F32, "bf16": N.BF16}[store]), ds.h)
    return ds


def eval_exact(kind, m, y, t, cnt):
    """The AGD_EVAL_* sums of rows (m, y) with multiplicities cnt, for least squares and hinge (every term a multiple of
    2^-8 far below 2^53, so the dot products are exact)."""
    _, loss = row_terms(kind, m, y)
    e = m - y
    counted = ((y == 0.0) | (y == 1.0)) & (kind == "hinge")
    pos, one = m > t, y == 1.0
    terms = [np.ones_like(m), loss, counted & pos & one, counted & pos & ~one, counted & ~pos & ~one, counted & ~pos & one,
             e, e * e, np.abs(e), y, y * y]
    out = []
    for tm in terms:
        tm = np.asarray(tm, dtype=np.float64)
        assert float(cnt @ np.abs(tm)) < 2.0 ** 44                  # the exactness argument's premise
        out.append(float(cnt @ tm))
    return out


def _eval_got(ev):
    return [ev.count, ev.loss_sum, ev.tp, ev.fp, ev.tn, ev.fn, ev.sum_err, ev.sum_err2, ev.sum_abs_err, ev.sum_y, ev.sum_y2]


def check_evaluate(agd, ds, w, m, y, cnt):
    """least squares and hinge bit for bit, logistic within the bounds of test_score_gpu; (m, y) are the distinct rows and
    cnt how often each is in ds."""
    for kind, t in (("least_squares", 0.5), ("hinge", 0.25)):
        got = _eval_got(ds.evaluate(_grad(agd, kind), w, B, t))
        ref = eval_exact(kind, m, y, t, cnt)
        assert np.array_equal(bits(got), bits(ref)), (kind, got, ref)
    rows_m, rows_y = np.repeat(m, cnt.astype(np.int64)), np.repeat(y, cnt.astype(np.int64))
    with np.errstate(over="ignore"):
        assert np.min(np.abs(1.0 / (1.0 + np.exp(-rows_m)) - 0.3)) > 1e-12
        ref = eval_reference("logistic", rows_m, rows_y, 0.3)
    ev = ds.evaluate(agd.LogisticGradient(), w, B, 0.3)
    for k, (g, (r, mag)) in enumerate(zip(_eval_got(ev), ref)):
        if k in (0, 2, 3, 4, 5):
            assert g == r, (k, g, r)
        else:
            assert abs(g - r) <= 1e-12 * mag, (k, g, r, mag)



def colstats_reference(xb, cnt):
    """Exact sums, counts, maxima and minima of the rows xb with multiplicities cnt; the pass-2 sums about mu = fl(sum / n)
    and the magnitudes of their terms."""
    n = float(cnt.sum())
    s = cnt @ xb
    mu = s / n
    dv = xb - mu
    sel = cnt > 0
    return dict(n=n, sum=s, sum_sq=cnt @ (xb * xb), sum_abs=cnt @ np.abs(xb), nnz=cnt @ (xb != 0).astype(np.float64),
                col_max=xb[sel].max(axis=0), col_min=xb[sel].min(axis=0), dev=cnt @ dv, dev2=cnt @ (dv * dv),
                dev_mag=cnt @ np.abs(dv), nb=int(sel.sum()))


def check_colstats(st, ref, exact_dev):
    assert st.count == ref["n"]
    for f in ("sum", "sum_sq", "sum_abs", "nnz", "col_max", "col_min"):
        assert np.array_equal(bits(getattr(st, f)), bits(ref[f])), (f, np.flatnonzero(getattr(st, f) != ref[f])[:5])
    if exact_dev:
        assert np.array_equal(bits(st.dev), bits(ref["dev"])) and np.array_equal(bits(st.dev2), bits(ref["dev2"]))
        assert np.all(st.dev == 0.0)
        var = (ref["dev2"] - ref["dev"] * ref["dev"] / ref["n"]) / (ref["n"] - 1.0)
        assert np.array_equal(bits(st.variance), bits(var))
    else:
        k = (ref["n"] + ref["nb"] + 2) * U
        assert np.all(np.abs(st.dev - ref["dev"]) <= k * ref["dev_mag"])
        assert np.all(np.abs(st.dev2 - ref["dev2"]) <= k * ref["dev2"])


def gramian_reference(xb, cnt, mu=None):
    a = np.concatenate([xb if mu is None else xb - mu, np.ones((xb.shape[0], 1))], axis=1)
    return a.T @ (cnt[:, None] * a)


def check_gramian(ds, xb, cnt, centered):
    n, aug = ds.gramian(centered)
    assert n == cnt.sum()
    mu = (cnt @ xb) / cnt.sum() if centered else None
    ref = gramian_reference(xb, cnt, mu)
    bad = aug != ref
    assert not bad.any(), (centered, np.argwhere(bad)[:5], aug[bad][:5], ref[bad][:5])


# ---------------------------------------------------------------- the long dense shards
@pytest.mark.gpu
@pytest.mark.parametrize("store,d", LONG_DENSE, ids=[f"{s}-{d}" for s, d in LONG_DENSE])
def test_long_dense(agd, ctx, store, d):
    """Margins, evaluation, colStats, the Gramian (up to d = 4096) and the curve of the whole shard, then of a sample view and a
    randomSplit view (row_in_view / view_bits over many CTAs, chunk ends and tile ends)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    blocks, h, n = long_rows(store, d, sms)
    assert score_steps(n, store, d, sms) >= MIN_STEPS and colstats_steps(n, store, d, sms) >= MIN_STEPS
    dz = Design(d, h, blocks, TAIL, seed=d * 3 + ELEM[store])
    assert dz.n == n
    ds = dz.load(agd, ctx, store)
    try:
        m = ds.margins(dz.w, B)
        ref = dz.mb[dz.idx]
        assert np.array_equal(bits(m), bits(ref)), np.flatnonzero(m != ref)[:5]
        for r0, r in ((n - 1, 1), (n - 2 * TAIL - 5, 2 * TAIL + 5), (n - 40961, 40961), (1, n - 1)):
            assert np.array_equal(bits(ds.margins_rows(0, r0, r, dz.w, B)), bits(ref[r0:r0 + r])), (r0, r)
        cnt = dz.counts()
        check_evaluate(agd, ds, dz.w, dz.mb, dz.y, cnt)
        ref = colstats_reference(dz.xb, cnt)
        assert np.array_equal(ref["sum"], ref["n"] * dz.c)                 # the design: mu = c exactly
        check_colstats(agd.Statistics.colStats(ds), ref, exact_dev=True)
        if d <= GRAMIAN_LONG_MAX_D:
            check_gramian(ds, dz.xb, cnt, centered=False)
            check_gramian(ds, dz.xb, cnt, centered=True)
        check_curve(ds, dz.w, B)
        for view in (ds.sample(False, 0.37, seed=5), ds.randomSplit([0.55, 0.45], seed=9)[1]):
            mask = view.row_mask(0, 0, n)
            cnt = dz.counts(mask)
            assert 0 < cnt.sum() < n
            assert np.array_equal(bits(view.margins(dz.w, B)), bits(dz.mb[dz.idx[mask]]))
            check_evaluate(agd, view, dz.w, dz.mb, dz.y, cnt)
            check_colstats(agd.Statistics.colStats(view), colstats_reference(dz.xb, cnt), exact_dev=False)
            if d <= GRAMIAN_LONG_MAX_D:
                check_gramian(view, dz.xb, cnt, centered=False)
            check_curve(view, dz.w, B)
    finally:
        ds.close()


# ---------------------------------------------------------------- the Gramian's splits, ring and staging forms
@pytest.mark.gpu
@pytest.mark.parametrize("store,d,rows", GRAMIAN_CASES, ids=[f"{s}-{d}-{n}" for s, d, n in GRAMIAN_CASES])
def test_gramian_splits_and_ring(agd, ctx, store, d, rows):
    dz = Design(d, rows // 2, 1, 0, seed=d + rows)
    ds = dz.load(agd, ctx, store)
    try:
        cnt = dz.counts()
        check_gramian(ds, dz.xb, cnt, centered=False)
        check_gramian(ds, dz.xb, cnt, centered=True)                  # mu = c exactly: z is an integer
        check_colstats(agd.Statistics.colStats(ds), colstats_reference(dz.xb, cnt), exact_dev=True)
    finally:
        ds.close()


# ---------------------------------------------------------------- CSR
def _csr_design(seed, n=CSR_ROWS):
    rng = np.random.default_rng(seed)
    d, k = CSR_D, 12
    cols = np.sort(rng.integers(0, d, (n, k)), axis=1)
    keep = (np.arange(k) < rng.integers(0, k + 1, n)[:, None])
    keep[:, 1:] &= cols[:, 1:] != cols[:, :-1]                    # one stored entry per column and row
    keep[[0, 7, n - 1]] = False                                    # empty rows, the last one included
    rp = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int64)
    ix = cols[keep].astype(np.int32)
    va = rng.integers(-4, 5, ix.shape[0]).astype(np.float64)       # zeros among them: explicitly stored
    y = (rng.random(n) < 0.45).astype(np.float64)
    y[rng.random(n) < 0.03] = 2.0
    w = rng.integers(-2, 3, d).astype(np.float64)
    return rp, ix, va, y, w


def _csr_margins(rp, ix, va, w):
    rows = np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp))
    return np.bincount(rows, weights=va * w[ix], minlength=rp.shape[0] - 1) + B


def _csr_colstats(rp, ix, va, d, keep):
    rows = np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp))
    s = keep[rows]
    i, v, n = ix[s], va[s], int(keep.sum())
    stored = np.bincount(i, minlength=d)
    mx = np.full(d, -np.inf)
    mn = np.full(d, np.inf)
    np.maximum.at(mx, i, v)
    np.minimum.at(mn, i, v)
    mx = np.where(stored < n, np.fmax(mx, 0.0), mx)
    mn = np.where(stored < n, np.fmin(mn, 0.0), mn)
    return dict(n=n, sum=np.bincount(i, weights=v, minlength=d), sum_sq=np.bincount(i, weights=v * v, minlength=d),
                sum_abs=np.bincount(i, weights=np.abs(v), minlength=d), nnz=np.bincount(i[v != 0], minlength=d).astype(float),
                col_max=mx, col_min=mn)


def _csr_gramian(rp, ix, va, d, keep):
    from scipy import sparse
    n = rp.shape[0] - 1
    X = sparse.csr_matrix((va, ix, rp), shape=(n, d))[np.flatnonzero(keep)]
    A = sparse.hstack([X, sparse.csr_matrix(np.ones((X.shape[0], 1)))]).tocsc()
    return (A.T @ A).toarray()


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_long_csr(agd, ctx, store):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert score_steps(CSR_ROWS, store, CSR_D, sms, csr=True) >= MIN_STEPS and gramian_csr_steps(CSR_ROWS, sms) >= MIN_STEPS
    rp, ix, va, y, w = _csr_design(17)
    n, d = CSR_ROWS, CSR_D
    h = 40_000
    ds = ctx.parallelize_csr(y[:h], rp[:h + 1], ix[:rp[h]], va[:rp[h]], d, store=store)
    try:
        ds.load_csr(y[h:], rp[h:] - rp[h], ix[rp[h]:], va[rp[h]:], d, store=store)   # an appended partition
        rps, ixs, vas, _ = _stored_csr(ds, store)
        assert np.array_equal(rps, rp) and np.array_equal(ixs, ix) and np.array_equal(vas, va)
        m = _csr_margins(rp, ix, va, w)
        assert np.array_equal(bits(ds.margins(w, B)), bits(m))
        for r0, r in ((n - 1, 1), (n - 33793, 33793)):
            assert np.array_equal(bits(ds.margins_rows(0, r0, r, w, B)), bits(m[r0:r0 + r]))
        views = [(ds, np.ones(n, bool)), (ds.sample(False, 0.37, seed=5), None), (ds.randomSplit([0.55, 0.45], seed=9)[1], None)]
        for v, keep in views:
            keep = v.row_mask(0, 0, n) if keep is None else keep
            check_evaluate(agd, v, w, m, y, keep.astype(np.float64))
            st = agd.Statistics.colStats(v)
            ref = _csr_colstats(rp, ix, va, d, keep)
            assert st.count == ref["n"]
            for f in ("sum", "sum_sq", "sum_abs", "nnz", "col_max", "col_min"):
                assert np.array_equal(bits(getattr(st, f)), bits(ref[f])), f
            cols = csr_cols(rp, ix, va, d, keep)
            sub = np.arange(0, d, 61)
            check_summary(_Sub(st, sub), [cols[j] for j in sub], int(keep.sum()))
            cnt, aug = v.gramian(False)
            assert cnt == keep.sum() and np.array_equal(aug, _csr_gramian(rp, ix, va, d, keep))
            check_curve(v, w, B)
    finally:
        ds.close()


# ---------------------------------------------------------------- ranking
@pytest.mark.gpu
def test_rank_distinct_keys_past_every_single_round(ctx):
    """K > 524,288 distinct margins over more than 512 tiles: the tile scans take three rounds, bin_hist8 strides and
    bin_area_final gives each thread several blocks."""
    rng = np.random.default_rng(21)
    n = RANK_DISTINCT
    x = (rng.permutation(n) - n // 2) * 0.375
    y = (rng.random(n) < 0.4).astype(np.float64)
    ds = ctx.parallelize(y, x.reshape(-1, 1), store="f64")
    try:
        _, K = check_curve(ds, np.array([1.0]), 0.0)
        assert K == n
        view = ds.sample(False, 0.7, seed=4)
        _, Kv = check_curve(view, np.array([1.0]), 0.0)
        assert Kv == int(view.row_mask(0, 0, n).sum()) and rank_geometry(Kv, Kv)[1] >= 2
    finally:
        ds.close()


@pytest.mark.gpu
def test_rank_heavy_ties_over_many_tiles(ctx):
    rng = np.random.default_rng(22)
    n = RANK_TIED
    x = rng.integers(-60, 61, n).astype(np.float64)
    y = (rng.random(n) < 0.5).astype(np.float64)
    ds = ctx.parallelize(y, x.reshape(-1, 1), store="f64")
    try:
        _, K = check_curve(ds, np.array([1.0]), 0.25)
        assert K == 121
    finally:
        ds.close()


# ---------------------------------------------------------------- one shard past 2^31 elements
@pytest.mark.gpu
@pytest.mark.parametrize("store", ["bf16", "f32"])
def test_shard_past_2_31_elements(agd, ctx, store):
    """A 65,536 x 1024 block appended 34 times into a reserved shard: 2.28e9 elements (4.6 GB in bf16, 9.1 GB in fp32).
    Every reference follows from the block: sums are 34 x the block's, the margins are the block's tiled, the curve's counts
    are 34 x the block's at the same keys.  The least-squares gradient is exact too: every fp32 margin, every bf16 x 3 split
    of a residual and every 16-row fp32 sum of the wgmma kernel is an integer below 2^24.  So is the projection, whose rows
    are the block's projected rows tiled (tests/test_project_long_gpu.py's exact design)."""
    rows_b, d, reps = 65536, 1024, 34
    dz = Design(d, rows_b // 2, 1, 0, seed=31)
    n = rows_b * reps
    assert n * d > 2 ** 31 and n * d * ELEM[store] > 2 ** 32
    blk = dz.base[dz.idx].astype(np.float32)
    yb = dz.y[dz.idx]
    xb = blk.astype(np.float64)
    ds = resident(agd, ctx, store, d, n)
    try:
        for _ in range(reps):
            ds.load_dense(yb, blk, store=store)
        assert ds.local_rows(0) == n
        cnt = np.full(rows_b, float(reps))
        ref = colstats_reference(xb, cnt)
        check_colstats(agd.Statistics.colStats(ds), ref, exact_dev=True)
        check_gramian(ds, xb, cnt, centered=False)
        check_gramian(ds, xb, cnt, centered=True)
        mb = xb @ dz.w + B
        m = ds.margins(dz.w, B)
        assert np.array_equal(bits(m), bits(np.tile(mb, reps)))
        summary, cm, tp, fp = ds.binary_curve(dz.w, B)
        rm, rtp, rfp, _ = R.curve(mb, yb)
        assert np.array_equal(bits(cm), bits(rm)) and np.array_equal(tp, reps * rtp) and np.array_equal(fp, reps * rfp)
        au, ap = R.areas(reps * rtp, reps * rfp)
        assert summary[0] == reps * rtp[-1] and summary[1] == reps * rfp[-1] and summary[2] == 0
        assert abs(summary[3] - au) <= 1e-12 * au and abs(summary[4] - ap) <= 1e-12 * ap
        # least-squares smooth: loss = sum (m - y)^2 / n, grad = sum 2 (m - y) x / n, with integer sums
        m0 = xb @ dz.w
        r = m0 - yb
        assert np.max(np.abs(m0)) < 2 ** 24 and np.max(np.abs(2 * r)) < 2 ** 24
        S = reps * (xb.T @ (2.0 * r))
        L = reps * float(r @ r)
        assert np.max(np.abs(S)) < 2 ** 53 and L < 2 ** 53
        for variant in (["ring", "tc"] if store == "bf16" else ["ring"]):
            ds.set_option("k1_variant", variant)
            loss, g, c = ds.smooth(agd.LeastSquaresGradient(), dz.w)
            assert c == n and loss == L / n, (variant, loss, L / n)
            assert np.array_equal(bits(g), bits(S / n)), (variant, np.flatnonzero(g != S / n)[:5])
        # the projection, with B and c in 2^-20 Z (exact: every sum is below 2^14): the block's rows tiled, into fp64 at k = 16,
        # into fp32 at k = 130 (two column tiles), and through a sample view of 17,408 row tiles (17 per scan thread).  Each
        # projection is closed before the next.
        from test_project_long_gpu import check_rows, exact_B, exact_projection, expected_bits
        rng = np.random.default_rng(32)
        ridx = np.arange(n) % rows_b
        view = ds.sample(False, 0.37, seed=5)
        for src, dest, k, sel in ((ds, "f64", 16, ridx), (ds, "f32", 130, ridx),
                                  (view, "f64", 16, ridx[view.row_mask(0, 0, n)])):
            Bp, cp = exact_B(rng, d, k)
            want = expected_bits(exact_projection(xb, Bp, cp), dest)
            p = src.project(Bp, cp, store=dest)
            try:
                check_rows(p, dest, k, want, sel, yb)
            finally:
                p.close()
    finally:
        ds.close()
