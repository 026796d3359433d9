"""The projection (agd_project, csrc/project.cu) on shards long enough to reach the code that a few thousand rows never run,
against exact references.  tests/test_project_gpu.py stops at 32 row tiles: one dense launch, a view scan whose threads each
take at most one tile, a CSR grid where no warp takes a second row, and outputs far below 2^31 elements.  Here the dense
kernel takes a second launch (more than 65,535 row tiles), the scan gives each thread 65 tiles with threads left idle, the
output passes 2^31 elements and 2^32 bytes, and every CSR warp takes dozens of rows over three 128-column passes.

Exact design.  Features are small integers (|x| <= 7, tests/test_long_streams_gpu.py's Design), exact in bf16, fp32 and fp64;
B has entries in 2^-20 Z with |b| <= 2 and the offset c entries in 2^-20 Z, all nonzero (so no correct row is all zeros).
Every product and partial sum is then a multiple of 2^-20 below 2^33, so numpy's fp64 X B + c over the base block is exact in
any order: fp64 destinations must equal it bit for bit, fp32 ones its round-to-nearest-even to fp32 and bf16 ones rne_bf16
of it.  The shard is made of rotated copies of the base block, so row i of a projection must be expected[idx[i]]: every row
is compared, downloaded in chunks.

Geometry.  The cases are derived from the launch rules restated below, with an upper bound on the CSR grid, so each regime is
reached whatever the occupancy; test_geometry_reaches_every_regime checks that without a GPU.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_long_streams_gpu import CSR_D, H100_SMS, Design, _csr_design, resident  # noqa: E402
from test_project_gpu import _B, _matrix, check_projection, rne_bf16  # noqa: E402
from test_score_gpu import _stored_csr, bits  # noqa: E402

# ---------------------------------------------------------------- the launch rules, restated
# kernel                 source                              rule
# project_dense_kernel   agd_common.cuh:310, project.cu:31,  kPjRows = 128 rows per CTA, kp / BN column tiles side by side
#                        104-116, 250-282, 286               (BN = 16, 32, 64 or 128 by k); one launch per kPjMaxGridY =
#                                                            65,535 row tiles, the launch at rt0 covering tiles rt0 ..
# project_scan_kernel    project.cu:28, 70-99                one CTA of 1,024 threads; thread t takes tiles [t per, t per +
#                                                            per), per = ceil(tiles / 1024)
# project_csr_kernel     project.cu:24, 30, 218-248, 301-314 one warp per row, grid-stride over rows; min(per_sm SMs,
#                                                            ceil(rows / 8)) CTAs of 8 warps, per_sm <= 2048 / 256; lanes over
#                                                            32 x 4 = 128 output columns per pass
# stored width           agd_api.cu:303-321,                 a dense row of user width d is stored padded to whole 16-byte
#                        k1_dense.cu:743-769                 vectors when the ring kernels take the padded width (at most
#                                                            512 vectors in bf16, 1024 otherwise); the dense kernel stages
#                                                            rows of whole vectors with cp.async, others with plain loads
KPJ_ROWS = 128
MAX_GRID_Y = 65535
SCAN_THREADS = 1024
CSR_WARPS = 256 // 32
CSR_PER_SM_MAX = 2048 // 256
CSR_PASS_COLS = 32 * 4


ELEM = {"f32": 4, "f64": 8, "bf16": 2}


def staging(store, d):
    """(stored width, form of the dense kernel) of a shard of user width d."""
    epv = 16 // ELEM[store]
    padded = -(-d // epv) * epv
    stored = padded if padded // epv <= (512 if store == "bf16" else 1024) else d
    return stored, "cp.async" if stored % epv == 0 else "plain"


def tile_cols(k):
    """project_tile_cols."""
    return 16 if k <= 16 else (32 if k <= 32 else (64 if k <= 64 else 128))


def dense_launches(rows):
    """(rt0, row tiles) of each launch of launch_dense."""
    tiles = -(-rows // KPJ_ROWS)
    return [(rt0, min(MAX_GRID_Y, tiles - rt0)) for rt0 in range(0, tiles, MAX_GRID_Y)]


def scan_geometry(rows):
    """(tiles, tiles per thread, threads with no tile) of project_scan_kernel."""
    tiles = -(-rows // KPJ_ROWS)
    per = -(-tiles // SCAN_THREADS)
    return tiles, per, SCAN_THREADS - -(-tiles // per)


def csr_rows_per_warp(rows, sms):
    """Fewest rows any warp of project_csr_kernel takes, with the grid at its upper bound."""
    grid = max(1, min(CSR_PER_SM_MAX * sms, -(-rows // CSR_WARPS)))
    return rows // (grid * CSR_WARPS)


# ---------------------------------------------------------------- the cases
G1_ROWS = MAX_GRID_Y * KPJ_ROWS + 3 * KPJ_ROWS + 77      # f32, d = 3, k = 16: a second launch of 4 tiles, the last one ragged
G2_ROWS = 2 ** 31 // 256 + 1001                          # bf16, d = 8, k = 256: Y past 2^31 elements and 2^32 bytes
G2_K = 256
CSR_LONG_ROWS = 300_007                                  # CSR, d = 1000, k = 5 and 300
SHARD_2_31_ROWS = 65536 * 34                             # test_long_streams_gpu.test_shard_past_2_31_elements (cp.async form)
P_ROWS, P_D = 2 ** 19, 4099                              # bf16: a source past 2^31 elements in the plain-load form


def geometry_table(sms):
    out = []
    for name, store, d, rows, k in (("G1 f32 d=3", "f32", 3, G1_ROWS, 16), ("G2 bf16 d=8", "bf16", 8, G2_ROWS, G2_K),
                                    ("P bf16 d=4099", "bf16", P_D, P_ROWS, 16)):
        ln = dense_launches(rows)
        stored, form = staging(store, d)
        out.append(dict(case=name, rows=rows, form=form, x_elems=rows * stored, launches=len(ln),
                        last_launch_tiles=ln[-1][1], ragged=rows % KPJ_ROWS, col_tiles=-(-k // tile_cols(k)), y_elems=rows * k))
    for name, rows in (("V view of G1", G1_ROWS), ("C csr view", CSR_LONG_ROWS), ("S view of the 2^31 shard", SHARD_2_31_ROWS)):
        t, per, idle = scan_geometry(rows)
        out.append(dict(case=name, rows=rows, tiles=t, tiles_per_thread=per, idle_threads=idle))
    out.append(dict(case="C csr", rows=CSR_LONG_ROWS, rows_per_warp=csr_rows_per_warp(CSR_LONG_ROWS, sms),
                    passes_k300=-(-300 // CSR_PASS_COLS)))
    return out


def test_geometry_reaches_every_regime():
    """Without a GPU: every case reaches the regime it is there for, under the launch rules restated above."""
    table = geometry_table(H100_SMS)
    for r in table:
        print("  ".join(f"{k}={v}" for k, v in r.items()))
    g = {r["case"]: r for r in table}
    g1, g2 = g["G1 f32 d=3"], g["G2 bf16 d=8"]
    assert g1["launches"] == 2 and g1["last_launch_tiles"] == 4 and g1["ragged"] == 77
    assert g2["launches"] == 2 and g2["col_tiles"] == 2
    assert g2["y_elems"] > 2 ** 31 and g2["y_elems"] * 4 > 2 ** 32      # the f32 destination
    assert g1["form"] == g2["form"] == "cp.async"
    assert g["P bf16 d=4099"]["form"] == "plain" and g["P bf16 d=4099"]["x_elems"] > 2 ** 31
    v = g["V view of G1"]
    assert v["tiles"] == 65539 and v["tiles"] > MAX_GRID_Y and v["tiles_per_thread"] == 65 and v["idle_threads"] > 0
    c = g["C csr view"]
    assert c["tiles"] > SCAN_THREADS and c["tiles_per_thread"] >= 2
    assert g["S view of the 2^31 shard"]["tiles"] == 17408 and g["S view of the 2^31 shard"]["tiles_per_thread"] == 17
    assert g["C csr"]["rows_per_warp"] >= 3 and g["C csr"]["passes_k300"] == 3
    # the launch rules restated here are the sources' own: a few fixed points of each
    assert dense_launches(MAX_GRID_Y * KPJ_ROWS) == [(0, MAX_GRID_Y)]
    assert dense_launches(MAX_GRID_Y * KPJ_ROWS + 1) == [(0, MAX_GRID_Y), (MAX_GRID_Y, 1)]
    assert scan_geometry(SCAN_THREADS * KPJ_ROWS) == (1024, 1, 0)
    assert scan_geometry(SCAN_THREADS * KPJ_ROWS + 1) == (1025, 2, 511)
    assert [tile_cols(k) for k in (1, 16, 17, 33, 64, 65, 300)] == [16, 16, 32, 64, 64, 128, 128]
    assert staging("f32", 3) == (4, "cp.async") and staging("f32", 4099) == (4099, "plain")
    assert staging("f64", 2048) == (2048, "cp.async") and staging("f64", 2051) == (2051, "plain")
    assert staging("bf16", 4090) == (4096, "cp.async") and staging("bf16", 4099) == (4099, "plain")
    assert csr_rows_per_warp(8448, 132) == 1 and csr_rows_per_warp(8447, 132) == 0     # 1,056 CTAs x 8 warps


# ---------------------------------------------------------------- exact designs and references
DT = {"f64": (np.float64, np.uint64), "f32": (np.float32, np.uint32), "bf16": (np.uint16, np.uint16)}


def long_design(d, rows, seed, h=32768):
    """A Design of exactly `rows` rows: rotated 2h-row blocks, a tail and, when rows is odd, one more row of P."""
    blocks, rem = divmod(rows, 2 * h)
    dz = Design(d, h, blocks, rem // 2, seed)
    if rem % 2:
        dz.parts.append(np.array([h // 3]))
        dz.idx = np.concatenate(dz.parts)
        dz.n = dz.idx.shape[0]
    assert dz.n == rows
    return dz


def exact_B(rng, d, k):
    """B in 2^-20 Z with |b| <= 2, and c in 2^-20 Z with every c_j nonzero."""
    B = rng.integers(-2 ** 21, 2 ** 21 + 1, (d, k)) * 2.0 ** -20
    c = rng.integers(1, 2 ** 21 + 1, k) * rng.choice([-1.0, 1.0], k) * 2.0 ** -20
    return B, c


def exact_projection(X, B, c):
    """X B + c for integer rows X (dense or scipy sparse, |x| <= 7): every term and partial sum is a multiple of 2^-20 below
    2^33, so this fp64 product is exact whatever order the BLAS sums in."""
    assert abs(X).max() <= 7
    assert np.max(abs(X) @ np.abs(B)) + np.max(np.abs(c)) < 2.0 ** 33
    Y = np.asarray(X @ B) + c
    assert not np.all(Y == 0, axis=1).any()
    return Y


def expected_bits(Y, dest):
    """The bits a `dest` destination must hold for the exact fp64 rows Y: Y itself, or rounded once to nearest-even."""
    if dest == "f64":
        return Y.view(np.uint64)
    if dest == "f32":
        return Y.astype(np.float32).view(np.uint32)
    return rne_bf16(Y)


def check_rows(p, dest, k, want, ridx, labels, chunk_bytes=256 << 20):
    """Row i of the projection p holds want[ridx[i]] bit for bit and the label labels[ridx[i]]: every row, downloaded in chunks
    of about chunk_bytes so host memory stays small."""
    n = p.local_rows(0)
    assert n == ridx.shape[0] and p.d == k, (n, ridx.shape[0], p.d, k)
    dt, ut = DT[dest]
    step = max(1, chunk_bytes // (k * np.dtype(dt).itemsize))
    for r0 in range(0, n, step):
        sel = ridx[r0:r0 + step]
        X, y = p.get_rows(0, r0, sel.shape[0], dtype=dt)
        bad = np.flatnonzero((X.view(ut) != want[sel]).any(axis=1))
        assert bad.shape[0] == 0, (dest, n, bad.shape[0], r0 + bad[:5], X[bad[:2]], want[sel[bad[:2]]].view(dt))
        badl = np.flatnonzero(bits(y) != bits(labels[sel]))
        assert badl.shape[0] == 0, (r0 + badl[:5], y[badl[:5]], labels[sel[badl[:5]]])


def fill(agd, ctx, store, dz, base, poison=None):
    """dz's shard with another base block of the same shape (Design.load's row order and labels); poison = (rows, values)
    replaces those rows."""
    ds = resident(agd, ctx, store, dz.d, dz.n)
    r0 = 0
    for part in dz.parts:
        X = base[part].astype(np.float32)
        if poison is not None:
            at = (poison[0] >= r0) & (poison[0] < r0 + part.shape[0])
            X[poison[0][at] - r0] = poison[1][at]
        ds.load_dense(dz.y[part], X, store=store)
        r0 += part.shape[0]
    assert ds.local_rows(0) == dz.n
    return ds


def _views(ds):
    return [ds.sample(False, 0.37, seed=5), ds.randomSplit([0.55, 0.45], seed=9)[1]]


# ---------------------------------------------------------------- dense: a second launch
@pytest.mark.gpu
def test_second_dense_launch(agd, ctx):
    """8,388,941 rows: 65,539 row tiles in two launches, the second of 4 tiles ending on a ragged one.  fp64 and fp32
    destinations, the labels, and randomSplit of the projection selecting the rows of the same split of the source."""
    n = G1_ROWS
    dz = long_design(3, n, seed=41)
    B, c = exact_B(np.random.default_rng(1), 3, 16)
    Y = exact_projection(dz.xb, B, c)
    ds = dz.load(agd, ctx, "f32")
    try:
        for dest in ("f64", "f32"):
            p = ds.project(B, c, store=dest)
            try:
                check_rows(p, dest, 16, expected_bits(Y, dest), dz.idx, dz.y)
                if dest == "f64":
                    for a, b in zip(ds.randomSplit([0.55, 0.45], seed=9), p.randomSplit([0.55, 0.45], seed=9)):
                        assert np.array_equal(a.row_mask(0, 0, n), b.row_mask(0, 0, n))
            finally:
                p.close()
    finally:
        ds.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dest", ["bf16", "f32"])
def test_output_past_2_31_elements(agd, ctx, dest):
    """8,389,609 bf16 rows of d = 8 (the cp.async form) into k = 256 columns: two launches, two 128-column tiles, and a
    destination of 2.15e9 elements (8.6 GB in fp32)."""
    dz = long_design(8, G2_ROWS, seed=43)
    B, c = exact_B(np.random.default_rng(2), 8, G2_K)
    want = expected_bits(exact_projection(dz.xb, B, c), dest)
    ds = dz.load(agd, ctx, "bf16")
    try:
        p = ds.project(B, c, store=dest)
        try:
            assert p.local_rows(0) * G2_K > 2 ** 31
            check_rows(p, dest, G2_K, want, dz.idx, dz.y)
        finally:
            p.close()
    finally:
        ds.close()


@pytest.mark.gpu
def test_plain_load_source_past_2_31_elements(agd, ctx):
    """524,288 bf16 rows of d = 4099 (rows of 8,198 bytes: the plain-load form) hold 2.15e9 elements (4.3 GB): the rows past
    2^31 elements are read at 64-bit offsets."""
    dz = Design(P_D, 4096, P_ROWS // 8192, 0, seed=53)
    assert dz.n == P_ROWS and dz.n * P_D > 2 ** 31
    B, c = exact_B(np.random.default_rng(6), P_D, 16)
    want = expected_bits(exact_projection(dz.xb, B, c), "f64")
    ds = dz.load(agd, ctx, "bf16")
    try:
        p = ds.project(B, c)
        try:
            check_rows(p, "f64", 16, want, dz.idx, dz.y)
        finally:
            p.close()
    finally:
        ds.close()


# ---------------------------------------------------------------- views: the scan over 65,539 tiles
@pytest.mark.gpu
def test_view_scan_over_many_tiles(agd, ctx):
    """G1's shard through a sample and a randomSplit view: the scan gives each thread 65 tiles and leaves 15 idle, and the kept
    rows of the second launch are placed after those of the first.  Then the same views of a copy with +-inf and NaN in rows
    outside both views, in tiles past the first 1,024 and in the second launch: they leave no trace."""
    n = G1_ROWS
    dz = long_design(3, n, seed=41)
    B, c = exact_B(np.random.default_rng(3), 3, 16)
    want = expected_bits(exact_projection(dz.xb, B, c), "f64")
    ds = dz.load(agd, ctx, "f32")
    try:
        masks = [v.row_mask(0, 0, n) for v in _views(ds)]
        for v, m in zip(_views(ds), masks):
            assert 0 < m.sum() < n and m[MAX_GRID_Y * KPJ_ROWS:].any()
            p = v.project(B, c)
            try:
                check_rows(p, "f64", 16, want, dz.idx[m], dz.y)
            finally:
                p.close()
    finally:
        ds.close()
    out = np.flatnonzero(~(masks[0] | masks[1]))
    rows = np.concatenate([out[out >= SCAN_THREADS * KPJ_ROWS][:40], out[out >= n // 2][:40],
                           out[out >= MAX_GRID_Y * KPJ_ROWS][:40], out[-3:]])
    vals = np.tile(np.array([[np.inf, 1, 2], [3, -np.inf, 4], [np.nan, 5, 6], [np.nan] * 3, [np.inf, np.nan, -np.inf]],
                            dtype=np.float32), (-(-rows.shape[0] // 5), 1))[:rows.shape[0]]
    ds = fill(agd, ctx, "f32", dz, dz.base, poison=(rows, vals))
    try:
        for v, m in zip(_views(ds), masks):
            assert np.array_equal(v.row_mask(0, 0, n), m)
            p = v.project(B, c)
            try:
                check_rows(p, "f64", 16, want, dz.idx[m], dz.y)
            finally:
                p.close()
    finally:
        ds.close()


# ---------------------------------------------------------------- position invariance, with rounding
@pytest.mark.gpu
def test_bits_depend_only_on_the_row(agd, ctx):
    """A G1-sized shard of copies of a random fp32 block, projected by a random fp64 B: every copy of a row has the bits of
    that row's projection in a short shard of the block alone (held to the gamma bound of test_project_gpu), whichever tile,
    launch and in-tile offset it lands in."""
    n = G1_ROWS
    dz = long_design(3, n, seed=47)
    rng = np.random.default_rng(4)
    base = _matrix(rng, dz.base.shape[0], 3).astype(np.float32)
    B, c = _B(rng, 3, 16)
    short = ctx.parallelize(dz.y, base, store="f32")
    try:
        p = short.project(B, c)
        try:
            Ys = p.get_rows(0, 0, base.shape[0], dtype=np.float64)[0]
        finally:
            p.close()
    finally:
        short.close()
    check_projection(Ys, base.astype(np.float64), B, c)
    ds = fill(agd, ctx, "f32", dz, base)
    try:
        p = ds.project(B, c)
        try:
            check_rows(p, "f64", 16, Ys.view(np.uint64), dz.idx, dz.y)
        finally:
            p.close()
    finally:
        ds.close()


# ---------------------------------------------------------------- CSR: many rows per warp, three column passes
@pytest.mark.gpu
@pytest.mark.parametrize("store", ["f32", "f64"])
def test_csr_many_rows_per_warp(agd, ctx, store):
    """300,007 CSR rows of at most 12 integer entries (empty rows, the last one included): every warp takes dozens of rows,
    k = 300 takes three 128-column passes, and a sample view's scan covers 2,344 tiles."""
    from scipy import sparse
    n, d = CSR_LONG_ROWS, CSR_D
    rp, ix, va, y, _ = _csr_design(29, n)
    assert rp[1] == rp[0] and rp[-1] == rp[-2]
    X = sparse.csr_matrix((va, ix, rp), shape=(n, d))
    ds = ctx.parallelize_csr(y, rp, ix, va, d, store=store)
    try:
        rps, ixs, vas, _ = _stored_csr(ds, store)
        assert np.array_equal(rps, rp) and np.array_equal(ixs, ix) and np.array_equal(vas, va)
        view = ds.sample(False, 0.37, seed=5)
        keep = np.flatnonzero(view.row_mask(0, 0, n))
        rng = np.random.default_rng(5)
        for k in (5, 300):
            B, c = exact_B(rng, d, k)
            want = expected_bits(exact_projection(X, B, c), "f64")
            for src, ridx in ((ds, np.arange(n)), (view, keep)):
                p = src.project(B, c)
                try:
                    check_rows(p, "f64", k, want, ridx, y)
                finally:
                    p.close()
    finally:
        ds.close()
