"""KMeans (agd_kmeans_*, csrc/kmeans.cu) on shards long enough to reach the code a few thousand rows never run, against exact
references: a dense assignment of more than 65,535 row tiles (a second launch, ending on a ragged tile), with one and with
three column tiles; a dense shard past 2^31 elements in the plain-load form; CSR warps that each take dozens of rows over three
128-centre passes.

Exact design.  Features are small integers (|x| <= 7, tests/test_long_streams_gpu.py's Design) and centres lie in 2^-10 Z with
|c| <= 4, so every score, distance, sum and cost is exact in fp64 in any order: assignments, distances, sums, counts and the
cost must equal numpy's bit for bit.  The shards are rotated copies of a base block, so the reference is computed once per
base row and expanded through the row map.

Geometry.  The cases follow from the launch rules restated below (the projection's row tile, tests/test_project_long_gpu.py,
and the warp-per-row grids of kmeans.cu); test_geometry_reaches_every_regime checks them without a GPU."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_long_streams_gpu import H100_SMS, _csr_design  # noqa: E402
from test_project_long_gpu import dense_launches, fill, long_design, staging, tile_cols  # noqa: E402
from test_score_gpu import bits  # noqa: E402

# ---------------------------------------------------------------- the launch rules, restated
# kernel                 source                              rule
# kmeans_dense_kernel    pj_tile.cuh pj_launch_rows,         kPjRows = 128 rows per CTA, kp / BN column tiles side by side;
#                        kmeans.cu launch_dense_t            one launch per 65,535 row tiles; kp > 128: kmeans_tiles_kernel
#                                                            merges kp / 128 tiles per row
# kmeans_csr_kernel      kmeans.cu warp_grid                 one warp per row, grid-stride; min(per_sm SMs, ceil(rows / 8))
#                                                            CTAs of 8 warps, per_sm <= 2048 / 256; 32 x 4 = 128 centres per pass
KPJ_ROWS = 128
CSR_WARPS = 256 // 32
CSR_PER_SM_MAX = 2048 // 256
CSR_PASS = 32 * 4

G1_ROWS = 65535 * KPJ_ROWS + 3 * KPJ_ROWS + 77      # f32, d = 3: a second launch of 4 row tiles, the last one ragged
P_ROWS, P_D = 2 ** 19, 4099                         # bf16: past 2^31 elements, plain loads
CSR_ROWS = 300_007


def csr_rows_per_warp(rows, sms):
    grid = max(1, min(CSR_PER_SM_MAX * sms, -(-rows // CSR_WARPS)))
    return rows // (grid * CSR_WARPS)


def test_geometry_reaches_every_regime():
    ln = dense_launches(G1_ROWS)
    assert len(ln) == 2 and ln[1] == (65535, 4) and G1_ROWS % KPJ_ROWS == 77
    assert staging("f32", 3) == (4, "cp.async")
    assert -(-300 // tile_cols(300)) == 3 and -(-16 // tile_cols(16)) == 1
    stored, form = staging("bf16", P_D)
    assert form == "plain" and P_ROWS * stored > 2 ** 31
    assert csr_rows_per_warp(CSR_ROWS, H100_SMS) >= 30 and -(-300 // CSR_PASS) == 3


def centres(k, d, seed):
    rng = np.random.default_rng(seed)
    C = rng.integers(-4 * 1024, 4 * 1024 + 1, (k, d)) / 1024.0
    if k >= 3:
        C[2] = C[1]
    return C


def base_reference(base, C):
    """(closest centre, exact residual) of every base row, in chunks."""
    b = base.astype(np.float64)
    cl = np.empty(b.shape[0], dtype=np.int64)
    dist = np.empty(b.shape[0])
    for i in range(0, b.shape[0], 4096):
        D = ((b[i:i + 4096, None, :] - C[None]) ** 2).sum(axis=2)
        cl[i:i + 4096] = np.argmin(D, axis=1)
        dist[i:i + 4096] = D[np.arange(D.shape[0]), cl[i:i + 4096]]
    return cl, dist


def check_long(ds, C, base, idx):
    cl, dist = base_reference(base, C)
    mult = np.bincount(idx, minlength=base.shape[0]).astype(np.float64)
    k = C.shape[0]
    counts = np.bincount(cl, weights=mult, minlength=k)
    sums = np.zeros_like(C)
    np.add.at(sums, cl, base.astype(np.float64) * mult[:, None])
    s, c, cost = ds.kmeans_step(C)
    np.testing.assert_array_equal(c, counts)
    assert np.array_equal(bits(s), bits(sums))
    assert cost == float((dist * mult).sum())
    got_cl, got_d = ds.kmeans_assign(C)
    assert np.array_equal(got_cl, cl[idx])
    assert np.array_equal(bits(got_d), bits(dist[idx]))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [16, 300])
def test_second_dense_launch(agd, ctx, k):
    dz = long_design(3, G1_ROWS, seed=41)
    ds = fill(agd, ctx, "f32", dz, dz.base)
    try:
        check_long(ds, centres(k, 3, k), dz.base, dz.idx)
    finally:
        ds.close()


@pytest.mark.gpu
def test_shard_past_2_31_elements_plain_loads(agd, ctx):
    dz = long_design(P_D, P_ROWS, seed=43, h=4096)
    ds = fill(agd, ctx, "bf16", dz, dz.base)
    try:
        check_long(ds, centres(16, P_D, 7), dz.base, dz.idx)
    finally:
        ds.close()


@pytest.mark.gpu
def test_csr_many_rows_per_warp(agd, ctx):
    import scipy.sparse as sp
    rp, ix, va, y, _ = _csr_design(9, CSR_ROWS)
    d = 1000
    X = sp.csr_matrix((va, ix, rp), shape=(CSR_ROWS, d))
    ds = ctx.parallelize_csr(y, rp, ix, va, d, store="f64")
    try:
        C = centres(300, d, 3)
        cn = (C * C).sum(axis=1)
        cl = np.empty(CSR_ROWS, dtype=np.int64)
        dist = np.empty(CSR_ROWS)
        for i in range(0, CSR_ROWS, 20000):
            blk = X[i:i + 20000]
            D = np.asarray(blk.multiply(blk).sum(axis=1)) - 2 * (blk @ C.T) + cn   # exact under the design
            cl[i:i + 20000] = np.argmin(D, axis=1)
            dist[i:i + 20000] = D[np.arange(D.shape[0]), cl[i:i + 20000]]
        got_cl, got_d = ds.kmeans_assign(C)
        assert np.array_equal(got_cl, cl)
        assert np.array_equal(bits(got_d), bits(dist))
        s, c, cost = ds.kmeans_step(C)
        np.testing.assert_array_equal(c, np.bincount(cl, minlength=300))
        sums = np.asarray((sp.csr_matrix((np.ones(CSR_ROWS), (cl, np.arange(CSR_ROWS))), shape=(300, CSR_ROWS)) @ X).todense())
        assert np.array_equal(bits(s), bits(sums))
        assert cost == float(dist.sum())
    finally:
        ds.close()
