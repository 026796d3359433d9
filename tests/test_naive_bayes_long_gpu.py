"""NaiveBayes and MulticlassMetrics (agd_label_classes / agd_class_sums / agd_linear_argmax / agd_linear_confusion) on a shard
long enough to reach the code a few thousand rows never run, against exact references: a dense argmax of more than 65,535 row
tiles (a second launch, ending on a ragged tile) with one and with three 128-class column tiles, a label sort over thousands of
tiles, and a confusion count in one and in several label slices.

Exact design (tests/test_naive_bayes_gpu.py): small nonnegative integer features, dyadic theta / pi, so class sums, counts and
scores are exact in fp64 in any order.  The shard is a 65,536-row block loaded again and again, so the reference is computed once
per block row and weighted by how often the row occurs.

Geometry.  The cases follow from the launch rules restated below; test_geometry_reaches_every_regime checks them without a GPU."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_naive_bayes_gpu import design, label_values, metric_values, same  # noqa: E402
from test_project_long_gpu import dense_launches, staging, tile_cols  # noqa: E402

# ---------------------------------------------------------------- the launch rules, restated
# kernel                   source                              rule
# kmeans_dense_kernel      pj_tile.cuh pj_launch_rows,         kPjRows = 128 rows per CTA, kp / BN column tiles side by side;
#  (kKmLinear)             kmeans.cu launch_dense_t            one launch per 65,535 row tiles; kp > 128: kmeans_tiles_kernel
# label_keys_kernel /      rank.cu bin_sort_pairs,             tiles of kTile = 256 x 8 = 2,048 keys; the offsets kernel scans
#  bin_sort_pairs          tiles_of                            the tile counts 256 at a time per digit
# label_confusion_kernel   classify.cu label_confusion_launch  shared histograms of lps = min(L, 12,288 / C) label rows;
#                                                              gridDim.y = ceil(L / lps) slices, the last one partial
KPJ_ROWS = 128
SORT_TILE = 256 * 8
SMEM_COUNTERS = 48 * 1024 // 4
BLOCK = 65_536
ROWS = 65535 * KPJ_ROWS + 3 * KPJ_ROWS + 77          # f32, d = 3: a second launch of 4 row tiles, the last one ragged
D = 3


def test_geometry_reaches_every_regime():
    ln = dense_launches(ROWS)
    assert len(ln) == 2 and ln[1] == (65535, 4) and ROWS % KPJ_ROWS == 77
    assert staging("f32", D) == (4, "cp.async")
    assert -(-300 // tile_cols(300)) == 3 and -(-16 // tile_cols(16)) == 1
    assert -(-ROWS // SORT_TILE) > 16 * 256                       # the tile scan takes many rounds of 256 tiles
    lps = SMEM_COUNTERS // 300
    assert 16 * 16 <= SMEM_COUNTERS and -(-300 // lps) == 8 and 300 % lps != 0   # C = 16: one slice; 300: 8, the last partial


@pytest.mark.gpu
@pytest.mark.parametrize("C", [16, 300])
def test_second_launch_and_long_sort(agd, ctx, C):
    from spark_agd_b200.classification import argmax_scores, naive_bayes_model
    X, y, theta, pi = design(BLOCK, D, C, seed=C)
    full, rem = divmod(ROWS, BLOCK)
    ds = agd.DeviceDataset(ctx)
    try:
        agd._native.check(agd._native.lib().agd_reserve(ds.h, 0, ROWS, D, agd._native.F32), ds.h)
        Xf = X.astype(np.float32)
        for _ in range(full):
            ds.load_dense(y, Xf, store="f32")
        ds.load_dense(y[:rem], Xf[:rem], store="f32")
        assert ds.local_rows(0) == ROWS
        mult = np.full(BLOCK, float(full))
        mult[:rem] += 1.0
        yn = y + 0.0
        labels, li = np.unique(yn, return_inverse=True)
        counts = np.bincount(li, weights=mult)
        sums = np.zeros((labels.shape[0], D))
        np.add.at(sums, li, X * mult[:, None])
        got_l, got_c, nan = ds.label_classes()
        assert same(got_l, labels) and nan == 0
        np.testing.assert_array_equal(got_c, counts)
        s, c, neg = ds.class_sums(labels)
        assert same(s, sums) and neg == 0
        np.testing.assert_array_equal(c, counts)
        m = agd.NaiveBayes.train(ds)
        pi_ref, theta_ref = naive_bayes_model(counts, sums, 1.0)
        assert same(m.pi, pi_ref) and same(m.theta, theta_ref)
        ref = argmax_scores(pi[None, :] + X @ theta.T)
        got = ds.linear_argmax(theta, pi)
        assert got.shape[0] == ROWS
        idx = np.arange(ROWS) % BLOCK
        assert np.array_equal(got, ref[idx])
        del got
        model = agd.NaiveBayesModel(label_values(C), pi, theta)
        host = agd.MulticlassMetrics(np.stack([model.labels[ref[idx]], y[idx]], axis=1))
        assert same(metric_values(agd.MulticlassMetrics(model, ds)), metric_values(host))
    finally:
        ds.close()
