"""agd_project in a process-per-rank world (tests/project_worker.py): worlds of 2 and 3 processes share one GPU over the
host-shipped CUDA IPC exchange.  Each rank's projected rows equal, bit for bit, the single-process projection of the same
rows (the bits of a row depend only on the row), computeSVD gives identical bits on every rank, and collective calls on the
projected dataset run over the new handle's own exchange and agree on every rank."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from project_worker import K, N_ROWS, data, rows_of  # noqa: E402


def _f64(rec):
    return np.array(rec, dtype=np.uint64).view(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_project_world_over_ipc(agd, ctx, tmp_path, world):
    res = run_world("project_worker.py", world, str(tmp_path / "res.json"), timeout=600)
    assert len(res) == world
    for key in ("evaluate", "colstats", "svd_s", "svd_V", "svd_UtU"):
        assert all(rr[key] == res[0][key] for rr in res), key               # identical bits on every rank
    X, y, B, c = data()
    whole = ctx.parallelize(y, X, store="f32")                               # the same rows in one process
    try:
        p = whole.project(B, c)
        try:
            Y = p.get_rows(0, 0, N_ROWS, dtype=np.float64)[0]
            ev = p.evaluate(agd.LeastSquaresGradient(), np.linspace(-1, 1, K), 0.5)
            assert ev.count == N_ROWS
            assert _f64(res[0]["evaluate"])[0] == N_ROWS
        finally:
            p.close()
        svd = agd.RowMatrix(whole).computeSVD(6)
    finally:
        whole.close()
    for r, rr in enumerate(res):
        lo, hi = rows_of(r, world, N_ROWS)
        assert np.array_equal(_f64(rr["rows"]).view(np.uint64), Y[lo:hi].ravel().view(np.uint64)), r
        assert np.array_equal(_f64(rr["labels"]), y[lo:hi]), r
        m = np.array(rr["view_mask"], bool)
        assert np.array_equal(_f64(rr["view_rows"]).view(np.uint64), Y[lo:hi][m].ravel().view(np.uint64)), r
    np.testing.assert_allclose(_f64(res[0]["svd_s"]), svd.s, rtol=1e-10)
    G = _f64(res[0]["svd_UtU"]).reshape(6, 6)
    s = _f64(res[0]["svd_s"])
    assert np.abs(G - np.eye(6)).max() <= 64 * (N_ROWS + 300) * 2.0 ** -53 * (s[0] / s[-1]) ** 2
