"""Ranking metrics in a process-per-rank world (tests/binmetrics_worker.py): worlds of 2 and 3 processes share one GPU over the
host-shipped CUDA IPC exchange.  Every rank gets the same bits, and on the whole data they equal a single-process run over the
same rows; the
dense lists span several chunks of the exchange's bulk area.  Collective calls after a curve keep their bits."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
import binmetrics_reference as R  # noqa: E402
from binmetrics_worker import B, dense_data  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_binary_curve_world_over_ipc(tmp_path, world):
    res = run_world("binmetrics_worker.py", world, str(tmp_path / "res.json"), timeout=600)
    assert len(res) == world
    for r in range(world):
        assert res[r]["curves"] == res[0]["curves"], r
        assert res[r]["collectives_identical"], r
    # a view of loaded shards numbers its rows by rank (agd_set_row_filter), so only the whole data is partitioning-free
    for name in ("dense", "csr"):
        assert res[0]["curves"][name] == res[0]["single"][name], name
    dense = res[0]["curves"]["dense"]
    assert 3 * len(dense[1]) // world > 65536          # a rank's list takes more than one bulk epoch
    # and the curve is the reference's, from fp64 margins of the same fp32 rows
    X, y, w = dense_data()
    m = X.astype(np.float64) @ w + B
    rm, rtp, rfp, _ = R.curve(m, y)
    assert len(dense[1]) == len(rm)
    assert dense[2] == rtp.tolist() and dense[3] == rfp.tolist()
    got = np.array(dense[1], dtype=np.uint64).view(np.float64)
    assert np.max(np.abs(got - rm)) < 1e-12 * np.max(np.abs(rm))
