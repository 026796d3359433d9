"""NaiveBayes and MulticlassMetrics in a process-per-rank world (tests/naive_bayes_worker.py): worlds of 2 and 3 processes
share one GPU over the host-shipped CUDA IPC exchange.  Every collective call -- the distinct labels, the class sums, the
trained model and both metrics -- gives identical bits on every rank, equal to the single-process run on the same rows, with a
label present on one rank only and, in the world of 3, a rank that holds no rows.  An evaluate keeps its bits across them (its sums depend on the partitioning, so it is compared
within a world only)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from naive_bayes_worker import LONE_LABEL, data, run  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_naive_bayes_world_over_ipc(agd, ctx, tmp_path, world):
    res = run_world("naive_bayes_worker.py", world, str(tmp_path / "res.json"), timeout=600)
    assert len(res) == world
    for key in res[0]:
        assert all(rr[key] == res[0][key] for rr in res), key            # identical bits on every rank
    X, y, _, _ = data()
    whole = ctx.parallelize(y, X, store="f32")                           # the same rows in one process
    try:
        one = run(agd, whole)
    finally:
        whole.close()
    for key in ("classes", "sums", "model", "metrics hand", "metrics trained"):
        assert res[0][key] == one[key], key
    assert res[0]["evaluate"] == res[0]["evaluate before"]
    labels = np.array(res[0]["classes"], dtype=np.uint64).view(np.float64)
    assert LONE_LABEL in labels
