"""agd_kmeans_* in a process-per-rank world (tests/kmeans_worker.py): worlds of 2 and 3 processes share one GPU over the
host-shipped CUDA IPC exchange.  Every collective call -- the step, the costs, the sampled rows, KMeans.train -- gives
identical bits on every rank.  Under the exact design the step and the costs equal the single-process run on the same rows,
and an evaluate keeps its bits across them.  (Loaded shards number their rows by rank, so views and draws, and with them the
sampled rows and the trained centres, depend on the partitioning, as views of loaded shards always have.)"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from kmeans_worker import data, run  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_kmeans_world_over_ipc(agd, ctx, tmp_path, world):
    res = run_world("kmeans_worker.py", world, str(tmp_path / "res.json"), timeout=600)
    assert len(res) == world
    for key in res[0]:
        assert all(rr[key] == res[0][key] for rr in res), key            # identical bits on every rank
    X, _ = data()
    whole = ctx.parallelize(np.zeros(X.shape[0]), X, store="f32")        # the same rows in one process
    try:
        one = run(agd, whole)
    finally:
        whole.close()
    for key in ("step", "costs"):
        assert res[0][key] == one[key], key
    assert res[0]["evaluate"] == res[0]["evaluate before"] and one["evaluate"] == one["evaluate before"]
    for mode in ("k-means||", "random"):
        assert np.all(np.isfinite(np.array(res[0]["train " + mode], dtype=np.uint64).view(np.float64)))
