"""Views in a process-per-rank world (tests/view_worker.py): worlds of 2 and 3 processes share one GPU over the host-shipped
CUDA IPC exchange.  A view's smooth, run and evaluate give the same bits on every rank; on a generated shard the view selects
the rows a 1-rank world selects and the run matches the oracle on them; collective calls after view calls keep their bits."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from view_reference import view_mask  # noqa: E402
from view_worker import GEN_D, GEN_ROWS, GEN_SEED, SPLIT_SEED  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_views_world_over_ipc(tmp_path, oracle, world):
    res = run_world("view_worker.py", world, str(tmp_path / "res.json"))
    assert len(res) == world
    for key in ("loss", "grad", "count", "w", "hist", "eval"):
        assert all(rr["view"][key] == res[0]["view"][key] for rr in res), key
    for r, rr in enumerate(res):
        assert rr["after_identical"] is True, r
        assert rr["view"]["memo_identical"] is True, r
        # loaded shards: rank r's rows are numbered r << 40
        n = len(rr["view"]["mask"])
        assert rr["view"]["mask"] == view_mask(((SPLIT_SEED, 0.0, 0.7, False),), r << 40, n).tolist()
    assert res[0]["view"]["count"] == sum(sum(rr["view"]["mask"]) for rr in res)
    # generated shard: global row numbering, so the selected rows do not depend on the world size
    sel = np.concatenate([np.array(rr["gen"]["mask"], bool) for rr in res])
    assert sel.tolist() == view_mask(((SPLIT_SEED, 0.0, 0.6, False),), 0, GEN_ROWS).tolist()
    assert all(rr["gen"]["w"] == res[0]["gen"]["w"] and rr["gen"]["hist"] == res[0]["gen"]["hist"] for rr in res)
    X = oracle.synth_dense_f32(GEN_SEED, 0, GEN_ROWS, GEN_D)
    y = oracle.synth_labels(GEN_SEED, "logistic", 0, X, oracle.synth_wtrue(GEN_SEED, GEN_D))
    ref = oracle.agd_run(oracle.Data(y[sel], X=X[sel]), "logistic", "squared_l2", np.zeros(GEN_D), convergence_tol=0.0,
                         num_iterations=5, reg_param=0.01, partitions=world)
    np.testing.assert_allclose(res[0]["gen"]["hist"], ref.loss_history, rtol=1e-9)
    w = np.array(res[0]["gen"]["w"])
    assert np.linalg.norm(w - ref.weights) <= 1e-9 * np.linalg.norm(ref.weights)
    assert res[0]["gen"]["passes"] == ref.passes
