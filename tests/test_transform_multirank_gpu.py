"""Feature transforms in a process-per-rank world (tests/transform_worker.py): worlds of 2 and 3 processes share one GPU over
the host-shipped CUDA IPC exchange.  The scaler fitted on the device, the transformed smooth, two-gradient sweep and run give
the same bits on every rank, also when the payload takes the reduce-scatter exchange, and they match the references."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
import k1_reference as R  # noqa: E402
from transform_worker import D, SPLIT_SEED, WIDE_D, host_data, rows_of, wide_data  # noqa: E402
from view_reference import view_mask  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_transform_world_over_ipc(tmp_path, oracle, world):
    res = run_world("transform_worker.py", world, str(tmp_path / "res.json"))
    assert len(res) == world
    for r, rr in enumerate(res):
        assert rr["std"] == res[0]["std"], r
        for key in ("loss", "grad", "count", "two"):
            assert rr["smooth"][key] == res[0]["smooth"][key], (r, key)
        for key in ("w", "hist", "passes"):
            assert rr["run"][key] == res[0]["run"][key], (r, key)
        assert rr["run"]["memo_identical"] is True, r
        assert rr["wide"] == res[0]["wide"], r
    X, y, w = host_data()
    std = np.array(res[0]["std"])
    np.testing.assert_allclose(std, np.sqrt(X.astype(np.float64).var(axis=0, ddof=1)), rtol=1e-12)
    s = np.where(std != 0, 1.0 / np.where(std != 0, std, 1.0), 0.0)
    mask = np.concatenate([np.array(rr["smooth"]["mask"], bool) for rr in res])
    for r in range(world):   # rank r's rows are numbered r << 40
        lo, hi = rows_of(r, world, len(y))
        assert mask[lo:hi].tolist() == view_mask(((SPLIT_SEED, 0.0, 0.7, False),), r << 40, hi - lo).tolist()
    Xp = np.concatenate([X.astype(np.float64) * s, np.ones((len(y), 1))], axis=1)[mask]
    lref, cref, gref = R.fold_shard("logistic", y[mask], w, X=Xp)
    sm = res[0]["smooth"]
    assert sm["count"] == cref
    assert abs(sm["loss"] - lref / cref) <= 1e-12 * abs(lref / cref)
    np.testing.assert_allclose(sm["grad"], gref / cref, rtol=0, atol=1e-12 * np.max(np.abs(gref / cref)))
    ref = oracle.agd_run(oracle.Data(y[mask], X=Xp), "logistic", "squared_l2", np.append(np.zeros(D), 1.0),
                         convergence_tol=0.0, num_iterations=5, reg_param=0.01, partitions=world)
    np.testing.assert_allclose(res[0]["run"]["hist"], ref.loss_history, rtol=1e-9)
    wr = np.array(res[0]["run"]["w"])
    assert np.linalg.norm(wr - ref.weights) <= 1e-9 * np.linalg.norm(ref.weights)
    assert res[0]["run"]["passes"] == ref.passes
    rowptr, idx, val, yw = wide_data()
    sw = np.linspace(0.5, 2.0, WIDE_D)
    sw = 1.0 / (1.0 / sw)                                   # the factor the worker's StandardScalerModel(1 / s) applies
    ww = np.random.default_rng(44).standard_normal(WIDE_D + 1) * 0.1
    n = len(yw)
    rp = rowptr + np.arange(n + 1)                          # one more entry per row: the bias column
    ni = np.insert(idx, rowptr[1:], WIDE_D).astype(np.int32)
    nv = np.insert(val * sw[idx], rowptr[1:], 1.0)
    lw, cw, gw = R.fold_shard("logistic", yw, ww, csr=(rp, ni, nv))
    wd = res[0]["wide"]
    assert wd["count"] == cw
    assert abs(wd["loss"] - lw / cw) <= 1e-12 * abs(lw / cw)
    np.testing.assert_allclose(wd["grad"], gw / cw, rtol=0, atol=1e-12 * np.max(np.abs(gw / cw)))
