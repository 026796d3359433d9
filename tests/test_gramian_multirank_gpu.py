"""agd_gramian in a process-per-rank world (tests/gramian_worker.py): worlds of 2 and 3 processes share one GPU over the
host-shipped CUDA IPC exchange.  Every rank gets identical bits, they match the whole world's reference within the bounds of
tests/test_gramian_gpu.py, dense results are bit-reproducible, and collective calls after a gramian keep their bits."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from gramian_worker import D_CSR, N_CSR, N_DENSE, csr_data, dense_data  # noqa: E402
from test_gramian_gpu import _csr_rows, check_close, check_gramian, ref_cov_bound  # noqa: E402


def _mat(rec, d):
    return np.array(rec, dtype=np.uint64).view(np.float64).reshape(d + 1, d + 1)


def _check(rec, Xs, csr):
    import spark_agd_b200 as S
    d = Xs.shape[1]
    check_gramian(_mat(rec["plain"], d), Xs)
    cov = S.linalg.covariance_from_augmented(_mat(rec["centered"], d))
    ref, tol = ref_cov_bound(Xs, csr)
    check_close(cov, ref, tol, "covariance")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_gramian_world_over_ipc(tmp_path, world):
    res = run_world("gramian_worker.py", world, str(tmp_path / "res.json"), timeout=600)
    assert len(res) == world
    for key in ("dense", "dense_view", "dense_again", "csr", "csr_view"):
        assert all(rr[key] == res[0][key] for rr in res), key                 # identical bits on every rank
    assert res[0]["dense_again"] == res[0]["dense"]                             # dense: bit-reproducible
    for r, rr in enumerate(res):
        assert rr["collectives_keep_bits"] is True, r
    X, _ = dense_data()
    X = X.astype(np.float64)
    _check(res[0]["dense"], X, False)
    m = np.concatenate([np.array(rr["dense_view_mask"], bool) for rr in res])
    assert m.shape == (N_DENSE,) and 0 < m.sum() < N_DENSE
    _check(res[0]["dense_view"], X[m], False)
    rp, ix, va, _ = csr_data()
    Xc = _csr_rows(rp, ix, va, D_CSR)
    _check(res[0]["csr"], Xc, True)
    mc = np.concatenate([np.array(rr["csr_view_mask"], bool) for rr in res])
    assert mc.shape == (N_CSR,) and 0 < mc.sum() < N_CSR
    _check(res[0]["csr_view"], Xc[mc], True)
