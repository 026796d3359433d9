"""Statistics.colStats in a process-per-rank world (tests/colstats_worker.py): worlds of 2 and 3 processes share one GPU over
the host-shipped CUDA IPC exchange.  Every rank gets identical bits, they match the whole world's reference within the
bounds of tests/test_colstats_gpu.py, and collective calls after colStats keep their bits."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from colstats_worker import FIELDS, N_CSR, N_DENSE, csr_data, dense_data, rows_of  # noqa: E402
from test_colstats_gpu import check_summary, csr_cols, dense_cols  # noqa: E402


class _Summary:
    """A summary rebuilt from the bits a rank reported (with the same derivation as MultivariateStatisticalSummary)."""

    def __init__(self, rec):
        import spark_agd_b200 as S
        a = {f: (rec[f] if f == "n" else np.array(rec[f], dtype=np.uint64).view(np.float64)) for f in FIELDS}
        s = S.MultivariateStatisticalSummary(**a)
        for f in ("count", "sum", "sum_sq", "mean", "variance", "numNonzeros", "max", "min", "normL1"):
            setattr(self, f, getattr(s, f))


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_colstats_world_over_ipc(tmp_path, world):
    res = run_world("colstats_worker.py", world, str(tmp_path / "res.json"), timeout=600)
    assert len(res) == world
    for key in ("dense", "dense_view", "dense_again", "csr", "csr_view", "csr_cols"):
        assert all(rr[key] == res[0][key] for rr in res), key                 # identical bits on every rank
    assert res[0]["dense_again"] == res[0]["dense"]                             # dense: bit-reproducible
    for r, rr in enumerate(res):
        assert rr["collectives_keep_bits"] is True, r
        assert rr["csr_untouched_zero"] is True, r
    X, _ = dense_data()
    X = X.astype(np.float64)
    check_summary(_Summary(res[0]["dense"]), dense_cols(X), N_DENSE)
    m = np.concatenate([np.array(rr["dense_view_mask"], bool) for rr in res])
    assert m.shape == (N_DENSE,) and 0 < m.sum() < N_DENSE
    check_summary(_Summary(res[0]["dense_view"]), dense_cols(X[m]), int(m.sum()))
    rp, ix, va, _ = csr_data()
    cols = np.array(res[0]["csr_cols"])
    assert np.array_equal(cols, np.unique(ix))
    allc = csr_cols(rp, ix, va, 1_000_000)
    check_summary(_Summary(res[0]["csr"]), [allc[j] for j in cols], N_CSR)
    mc = np.concatenate([np.array(rr["csr_view_mask"], bool) for rr in res])
    assert mc.shape == (N_CSR,)
    vc = csr_cols(rp, ix, va, 1_000_000, keep=mc)
    check_summary(_Summary(res[0]["csr_view"]), [vc[j] for j in cols], int(mc.sum()))
    for r in range(world):                                                     # each rank loaded its own slice
        lo, hi = rows_of(r, world, N_DENSE)
        assert len(res[r]["dense_view_mask"]) == hi - lo
