"""Scoring in a process-per-rank world (tests/score_worker.py): worlds of 2 and 3 processes share one GPU over the
host-shipped CUDA IPC exchange.  Margins are rank-local; agd_evaluate reduces over the world and gives every rank the same
bits; collective calls around an evaluation keep their bits."""
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from rank_world import run_world  # noqa: E402
from k1_reference import row_terms  # noqa: E402
from score_worker import B, N_CSR, N_DENSE, T, csr_data, dense_data, rows_of  # noqa: E402

U = 2.0 ** -53


def _sums(kind, m, y, t):
    _, loss = row_terms(kind, m, y)
    pos = (1.0 / (1.0 + np.exp(-m)) > t) if kind == "logistic" else (m > t)
    cnt = np.ones_like(m) if kind in ("logistic", "hinge") else np.zeros_like(m)
    one = y == 1.0
    e = m - y
    terms = [np.ones_like(m), loss, cnt * (pos & one), cnt * (pos & ~one), cnt * (~pos & ~one), cnt * (~pos & one),
             e, e * e, np.abs(e), y, y * y]
    return [(math.fsum(tm.astype(np.float64)), float(np.sum(np.abs(tm)))) for tm in terms]


def _check_sums(got, ref):
    for k, (g, (r, mag)) in enumerate(zip(got, ref)):
        if k in (0, 2, 3, 4, 5):
            assert g == r, (k, g, r)
        else:
            assert abs(g - r) <= 1e-12 * mag, (k, g, r, mag)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_score_world_over_ipc(tmp_path, world):
    res = run_world("score_worker.py", world, str(tmp_path / "res.json"))
    assert len(res) == world
    X, y, w = dense_data()
    X = X.astype(np.float64)
    m_all = np.array([math.fsum(list(X[i] * w) + [B]) for i in range(N_DENSE)])
    rp, ix, va, yc, wc = csr_data()
    mc_all = np.array([math.fsum(list(va[rp[i]:rp[i + 1]] * wc[0]) + [B]) for i in range(N_CSR)])
    for r, rr in enumerate(res):
        lo, hi = rows_of(r, world, N_DENSE)
        m = np.array(rr["margins"])
        scale = np.abs(X[lo:hi]) @ np.abs(w) + abs(B)
        assert m.shape == (hi - lo,)
        assert np.all(np.abs(m - m_all[lo:hi]) <= (X.shape[1] + 2) * U * scale), r
        lo, hi = rows_of(r, world, N_CSR)
        mc = np.array(rr["csr_margins"])
        assert mc.shape == (hi - lo,)
        assert np.all(np.abs(mc - mc_all[lo:hi]) <= 3 * U * (np.abs(mc_all[lo:hi] - B) + abs(B))), r
        assert rr["run_after_evaluate_identical"] is True, r
        lc1, lc2 = rr["csr_smooth"]
        assert abs(lc1 - lc2) <= 1e-13 * abs(lc1), r
    # identical bits on every rank, equal to the numpy sum over the whole world
    for kind in ("logistic", "hinge", "least_squares"):
        got = [rr["eval"][kind] for rr in res]
        assert all(g == got[0] for g in got), kind
        _check_sums(got[0], _sums(kind, m_all, y, T))
    got = [rr["csr_eval"] for rr in res]
    assert all(g == got[0] for g in got)
    _check_sums(got[0], _sums("hinge", mc_all, yc, T))
