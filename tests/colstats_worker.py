"""One rank of a multi-process column-statistics world (spawned by tests/test_colstats_multirank_gpu.py; not a test module).

  python tests/colstats_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data -- dense fp32 at d = 100 (pass-1 sums in three epochs of the
one-shot exchange) and CSR at d = 10^6 (several reduce-scatter epochs) -- and runs Statistics.colStats on the whole data
and on a view, with collective calls around it.  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N_DENSE, D_DENSE = 4003, 100
N_CSR, D_CSR, K_CSR = 3001, 1_000_000, 12
FIELDS = ("n", "sum", "sum_sq", "sum_abs", "nnz", "dev", "dev2", "col_max", "col_min")


def dense_data():
    rng = np.random.default_rng(31)
    X = rng.standard_normal((N_DENSE, D_DENSE)) * 2.0 + np.linspace(-5, 5, D_DENSE)
    X[rng.random(X.shape) < 0.1] = 0.0
    return X.astype(np.float32), (rng.random(N_DENSE) > 0.5).astype(np.float64)


def csr_data():
    rng = np.random.default_rng(32)
    nnz = rng.integers(0, K_CSR + 1, size=N_CSR)
    hot = rng.choice(D_CSR, 40, replace=False)                 # most entries land on a few columns, the rest anywhere

    def row(k):   # sorted distinct column ids (duplicates drawn are merged, so a row may hold fewer than k)
        return np.unique(np.where(rng.random(k) < 0.7, rng.choice(hot, k), rng.integers(0, D_CSR, k)))

    parts = [row(k) for k in nnz]
    nnz = np.array([p.shape[0] for p in parts])
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate(parts).astype(np.int32)
    va = rng.standard_normal(ix.shape[0]) - 0.5
    va[::11] = 0.0
    return rp, ix, va, (rng.random(N_CSR) > 0.5).astype(np.float64)


def rows_of(rank, world, n):
    return rank * n // world, (rank + 1) * n // world


def _summary(st):
    return {f: (float(getattr(st, f)) if f == "n" else np.asarray(getattr(st, f)).view(np.uint64).tolist()) for f in FIELDS}


def main():
    rank, world, port, dev, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import spark_agd_b200 as S
    ctx = S.Context.from_torch_distributed(dev, transport="ipc")
    res = {}
    X, y = dense_data()
    lo, hi = rows_of(rank, world, N_DENSE)
    data = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    w = np.linspace(-0.1, 0.1, D_DENSE)
    l1, g1, _ = data.smooth(S.LogisticGradient(), w)
    e1 = list(data.evaluate(S.LogisticGradient(), w).__dict__.values())
    res["dense"] = _summary(S.Statistics.colStats(data))
    view = data.sample(False, 0.3, seed=4)
    res["dense_view"] = _summary(S.Statistics.colStats(view))
    res["dense_view_mask"] = view.row_mask(0, 0, hi - lo).tolist()
    res["dense_again"] = _summary(S.Statistics.colStats(data))
    l2, g2, _ = data.smooth(S.LogisticGradient(), w)
    e2 = list(data.evaluate(S.LogisticGradient(), w).__dict__.values())
    res["collectives_keep_bits"] = bool(l1 == l2 and np.array_equal(g1, g2) and e1 == e2)
    data.close()
    rp, ix, va, yc = csr_data()
    lo, hi = rows_of(rank, world, N_CSR)
    a, b = int(rp[lo]), int(rp[hi])
    csr = ctx.parallelize_csr(yc[lo:hi], rp[lo:hi + 1] - rp[lo], ix[a:b], va[a:b], D_CSR, store="f64")
    st = S.Statistics.colStats(csr)
    cols = np.unique(ix)
    res["csr_cols"] = cols.tolist()
    res["csr"] = {f: (float(st.n) if f == "n" else np.asarray(getattr(st, f))[cols].view(np.uint64).tolist()) for f in FIELDS}
    others = np.setdiff1d(np.arange(0, D_CSR, 997), cols)
    res["csr_untouched_zero"] = bool(np.all(st.sum[others] == 0) and np.all(st.col_max[others] == 0)
                                     and np.all(st.col_min[others] == 0) and np.all(st.nnz[others] == 0)
                                     and np.all(st.variance[others] == 0))
    cv = csr.sample(False, 0.5, seed=8)
    sv = S.Statistics.colStats(cv)
    res["csr_view"] = {f: (float(sv.n) if f == "n" else np.asarray(getattr(sv, f))[cols].view(np.uint64).tolist()) for f in FIELDS}
    res["csr_view_mask"] = cv.row_mask(0, 0, hi - lo).tolist()
    csr.close()
    everyone = [None] * world
    dist.all_gather_object(everyone, res)
    if rank == 0:
        with open(out, "w") as f:
            json.dump(everyone, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
