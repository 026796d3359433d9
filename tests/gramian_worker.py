"""One rank of a multi-process cross-products world (spawned by tests/test_gramian_multirank_gpu.py; not a test module).

  python tests/gramian_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data -- dense fp32 at d = 300 (the packed sums, about 45 000 doubles,
cross ranks in several epochs of the one-shot exchange) and CSR fp64 at d = 200 -- and runs agd_gramian (both forms) on the
whole data and on a view, with collective calls around it.  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N_DENSE, D_DENSE = 3001, 300
N_CSR, D_CSR, K_CSR = 2003, 200, 24


def dense_data():
    rng = np.random.default_rng(41)
    X = rng.standard_normal((N_DENSE, D_DENSE)) * 2.0 + np.linspace(-5, 5, D_DENSE)
    X[rng.random(X.shape) < 0.1] = 0.0
    return X.astype(np.float32), (rng.random(N_DENSE) > 0.5).astype(np.float64)


def csr_data():
    rng = np.random.default_rng(42)
    nnz = rng.integers(0, K_CSR + 1, size=N_CSR)
    parts = [np.sort(rng.choice(D_CSR, k, replace=False)) for k in nnz]
    rp = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    ix = np.concatenate(parts).astype(np.int32)
    va = rng.standard_normal(ix.shape[0]) - 0.5
    va[::11] = 0.0
    return rp, ix, va, (rng.random(N_CSR) > 0.5).astype(np.float64)


def rows_of(rank, world, n):
    return rank * n // world, (rank + 1) * n // world


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel().tolist()


def _both(ds):
    return {"plain": _bits(ds.gramian(False)[1]), "centered": _bits(ds.gramian(True)[1])}


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
    res["dense"] = _both(data)
    view = data.sample(False, 0.3, seed=4)
    res["dense_view"] = _both(view)
    res["dense_view_mask"] = view.row_mask(0, 0, hi - lo).tolist()
    res["dense_again"] = _both(data)
    l2, g2, _ = data.smooth(S.LogisticGradient(), w)
    e2 = list(data.evaluate(S.LogisticGradient(), w).__dict__.values())
    res["collectives_keep_bits"] = bool(l1 == l2 and np.array_equal(g1, g2) and e1 == e2)
    data.close()
    rp, ix, va, yc = csr_data()
    lo, hi = rows_of(rank, world, N_CSR)
    a, b = int(rp[lo]), int(rp[hi])
    csr = ctx.parallelize_csr(yc[lo:hi], rp[lo:hi + 1] - rp[lo], ix[a:b], va[a:b], D_CSR, store="f64")
    res["csr"] = _both(csr)
    cv = csr.sample(False, 0.5, seed=8)
    res["csr_view"] = _both(cv)
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
