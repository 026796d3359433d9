"""One rank of a multi-process projection world (spawned by tests/test_project_multirank_gpu.py; not a test module).

  python tests/project_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data (dense fp32 at d = 300), projects it and a view of it with the
same B and offset (rank-local), runs computeSVD with U (collective), and evaluate and colStats on the projected dataset (the
new handle's own exchange).  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N_ROWS, D, K = 3001, 300, 40


def data():
    rng = np.random.default_rng(51)
    X = rng.standard_normal((N_ROWS, D)) * 2.0 + np.linspace(-5, 5, D)
    X[rng.random(X.shape) < 0.1] = 0.0
    B = rng.standard_normal((D, K)) / np.sqrt(D)
    return X.astype(np.float32), (rng.random(N_ROWS) > 0.5).astype(np.float64), B, rng.standard_normal(K)


def rows_of(rank, world, n):
    return rank * n // world, (rank + 1) * n // world


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel().tolist()


def main():
    rank, world, port, dev, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import spark_agd_b200 as S
    ctx = S.Context.from_torch_distributed(dev, transport="ipc")
    X, y, B, c = data()
    lo, hi = rows_of(rank, world, N_ROWS)
    src = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    res = {}
    p = src.project(B, c)
    Y, yl = p.get_rows(0, 0, p.local_rows(0), dtype=np.float64)
    res["rows"], res["labels"] = _bits(Y), _bits(yl)
    ev = p.evaluate(S.LeastSquaresGradient(), np.linspace(-1, 1, K), 0.5)
    res["evaluate"] = _bits(list(ev.__dict__.values()))
    cs = S.Statistics.colStats(p)
    res["colstats"] = _bits(np.concatenate([cs.mean, cs.variance, [cs.count]]))
    p.close()
    view = src.sample(False, 0.4, seed=6)
    res["view_mask"] = view.row_mask(0, 0, hi - lo).tolist()
    pv = view.project(B, c)
    res["view_rows"] = _bits(pv.get_rows(0, 0, pv.local_rows(0), dtype=np.float64)[0])
    pv.close()
    svd = S.RowMatrix(src).computeSVD(6, computeU=True)
    res["svd_s"], res["svd_V"] = _bits(svd.s), _bits(svd.V)
    Ud = svd.U.data
    res["svd_U"] = _bits(Ud.get_rows(0, 0, Ud.local_rows(0), dtype=np.float64)[0])
    res["svd_UtU"] = _bits(S.RowMatrix(Ud).computeGramianMatrix())
    Ud.close()
    src.close()
    everyone = [None] * world
    dist.all_gather_object(everyone, res)
    if rank == 0:
        with open(out, "w") as f:
            json.dump(everyone, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
