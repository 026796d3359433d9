"""One rank of a multi-process k-means world (spawned by tests/test_kmeans_multirank_gpu.py; not a test module).

  python tests/kmeans_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of the exact design (dense fp32, d = 23) and runs, collectively: a step, the k-means||
cost update and weighted sample, an unweighted sample of a view, KMeans.train in both initialisation modes, and an evaluate
before and after them.  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

N_ROWS, D, K = 2501, 23, 9


def data():
    from test_kmeans_gpu import design
    X, C = design(N_ROWS, D, K, seed=77)
    return X.astype(np.float32), C


def rows_of(rank, world, n):
    return rank * n // world, (rank + 1) * n // world


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel().tolist()


def run(S, ds):
    X, C = data()
    w = np.linspace(-1, 1, D)
    res = {"evaluate before": _bits(list(ds.evaluate(S.LeastSquaresGradient(), w, 0.5).__dict__.values()))}
    s, c, cost = ds.kmeans_step(C)
    res["step"] = _bits(np.concatenate([s.ravel(), c, [cost]]))
    total = ds.kmeans_costs(C[:3], keep=False)
    total2 = ds.kmeans_costs(C[3:5], keep=True)
    rows, draws = ds.kmeans_sample(5, 4.0 * K / total2, weighted=True)
    res["costs"] = _bits([total, total2])
    res["sample"] = _bits(np.concatenate([rows.ravel(), draws]))
    v = ds.sample(False, 0.5, seed=3)
    rows, draws = v.kmeans_sample(8, 0.1, weighted=False)
    res["view_sample"] = _bits(np.concatenate([rows.ravel(), draws]))
    for mode in ("k-means||", "random"):
        m = S.KMeans.train(ds, K, 10, initializationMode=mode, seed=19)
        res["train " + mode] = _bits(m.clusterCenters)
    res["evaluate"] = _bits(list(ds.evaluate(S.LeastSquaresGradient(), w, 0.5).__dict__.values()))
    return res


def main():
    rank, world, port, dev, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import spark_agd_b200 as S
    ctx = S.Context.from_torch_distributed(dev, transport="ipc")
    X, _ = data()
    lo, hi = rows_of(rank, world, N_ROWS)
    ds = ctx.parallelize(np.zeros(hi - lo), X[lo:hi], store="f32")
    res = run(S, ds)
    ds.close()
    everyone = [None] * world
    dist.all_gather_object(everyone, res)
    if rank == 0:
        with open(out, "w") as f:
            json.dump(everyone, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
