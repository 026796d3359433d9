"""One rank of a multi-process NaiveBayes world (spawned by tests/test_naive_bayes_multirank_gpu.py; not a test module).

  python tests/naive_bayes_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its slice of the exact design (dense fp32, d = 23): in a world of 3, rank 1 holds no rows, and a label that
only the last rows carry lives on the last rank alone.  Each rank then runs, collectively: label_classes, class_sums,
NaiveBayes.train, MulticlassMetrics of a hand-built model and of the trained one, and an evaluate before and after them.  Rank 0
writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

N_ROWS, D, C = 2501, 23, 9
LONE_LABEL = 99.25


def data():
    from test_naive_bayes_gpu import design
    X, y, theta, pi = design(N_ROWS, D, C, seed=77)
    y[-5:] = LONE_LABEL
    return X.astype(np.float32), y, theta, pi


def rows_of(rank, world, n):
    if world == 3:   # rank 1 holds no rows
        return [(0, n // 2), (n // 2, n // 2), (n // 2, n)][rank]
    return rank * n // world, (rank + 1) * n // world


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel().tolist()


def run(S, ds):
    from test_naive_bayes_gpu import metric_values
    _, _, theta, pi = data()
    w = np.linspace(-1, 1, D)
    res = {"evaluate before": _bits(list(ds.evaluate(S.LeastSquaresGradient(), w, 0.5).__dict__.values()))}
    labels, counts, nan = ds.label_classes()
    res["classes"] = _bits(np.concatenate([labels, counts, [nan]]))
    s, c, neg = ds.class_sums(labels)
    res["sums"] = _bits(np.concatenate([s.ravel(), c, [neg]]))
    m = S.NaiveBayes.train(ds, lambda_=0.5)
    res["model"] = _bits(np.concatenate([m.labels, m.pi, m.theta.ravel()]))
    hand = S.NaiveBayesModel(np.append(np.arange(C - 1) * 0.75 - 3.0, LONE_LABEL), pi, theta)
    res["metrics hand"] = _bits(metric_values(S.MulticlassMetrics(hand, ds)))
    res["metrics trained"] = _bits(metric_values(S.MulticlassMetrics(m, ds)))
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
    X, y, _, _ = data()
    lo, hi = rows_of(rank, world, N_ROWS)
    ds = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
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
