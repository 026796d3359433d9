"""One rank of a multi-process world running on views (spawned by tests/test_views_multirank_gpu.py; not a test module itself).

  python tests/view_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data and runs smooth / run / evaluate on a view of it; it also generates a
synthetic shard in place and trains on a view of that.  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N, D = 4003, 96
GEN_ROWS, GEN_D, GEN_SEED = 3001, 128, 42
SPLIT_SEED = 77


def host_data():
    rng = np.random.default_rng(31)
    X = rng.standard_normal((N, D)).astype(np.float32)
    w = rng.standard_normal(D) * 0.2
    y = (rng.random(N) > 0.5).astype(np.float64)
    return X, y, w


def rows_of(rank, world, n):
    return rank * n // world, (rank + 1) * n // world


def main():
    rank, world, port, dev, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import spark_agd_b200 as S
    ctx = S.Context.from_torch_distributed(dev, transport="ipc")
    res = {}
    X, y, w = host_data()
    lo, hi = rows_of(rank, world, N)
    data = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    grad, upd = S.LogisticGradient(), S.SquaredL2Updater()
    l0, g0, _ = data.smooth(grad, w)
    w0, h0, _ = S.run_with_stats(data, grad, upd, 0.0, 5, 0.01, np.zeros(D))
    train, test = data.randomSplit([0.7, 0.3], seed=SPLIT_SEED)
    lv, gv, cv = train.smooth(grad, w)
    wv, hv, _ = S.run_with_stats(train, grad, upd, 0.0, 5, 0.01, np.zeros(D))
    wvm, hvm, _ = S.run_with_stats(train, grad, upd, 0.0, 5, 0.01, np.zeros(D), memoize=True)
    ev = test.evaluate(grad, wv)
    res["view"] = {"loss": lv, "grad": gv.tolist(), "count": cv, "w": wv.tolist(), "hist": hv.tolist(),
                   "memo_identical": bool(np.array_equal(wv, wvm) and np.array_equal(hv, hvm)),
                   "eval": list(ev.__dict__.values()), "mask": train.row_mask(0, 0, hi - lo).tolist()}
    # collective calls after view calls give the bits they give without them
    l1, g1, _ = data.smooth(grad, w)
    w1, h1, _ = S.run_with_stats(data, grad, upd, 0.0, 5, 0.01, np.zeros(D))
    res["after_identical"] = bool(l0 == l1 and np.array_equal(g0, g1) and np.array_equal(w0, w1) and np.array_equal(h0, h1))
    data.close()
    # a generated shard: the view selects the same global rows as in a 1-rank world
    gen = ctx.synthetic(GEN_ROWS, GEN_D, grad, seed=GEN_SEED, store="f32")
    gv_train = gen.sample(False, 0.6, seed=SPLIT_SEED)
    wg, hg, sg = S.run_with_stats(gv_train, grad, upd, 0.0, 5, 0.01, np.zeros(GEN_D))
    glo, ghi = rows_of(rank, world, GEN_ROWS)
    res["gen"] = {"w": wg.tolist(), "hist": hg.tolist(), "passes": sg.passes, "lo": glo,
                  "mask": gv_train.row_mask(0, 0, ghi - glo).tolist()}
    gen.close()
    everyone = [None] * world
    dist.all_gather_object(everyone, res)
    if rank == 0:
        with open(out, "w") as f:
            json.dump(everyone, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
