"""One rank of a multi-process scoring world (spawned by tests/test_score_multirank_gpu.py; not a test module itself).

  python tests/score_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data (dense fp32 and CSR at d = 1), scores its own rows, evaluates
over the world, and runs the AGD loop on a handle that evaluated and on one that never did.  Rank 0 writes what every
rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N_DENSE, D_DENSE = 5003, 100
N_CSR = 4001
B, T = 0.375, 0.4


def dense_data():
    rng = np.random.default_rng(21)
    X = rng.standard_normal((N_DENSE, D_DENSE)).astype(np.float32)
    w = rng.standard_normal(D_DENSE) * 0.2
    y = (rng.random(N_DENSE) > 0.5).astype(np.float64)
    return X, y, w


def csr_data():
    """d = 1: every row holds its one feature or nothing (the exchange slot of a d = 1 CSR shard is the smallest)."""
    rng = np.random.default_rng(22)
    has = rng.random(N_CSR) < 0.8
    rp = np.concatenate([[0], np.cumsum(has)]).astype(np.int64)
    ix = np.zeros(int(has.sum()), dtype=np.int32)
    va = rng.standard_normal(int(has.sum()))
    y = (rng.random(N_CSR) > 0.5).astype(np.float64)
    return rp, ix, va, y, np.array([1.3])


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
    X, y, w = dense_data()
    lo, hi = rows_of(rank, world, N_DENSE)
    data = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    res["margins"] = data.margins(w, B).tolist()
    res["eval"] = {k: list(data.evaluate(g, w, B, T).__dict__.values())
                   for k, g in (("logistic", S.LogisticGradient()), ("hinge", S.HingeGradient()),
                                ("least_squares", S.LeastSquaresGradient()))}
    # collective calls around an evaluation give the bits they give without it
    l1, g1, _ = data.smooth(S.LogisticGradient(), w)
    data.evaluate(S.LogisticGradient(), w, B, T)
    l2, g2, _ = data.smooth(S.LogisticGradient(), w)
    wa, ha, _ = S.run_with_stats(data, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 6, 0.01, np.zeros(D_DENSE))
    data.evaluate(S.HingeGradient(), w, 0.0, 0.0)
    wm, hm, _ = S.run_with_stats(data, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 6, 0.01, np.zeros(D_DENSE),
                                 memoize=True)
    data.close()
    fresh = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    l3, g3, _ = fresh.smooth(S.LogisticGradient(), w)
    wb, hb, _ = S.run_with_stats(fresh, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 6, 0.01, np.zeros(D_DENSE))
    wn, hn, _ = S.run_with_stats(fresh, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 6, 0.01, np.zeros(D_DENSE),
                                 memoize=True)
    fresh.close()
    res["run_after_evaluate_identical"] = bool(
        l1 == l2 == l3 and np.array_equal(g1, g2) and np.array_equal(g1, g3) and np.array_equal(wa, wb)
        and np.array_equal(ha, hb) and np.array_equal(wm, wn) and np.array_equal(hm, hn) and len(ha) == 6)
    rp, ix, va, yc, wc = csr_data()
    lo, hi = rows_of(rank, world, N_CSR)
    a, b = int(rp[lo]), int(rp[hi])
    csr = ctx.parallelize_csr(yc[lo:hi], rp[lo:hi + 1] - rp[lo], ix[a:b], va[a:b], 1, store="f64")
    res["csr_margins"] = csr.margins(wc, B).tolist()
    res["csr_eval"] = list(csr.evaluate(S.HingeGradient(), wc, B, T).__dict__.values())
    lc1, _, _ = csr.smooth(S.HingeGradient(), wc)
    csr.evaluate(S.LogisticGradient(), wc, B, T)
    lc2, _, _ = csr.smooth(S.HingeGradient(), wc)
    res["csr_smooth"] = [lc1, lc2]          # the CSR gradient kernel scatters with RED.ADD: equal to rounding, not in bits
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
