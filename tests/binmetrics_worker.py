"""One rank of a multi-process ranking-metrics world (spawned by tests/test_binmetrics_multirank_gpu.py; not a test module).

  python tests/binmetrics_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data (dense fp32 with enough distinct margins that a rank's list spans
several chunks of the exchange's bulk area, and CSR at d = 1 with heavy ties), computes the curve over the world on the
whole data and on a view, and checks that collective calls around it keep their bits.  Rank 0 also computes the same curves in
a single-process world of its own over all rows.  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N_DENSE, D_DENSE = 70001, 24
N_CSR = 4001
B = 0.125


def dense_data():
    rng = np.random.default_rng(31)
    X = rng.standard_normal((N_DENSE, D_DENSE)).astype(np.float32)
    w = rng.standard_normal(D_DENSE) * 0.3
    y = (rng.random(N_DENSE) < 0.4).astype(np.float64)
    return X, y, w


def csr_data():
    rng = np.random.default_rng(32)
    has = rng.random(N_CSR) < 0.8
    rp = np.concatenate([[0], np.cumsum(has)]).astype(np.int64)
    ix = np.zeros(int(has.sum()), dtype=np.int32)
    va = rng.integers(-3, 4, int(has.sum())).astype(np.float64)
    y = (rng.random(N_CSR) > 0.5).astype(np.float64)
    return rp, ix, va, y, np.array([1.5])


def rows_of(rank, world, n):
    return rank * n // world, (rank + 1) * n // world


def curves(dense, csr, w, wc):
    """The curves this world computes: whole dense data, a view of it, CSR."""
    out = {}
    for name, ds, ww, b in (("dense", dense, w, B), ("csr", csr, wc, -0.5)):
        s, m, tp, fp = ds.binary_curve(ww, b)
        out[name] = [s.view(np.uint64).tolist(), m.view(np.uint64).tolist(), tp.tolist(), fp.tolist()]
    va = dense.randomSplit([0.6, 0.4], seed=9)[1]
    s, m, tp, fp = va.binary_curve(w, B)
    out["view"] = [s.view(np.uint64).tolist(), m.view(np.uint64).tolist(), tp.tolist(), fp.tolist()]
    return out


def main():
    rank, world, port, dev, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import spark_agd_b200 as S
    ctx = S.Context.from_torch_distributed(dev, transport="ipc")
    X, y, w = dense_data()
    rp, ix, va, yc, wc = csr_data()
    lo, hi = rows_of(rank, world, N_DENSE)
    data = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    lc, hc = rows_of(rank, world, N_CSR)
    a, b = int(rp[lc]), int(rp[hc])
    csr = ctx.parallelize_csr(yc[lc:hc], rp[lc:hc + 1] - rp[lc], ix[a:b], va[a:b], 1, store="f64")
    res = {"curves": curves(data, csr, w, wc)}
    # collective calls after a curve give the bits they give without it
    l1, g1, _ = data.smooth(S.LogisticGradient(), w)
    e1 = list(data.evaluate(S.LogisticGradient(), w, B, 0.5).__dict__.values())
    c1 = S.Statistics.colStats(data).mean.tolist()
    data.binary_curve(w, B)
    l2, g2, _ = data.smooth(S.LogisticGradient(), w)
    data.binary_curve(w, B)
    e2 = list(data.evaluate(S.LogisticGradient(), w, B, 0.5).__dict__.values())
    data.binary_curve(w, B)
    c2 = S.Statistics.colStats(data).mean.tolist()
    res["collectives_identical"] = bool(l1 == l2 and np.array_equal(g1, g2) and e1 == e2 and c1 == c2)
    if rank == 0:   # the same rows in a world of one process
        solo = S.Context(devices=[dev])
        d1 = solo.parallelize(y, X, store="f32")
        c1s = solo.parallelize_csr(yc, rp, ix, va, 1, store="f64")
        res["single"] = curves(d1, c1s, w, wc)
        d1.close()
        c1s.close()
    data.close()
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
