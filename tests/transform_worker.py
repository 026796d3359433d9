"""One rank of a multi-process world training on a transformed view (spawned by tests/test_transform_multirank_gpu.py; not a
test module itself).

  python tests/transform_worker.py RANK WORLD PORT DEVICE OUT.json

Every rank loads its contiguous slice of seeded host data, scales it with a scaler fitted on the device (colStats over the
world), appends the bias column and runs smooth / smooth_two / run on a row view of that; a wide CSR shard takes the
reduce-scatter form of the exchange.  Rank 0 writes what every rank reported."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N, D = 4003, 512                      # d = 512 fp32: a ring shape with the two-gradient sweep
WIDE_N, WIDE_D = 601, 40000          # D + 5 > 32768 doubles: the reduce-scatter exchange
SPLIT_SEED = 77


def host_data():
    rng = np.random.default_rng(41)
    X = (rng.standard_normal((N, D)) * rng.uniform(0.5, 5.0, D) + 1.0).astype(np.float32)
    w = rng.standard_normal(D + 1) * 0.1
    y = (rng.random(N) > 0.5).astype(np.float64)
    return X, y, w


def wide_data():
    rng = np.random.default_rng(43)
    rowptr = np.arange(WIDE_N + 1, dtype=np.int64) * 16
    idx = np.sort(rng.integers(0, WIDE_D, size=(WIDE_N, 16)), axis=1).astype(np.int32).ravel()
    val = rng.standard_normal(WIDE_N * 16)
    y = (rng.random(WIDE_N) > 0.5).astype(np.float64)
    return rowptr, idx, val, y


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
    scaler = S.StandardScaler().fit(data)
    train = S.MLUtils.appendBias(scaler.transform(data)).randomSplit([0.7, 0.3], seed=SPLIT_SEED)[0]
    l, g, c = train.smooth(grad, w)
    l_, g_, c_, l2, g2 = train.smooth_two(grad, w, 0.5 * w)
    w0 = np.zeros(D + 1)
    w0[-1] = 1.0
    wr, hr, sr = S.run_with_stats(train, grad, upd, 0.0, 5, 0.01, w0)
    wm, hm, _ = S.run_with_stats(train, grad, upd, 0.0, 5, 0.01, w0, memoize=True)
    res["std"] = scaler.std.tolist()
    res["smooth"] = {"loss": l, "grad": g.tolist(), "count": c, "two": [l_, g_.tolist(), c_, l2, g2.tolist()],
                     "mask": train.row_mask(0, 0, hi - lo).tolist()}
    res["run"] = {"w": wr.tolist(), "hist": hr.tolist(), "passes": sr.passes,
                  "memo_identical": bool(np.array_equal(wr, wm) and np.array_equal(hr, hm))}
    data.close()
    rowptr, idx, val, yw = wide_data()
    a, b = rows_of(rank, world, WIDE_N)
    wide = ctx.parallelize_csr(yw[a:b], rowptr[a:b + 1] - rowptr[a], idx[rowptr[a]:rowptr[b]], val[rowptr[a]:rowptr[b]],
                               WIDE_D, store="f64")
    s = np.linspace(0.5, 2.0, WIDE_D)
    ww = np.random.default_rng(44).standard_normal(WIDE_D + 1) * 0.1
    lw, gw, cw = S.MLUtils.appendBias(S.StandardScalerModel(1.0 / s).transform(wide)).smooth(grad, ww)
    res["wide"] = {"loss": lw, "grad": gw.tolist(), "count": cw}
    wide.close()
    everyone = [None] * world
    dist.all_gather_object(everyone, res)
    if rank == 0:
        with open(out, "w") as f:
            json.dump(everyone, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
