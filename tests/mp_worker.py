"""One rank of a multi-process world (spawned by tests/test_multirank_gpu.py; not a test module itself).

  python tests/mp_worker.py RANK WORLD PORT DEVICE TRANSPORT OUT.json

Every rank loads its contiguous slice of a seeded host dataset (and, second, generates its slice of the synthetic
workload in place), runs applySmooth and the AGD loop through the C-ABI mirror, and rank 0 writes the results."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def make_data(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    w_true = rng.standard_normal(d) / np.sqrt(d)
    y = (X.astype(np.float64) @ w_true + rng.logistic(size=n) > 0).astype(np.float64)
    return X, y


def make_csr(n, d, k, seed):
    """n rows with k stored entries each (strictly increasing columns), hinge-style labels."""
    rng = np.random.default_rng(seed)
    idx = np.sort(np.stack([rng.choice(d, k, replace=False) for _ in range(512)]), axis=1).astype(np.int32)
    idx = idx[rng.integers(0, 512, size=n)]
    val = rng.standard_normal((n, k)).astype(np.float32)
    w_true = rng.standard_normal(d)
    y = (np.einsum("ij,ij->i", val.astype(np.float64), w_true[idx]) + 0.3 * rng.standard_normal(n) > 0).astype(np.float64)
    return np.arange(n + 1, dtype=np.int64) * k, idx, val, y


def main():
    rank, world, port, dev, transport, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5], sys.argv[6]
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(dev)
    backend = "nccl" if transport == "nccl" else "gloo"
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            **({"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}))
    import spark_agd_b200 as S
    ctx = S.Context.from_torch_distributed(dev, transport=transport)
    res = {}
    n, d = 6001, 1024
    X, y = make_data(n, d, 7)
    lo, hi = rank * n // world, (rank + 1) * n // world
    data = ctx.parallelize(y[lo:hi], X[lo:hi], store="f32")
    rng = np.random.default_rng(11)
    w = rng.standard_normal(d) * 0.1
    loss, g, cnt = data.smooth(S.LogisticGradient(), w)
    res["smooth"] = {"loss": loss, "grad": g.tolist(), "count": cnt}
    wf, hist, st = S.run_with_stats(data, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 8, 0.01, np.zeros(d))
    res["run"] = {"w": wf.tolist(), "hist": hist.tolist(), "passes": st.passes, "backtracks": st.backtracks,
                  "restarts": st.restarts, "collective_kind": st.collective_kind, "collective_calls": st.collective_calls}
    # the other pass structures exchange different payloads (d + 4 or 2 (d + 4) doubles per sweep) through the same buffers:
    # they must give the same bits on every rank
    wm, hm, sm = S.run_with_stats(data, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 8, 0.01, np.zeros(d), memoize=True)
    wu, hu, su = S.run_with_stats(data, S.LogisticGradient(), S.SquaredL2Updater(), 0.0, 8, 0.01, np.zeros(d), fuse=False)
    same = bool(np.array_equal(wm, wf) and np.array_equal(hm, hist) and np.array_equal(wu, wf) and np.array_equal(hu, hist))
    flags = [None] * world
    dist.all_gather_object(flags, same)
    res["modes_bit_identical_on_every_rank"] = bool(all(flags))
    res["memo_fused_passes"] = sm.fused_passes
    # a second dimension on the same handle: the exchange is rebuilt (export / import again under transport="ipc")
    data.unpersist()
    d2 = 260
    X2, y2 = make_data(3000, d2, 9)
    lo, hi = rank * 3000 // world, (rank + 1) * 3000 // world
    data.load_dense(y2[lo:hi], X2[lo:hi], store="f64")
    loss2, g2, cnt2 = data.smooth(S.LeastSquaresGradient(), np.full(d2, 0.01))
    res["smooth_d2"] = {"loss": loss2, "grad": g2.tolist(), "count": cnt2}
    data.close()
    # the synthetic workload generated in place: every rank owns rows [r*n/W, (r+1)*n/W) of the same global matrix
    syn = ctx.synthetic(20000, 512, S.LogisticGradient(), seed=42, store="f32")
    ws, hs, ss = S.run_with_stats(syn, S.LogisticGradient(), S.SimpleUpdater(), 0.0, 5, 0.0, np.zeros(512))
    res["synthetic"] = {"w": ws.tolist(), "hist": hs.tolist(), "passes": ss.passes, "rows_local": syn.local_rows(0)}
    syn.close()
    # mini-batch runs on bf16 shards through the wgmma kernel: the row mask is keyed by the global row id, so every rank
    # but 0 needs its shard's row_base.  Generated in place: rank r's rows start at r * n / W (the oracle's row ids);
    # loaded: rank r's rows are numbered from r << 40
    synb = ctx.synthetic(20000, 512, S.LogisticGradient(), seed=42, store="bf16")
    synb.set_option("k1_variant", "tc")
    wb, hb = S.GradientDescent.runMiniBatchSGD(synb, S.LogisticGradient(), S.SquaredL2Updater(), 0.5, 8, 0.01, 0.25, np.zeros(512))
    labels = [None] * world
    dist.all_gather_object(labels, synb.get_labels(0, 0, synb.local_rows(0)).tolist())
    res["minibatch_bf16_synthetic"] = {"w": wb.tolist(), "hist": hb.tolist(), "labels": sum(labels, [])}
    synb.close()
    lo, hi = rank * n // world, (rank + 1) * n // world
    ldb = ctx.parallelize(y[lo:hi], X[lo:hi], store="bf16")
    ldb.set_option("k1_variant", "tc")
    wl, hl = S.GradientDescent.runMiniBatchSGD(ldb, S.LogisticGradient(), S.SimpleUpdater(), 0.5, 6, 0.0, 0.25, np.zeros(d))
    res["minibatch_bf16_loaded"] = {"w": wl.tolist(), "hist": hl.tolist()}
    ldb.close()
    # a wide sparse shard: d + 4 = 100004 doubles per sweep takes the reduce-scatter + all-gather form of the exchange
    n3, d3, k3 = 9000, 100000, 12
    rp, ix, va, y3 = make_csr(n3, d3, k3, 13)
    lo, hi = rank * n3 // world, (rank + 1) * n3 // world
    wide = ctx.parallelize_csr(y3[lo:hi], rp[lo:hi + 1] - rp[lo], ix[lo:hi].ravel(), va[lo:hi].ravel(), d3, store="f32")
    w3 = np.random.default_rng(17).standard_normal(d3) * 0.1
    l3, g3, c3 = wide.smooth(S.HingeGradient(), w3)
    ww, hw, sw = S.run_with_stats(wide, S.HingeGradient(), S.SquaredL2Updater(), 0.0, 5, 0.05, np.zeros(d3))
    wm3, hm3, sm3 = S.run_with_stats(wide, S.HingeGradient(), S.SquaredL2Updater(), 0.0, 5, 0.05, np.zeros(d3), memoize=True)
    res["wide"] = {"loss": l3, "grad_l2": float(np.linalg.norm(g3)), "grad_head": g3[:64].tolist(), "count": c3,
                   "w_l2": float(np.linalg.norm(ww)), "w_head": ww[:64].tolist(), "hist": hw.tolist(), "passes": sw.passes,
                   "collective_kind": sw.collective_kind, "memo_hist": hm3.tolist(), "memo_w_l2": float(np.linalg.norm(wm3))}
    wide.close()
    if rank == 0:
        with open(out, "w") as f:
            json.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
