"""NaiveBayes and MulticlassMetrics on resident shards: NaiveBayes.train, device predict and MulticlassMetrics(model, data),
against `evaluate` (one read of X) and the k-means assignment kernel at k = C.

  python tools/nb_bench.py [--reps 5] [--shapes f32,bf16,csr] [--cs 2,16,256] [--out result.json]

Generated features are Gaussian and NaiveBayes refuses negative features, so each shard is one nonnegative block of 65,536 rows
(small integers, labels from C classes spread over the block) appended into the shard until it holds the rows of the shape:
dense shards into a reserved shard, CSR shards (64 stored entries per row) in chunks of 32 blocks.  For each shape and C, train,
predict (this process's rows, DeviceDataset.linear_argmax and the label lookup) and MulticlassMetrics are alternated with
`evaluate` on the same shard, each timed by a host clock around the call (median and min-max after a warm-up).  Kernel times
come from torch.profiler runs of their own.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
from gramian_bench import card, kernel_ms, pick, spread, timed  # noqa: E402

SHAPES = {  # name: (rows, d, store, nnz per row or None)
    "f32": (10_000_000, 1024, "f32", None),
    "bf16": (10_000_000, 1024, "bf16", None),
    "csr": (20_000_000, 4096, "f32", 64),
}
BLOCK = 65_536


def block(d, nnz, C, seed):
    """One nonnegative block: rows whose features favour their class's columns, labels -C/2 .. C/2 - 1 in steps of 0.5"""
    rng = np.random.default_rng(seed)
    cls = rng.integers(0, C, BLOCK)
    y = (cls - C // 2) * 0.5
    if nnz is None:
        X = rng.integers(0, 3, (BLOCK, d)).astype(np.float32)
        X[np.arange(BLOCK), (cls * 7) % d] += 4.0
        return y, X
    idx = np.sort(rng.choice(d, (BLOCK, nnz)), axis=1).astype(np.int32)
    idx[:, 0] = (cls * 7) % d
    idx = np.sort(idx, axis=1)
    val = rng.integers(1, 4, (BLOCK, nnz)).astype(np.float32)
    return y, (idx, val)


def load(S, ctx, rows, d, store, nnz, C):
    N, opt = S._native, S.optimization
    y, X = block(d, nnz, C, seed=C)
    ds = S.DeviceDataset(ctx)
    reps = (rows + BLOCK - 1) // BLOCK
    if nnz is None:
        N.check(N.lib().agd_reserve(ds.h, 0, reps * BLOCK, d, opt._STORE[store]), ds.h)
        for _ in range(reps):
            ds.load_dense(y, X, store=store)
        return ds
    idx, val = X
    per = 32
    for r0 in range(0, reps, per):
        n = min(per, reps - r0)
        rp = np.arange(n * BLOCK + 1, dtype=np.int64) * nnz
        ds.load_csr(np.tile(y, n), rp, np.tile(idx, (n, 1)).ravel(), np.tile(val, (n, 1)).ravel(), d, store=store)
    return ds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--cs", default="2,16,256")
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if args.reps < 3:
        ap.error("--reps must be at least 3")
    import spark_agd_b200 as S
    ctx = S.Context(devices=[0])
    result = {"card": card(), "reps": args.reps, "runs": {}}
    print(json.dumps({"card": result["card"]}), flush=True)
    for name in args.shapes.split(","):
        rows, d, store, nnz = SHAPES[name]
        for C in (int(x) for x in args.cs.split(",")):
            ds = load(S, ctx, rows, d, store, nnz, C)
            w = np.linspace(-0.1, 0.1, d)
            ev = lambda: ds.evaluate(S.LogisticGradient(), w)          # noqa: E731
            train = lambda: S.NaiveBayes.train(ds)                      # noqa: E731
            model = train()
            predict = lambda: model.predict(ds)                         # noqa: E731
            metrics = lambda: S.MulticlassMetrics(model, ds)            # noqa: E731
            centres = np.random.default_rng(C).random((C, d))
            assign = lambda: ds.kmeans_assign_rows(0, 0, ds.local_rows(0), centres)   # noqa: E731
            argmax = lambda: ds.linear_argmax_rows(0, 0, ds.local_rows(0), model.theta, model.pi)   # noqa: E731
            fns = {"train": train, "predict": predict, "metrics": metrics, "evaluate": ev}
            for f in fns.values():
                f()
            times = {k: [] for k in fns}
            for _ in range(args.reps):
                for k, f in fns.items():
                    times[k].append(timed(f))
            res = {"rows": ds.count(), "d": d, "store": store, "nnz_per_row": nnz, "C": C,
                   "accuracy": metrics().precision()}
            res.update({k: spread(v) for k, v in times.items()})
            if not args.no_profile:
                assign_kernels = r"kmeans_(dense|csr|tiles)_kernel"
                res["kernel_ms"] = {
                    "train": sum(kernel_ms(train).values()),
                    "argmax": pick(kernel_ms(argmax), assign_kernels),
                    "kmeans_assign_k_eq_C": pick(kernel_ms(assign), assign_kernels),
                    "metrics_all": sum(kernel_ms(metrics).values()),
                    "evaluate": pick(kernel_ms(ev), r"score_"),
                }
            key = f"{name}_C{C}"
            result["runs"][key] = res
            print(json.dumps({key: res}), flush=True)
            ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
