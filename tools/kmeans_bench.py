"""KMeans on resident shards: time of a Lloyd step (agd_kmeans_step), its kernel split, and the k-means|| initialisation.

  python tools/kmeans_bench.py [--reps 5] [--shapes f32,bf16,csr] [--ks 16,64,256] [--init-k 16] [--out result.json]

Shards are generated in place (agd_generate / agd_generate_csr).  For each shape and k a step with sums (DeviceDataset.
kmeans_step) is alternated with `evaluate` on the same shard, the yardstick for one read of X; both are timed by a host clock
around the call and reported as median and min-max after a warm-up of each.  The bar for a dense step is the projection
kernel at the same k plus one evaluate read.  Kernel times come from a separate torch.profiler run (CUDA activities).  The
k-means|| initialisation (five rounds, LocalKMeans on the host) is timed once per shape at --init-k.  The card name and power
limit are read in the same run."""
import argparse
import json
import os
import sys
import time

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--ks", default="16,64,256")
    ap.add_argument("--init-k", type=int, default=16)
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
        if nnz:
            ds = S.optimization._synthetic_csr(ctx, rows, d, nnz, S.HingeGradient(), seed=42, store=store)
        else:
            ds = ctx.synthetic(rows, d, S.LogisticGradient(), seed=42, store=store)
        w = np.linspace(-0.1, 0.1, d)
        ev = lambda: ds.evaluate(S.LogisticGradient(), w)          # noqa: E731
        for k in (int(x) for x in args.ks.split(",")):
            C = np.random.default_rng(k).standard_normal((k, d)) * 0.5
            step = lambda: ds.kmeans_step(C)                        # noqa: E731
            step()
            ev()
            ts, te = [], []
            for _ in range(args.reps):
                ts.append(timed(step))
                te.append(timed(ev))
            res = {"rows": rows, "d": d, "store": store, "nnz_per_row": nnz, "k": k, "step": spread(ts), "evaluate": spread(te)}
            if not args.no_profile:
                kt = kernel_ms(step)
                res["kernel_ms"] = {"assign": pick(kt, r"kmeans_(dense|csr|tiles)_kernel"),
                                    "sort": pick(kt, r"kmeans_keys|bin_"),
                                    "sums": pick(kt, r"kmeans_sums|kmeans_cost|kmeans_counts"),
                                    "copies": pick(kt, r"[Mm]emcpy|[Mm]emset"), "all": sum(kt.values())}
                res["evaluate_kernel_ms"] = pick(kernel_ms(ev), r"score_")
            key = f"{name}_k{k}"
            result["runs"][key] = res
            print(json.dumps({key: res}), flush=True)
        km = S.KMeans(k=args.init_k, seed=5)
        n = ds.count()
        t0 = time.perf_counter()
        init = km._init_parallel(ds, 5, n)
        t1 = time.perf_counter()
        result["runs"][f"{name}_init_k{args.init_k}"] = {"kmeans_parallel_s": t1 - t0, "centres": int(init.shape[0])}
        print(json.dumps({f"{name}_init": t1 - t0}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
