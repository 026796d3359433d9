"""What a view costs: one gradient sweep (agd_smooth) on a whole generated shard against a 0.8 view of it (one predicate
and two), and evaluate on the whole shard against a 0.2 view.

  python tools/split_bench.py [--reps 7] [--shapes f32,f32w,bf16,bf16ring,csr] [--out result.json]

Shards are generated in place.  Every sweep is one agd_smooth call -- the same single-point kernel form on the whole shard
and on the views, so the comparison is like for like -- timed by a host clock around the call (it ends in a device
synchronise); the whole shard and the views alternate.  The ring and wgmma kernels read a view as a bitmap of the shard's
rows, drawn when the view first runs after another filter: "first" is a call that draws it (what one call on a view costs
when views alternate), "sweep" the call right after it on the same view (what every further sweep of a run costs).
evaluate is timed the same way, alternating too.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SHAPES = {  # name: (rows, d, store, nnz per row or None, options)
    "f32": (10_000_000, 1024, "f32", None, {}),                        # ring, one vector per thread (the headline shape)
    "f32w": (2_500_000, 4096, "f32", None, {}),                        # ring, four vectors per thread
    "bf16": (10_000_000, 1024, "bf16", None, {}),                      # wgmma
    "bf16ring": (10_000_000, 1024, "bf16", None, {"k1_variant": "ring"}),  # the ring kernel on bf16 storage
    "csr": (20_000_000, 1_000_000, "f32", 64, {}),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def spread(ms):
    a = np.array(ms)
    return {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import spark_agd_b200 as S
    ctx = S.Context(devices=[0])
    result = {"card": card(), "reps": args.reps, "shapes": {}}
    for name in args.shapes.split(","):
        rows, d, store, k, opts = SHAPES[name]
        g = S.HingeGradient() if k else S.LogisticGradient()
        ds = ctx.synthetic_csr(rows, d, k, g, seed=42, store=store) if k else ctx.synthetic(rows, d, g, seed=42, store=store)
        for key, val in opts.items():
            ds.set_option(key, val)
        one = ds.sample(False, 0.8, seed=7)
        two = ds.randomSplit([0.9, 0.1], seed=8)[0].sample(False, 0.8 / 0.9, seed=9)
        test = ds.randomSplit([0.8, 0.2], seed=10)[1]
        w = np.random.default_rng(1).standard_normal(d) / np.sqrt(k or d)

        def sweep(data):
            t0 = time.perf_counter()
            data.smooth(g, w)
            return (time.perf_counter() - t0) * 1e3

        def ev(data):
            t0 = time.perf_counter()
            data.evaluate(g, w)
            return (time.perf_counter() - t0) * 1e3

        views = {"whole": ds, "view0.8_1pred": one, "view0.8_2pred": two}
        for v in views.values():   # warm-up
            sweep(v)
        t = {key: [] for key in views}
        t1 = {key: [] for key in views}
        for _ in range(args.reps):
            for key, v in views.items():
                t1[key].append(sweep(v))
                t[key].append(sweep(v))
        ev(ds); ev(test)
        te = {"whole": [], "view0.2": []}
        for _ in range(args.reps):
            te["whole"].append(ev(ds))
            te["view0.2"].append(ev(test))
        res = {"rows": rows, "d": d, "store": store, "nnz_per_row": k, "kernel": ds.kernel_name(0),
               "smooth": {key: spread(v) for key, v in t.items()},
               "smooth_first": {key: spread(v) for key, v in t1.items()},
               "evaluate": {key: spread(v) for key, v in te.items()},
               "counts": {"whole": rows, "view0.8_1pred": one.count(), "view0.8_2pred": two.count(), "view0.2": test.count()}}
        base = res["smooth"]["whole"]["median_ms"]
        res["smooth_view_over_whole"] = {key: res["smooth"][key]["median_ms"] / base for key in views}
        result["shapes"][name] = res
        print(json.dumps({name: res}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
