"""Ranking metrics vs evaluation on the same resident shard: DeviceDataset.binary_curve (areas only, one agd_binary_curve
call) against DeviceDataset.evaluate.

  python tools/binmetrics_bench.py [--reps 10] [--shapes f32,bf16,csr] [--out result.json]

Shards are generated in place; nothing is copied from the host.  Each shape is warmed up, then the two calls alternate, each
timed by a host clock around one call (both end in a device synchronise).  A separate torch.profiler run of one call per shape
splits its kernel time into the key sweep (score_*_kernel) and the sort, run-length reduce and areas (bin_*_kernel): the sort's
share.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SHAPES = {  # name: (rows, d, store, nnz per row or None)
    "f32": (10_000_000, 1024, "f32", None),
    "bf16": (10_000_000, 1024, "bf16", None),
    "csr": (20_000_000, 1_000_000, "f32", 64),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def kernel_split(fn):
    """CUDA kernel time (ms) of one call of fn, by kernel family."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    split = {"key_sweep_ms": 0.0, "sort_reduce_areas_ms": 0.0, "other_ms": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        ms = t / 1e3
        if "score_" in e.key:
            split["key_sweep_ms"] += ms
        elif "bin_" in e.key:
            split["sort_reduce_areas_ms"] += ms
        elif "Memcpy" not in e.key and "Memset" not in e.key:
            split["other_ms"] += ms
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import spark_agd_b200 as S
    ctx = S.Context(devices=[0])
    result = {"card": card(), "reps": args.reps, "shapes": {}}
    for name in args.shapes.split(","):
        rows, d, store, k = SHAPES[name]
        g = S.HingeGradient() if k else S.LogisticGradient()
        ds = ctx.synthetic_csr(rows, d, k, g, seed=42, store=store) if k else ctx.synthetic(rows, d, g, seed=42, store=store)
        w = np.random.default_rng(1).standard_normal(d) / np.sqrt(k or d)
        ev = lambda: ds.evaluate(g, w, 0.25, 0.5)  # noqa: E731
        bc = lambda: ds.binary_curve(w, 0.25, curve=False)  # noqa: E731
        ev(); bc(); ev(); bc()                                             # warm-up (and scratch allocation)
        t_ev, t_bc = [], []
        for _ in range(args.reps):
            t_ev.append(timed(ev))
            t_bc.append(timed(bc))
        s = bc()[0]
        res = {"rows": rows, "d": d, "store": store, "nnz_per_row": k,
               "evaluate_median_ms": float(np.median(t_ev)), "evaluate_min_ms": float(np.min(t_ev)),
               "evaluate_max_ms": float(np.max(t_ev)),
               "binary_curve_median_ms": float(np.median(t_bc)), "binary_curve_min_ms": float(np.min(t_bc)),
               "binary_curve_max_ms": float(np.max(t_bc)),
               "areaUnderROC": float(s[3]), "positives": int(s[0]), "negatives": int(s[1])}
        res["binary_curve_over_evaluate"] = res["binary_curve_median_ms"] / res["evaluate_median_ms"]
        res.update(kernel_split(bc))
        kt = res["key_sweep_ms"] + res["sort_reduce_areas_ms"] + res["other_ms"]
        res["sort_share_of_kernel_time"] = res["sort_reduce_areas_ms"] / kt if kt > 0 else float("nan")
        result["shapes"][name] = res
        print(json.dumps({name: res}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
