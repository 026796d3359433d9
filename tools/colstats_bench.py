"""Column statistics against the scoring and gradient sweeps on the same resident shard: Statistics.colStats against
DeviceDataset.evaluate and DeviceDataset.smooth.

  python tools/colstats_bench.py [--reps 9] [--shapes f32,bf16,bf16w,csr] [--out result.json] [--no-profile]

Shards are generated in place (agd_generate / agd_generate_csr), the shapes of tools/score_bench.py.  Each shape is warmed
up, then colStats, evaluate and smooth alternate, each timed by a host clock around one call (all three end in a device
synchronise); reported are the median and the min-max.  colStats reads X twice; the per-pass kernel times come from a
separate torch.profiler run (CUDA activities) of a few calls after the timed ones, with the evaluation kernel's time from
the same run beside them.  Rates are algorithmic bytes over time (X; CSR: values, column ids and row pointers; evaluate
adds the labels).  The card name and power limit are read in the same run."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SHAPES = {  # name: (rows, d, store, nnz per row or None)
    "f32": (10_000_000, 1024, "f32", None),
    "bf16": (10_000_000, 1024, "bf16", None),
    "bf16w": (6_250_000, 4096, "bf16", None),
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


def spread(ms):
    a = np.array(ms)
    return {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max())}


def kernel_ms(fns, calls=3):
    """Mean device time per call of each kernel (by name) over `calls` calls of every fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            for fn in fns:
                fn()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            out[ev.key] = out.get(ev.key, 0.0) + t / 1e3 / calls
    return out


def pick(kt, pattern):
    return sum(v for k, v in kt.items() if re.search(pattern, k))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if args.reps < 7:
        ap.error("--reps must be at least 7")
    import spark_agd_b200 as S
    ctx = S.Context(devices=[0])
    result = {"card": card(), "reps": args.reps, "shapes": {}}
    for name in args.shapes.split(","):
        rows, d, store, k = SHAPES[name]
        g = S.HingeGradient() if k else S.LogisticGradient()
        if k:
            ds = S.optimization._synthetic_csr(ctx, rows, d, k, g, seed=42, store=store)
            eb = 4 if store == "f32" else 8
            x_bytes = rows * k * (eb + 4) + (rows + 1) * 8
        else:
            ds = ctx.synthetic(rows, d, g, seed=42, store=store)
            eb = {"f32": 4, "f64": 8, "bf16": 2}[store]
            x_bytes = rows * d * eb
        w = np.random.default_rng(1).standard_normal(d) / np.sqrt(k or d)
        cs = lambda: S.Statistics.colStats(ds)  # noqa: E731
        ev = lambda: ds.evaluate(g, w, 0.25, 0.5)  # noqa: E731
        sm = lambda: ds.smooth(g, w)  # noqa: E731
        for _ in range(2):                                                 # warm-up
            cs(); ev(); sm()
        t_cs, t_ev, t_sm = [], [], []
        for _ in range(args.reps):
            t_cs.append(timed(cs))
            t_ev.append(timed(ev))
            t_sm.append(timed(sm))
        c, e, s = spread(t_cs), spread(t_ev), spread(t_sm)
        res = {"rows": rows, "d": d, "store": store, "nnz_per_row": k, "x_bytes": x_bytes, "smooth_kernel": ds.kernel_name(0),
               "colStats": c, "evaluate": e, "smooth": s,
               "colStats_over_evaluate": c["median_ms"] / e["median_ms"],
               "colStats_GBps_two_reads": 2 * x_bytes / (c["median_ms"] * 1e-3) / 1e9}
        if not args.no_profile:
            kt = kernel_ms([cs, ev])
            p1 = pick(kt, r"colstats_(dense|csr)_kernel<.*, 1>")
            p2 = pick(kt, r"colstats_(dense|csr)_kernel<.*, 2>")
            ek = pick(kt, r"score_(dense|csr)_kernel")
            res["kernel_ms"] = {"pass1": p1, "pass2": p2, "evaluate": ek,
                                "colStats_other": pick(kt, r"colstats_(max_reduce|unkey|mu|fill)|k1_reduce")}
            if p1 > 0 and p2 > 0 and ek > 0:
                res["pass1_over_evaluate"] = p1 / ek
                res["pass2_over_evaluate"] = p2 / ek
                res["pass1_GBps"] = x_bytes / (p1 * 1e-3) / 1e9
                res["pass2_GBps"] = x_bytes / (p2 * 1e-3) / 1e9
            res["kernels"] = {kk: v for kk, v in sorted(kt.items(), key=lambda t: -t[1])[:12]}
        result["shapes"][name] = res
        print(json.dumps({name: res}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
