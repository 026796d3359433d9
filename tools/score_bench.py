"""Scoring sweep vs gradient sweep on the same resident shard: DeviceDataset.evaluate against DeviceDataset.smooth.

  python tools/score_bench.py [--reps 10] [--shapes f32,bf16,bf16w,csr] [--out result.json]

Shards are generated in place (agd_generate / agd_generate_csr); nothing is copied from the host.  Each shape is warmed up,
then evaluate and smooth alternate, each timed by a host clock around one call (both end in a device synchronise).
Reported: the spread over repetitions and the algorithmic bytes over time (X, labels; CSR: values, column ids, row
pointers, labels) against the H100 SXM data sheet's 3.35 TB/s, which is a data-sheet figure, not a measured one.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

DATASHEET_HBM_BPS = 3.35e12

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import spark_agd_b200 as S
    ctx = S.Context(devices=[0])
    result = {"card": card(), "hbm_peak_bps": DATASHEET_HBM_BPS, "hbm_peak_note": "H100 SXM data sheet, not measured",
              "reps": args.reps, "shapes": {}}
    for name in args.shapes.split(","):
        rows, d, store, k = SHAPES[name]
        g = S.HingeGradient() if k else S.LogisticGradient()
        if k:
            ds = ctx.synthetic_csr(rows, d, k, g, seed=42, store=store)
            eb = 4 if store == "f32" else 8
            nbytes = rows * k * (eb + 4) + (rows + 1) * 8 + rows * 8
        else:
            ds = ctx.synthetic(rows, d, g, seed=42, store=store)
            eb = {"f32": 4, "f64": 8, "bf16": 2}[store]
            nbytes = rows * d * eb + rows * 8
        w = np.random.default_rng(1).standard_normal(d) / np.sqrt(k or d)
        ev = lambda: ds.evaluate(g, w, 0.25, 0.5)  # noqa: E731
        sm = lambda: ds.smooth(g, w)  # noqa: E731
        ev(); sm(); ev(); sm()                                             # warm-up
        t_ev, t_sm = [], []
        for _ in range(args.reps):
            t_ev.append(timed(ev))
            t_sm.append(timed(sm))
        e, s = spread(t_ev), spread(t_sm)
        res = {"rows": rows, "d": d, "store": store, "nnz_per_row": k, "bytes": nbytes, "smooth_kernel": ds.kernel_name(0),
               "evaluate": e, "smooth": s,
               "evaluate_GBps": nbytes / (e["median_ms"] * 1e-3) / 1e9, "smooth_GBps": nbytes / (s["median_ms"] * 1e-3) / 1e9,
               "evaluate_over_smooth": e["median_ms"] / s["median_ms"]}
        res["evaluate_share_of_datasheet_hbm"] = res["evaluate_GBps"] * 1e9 / DATASHEET_HBM_BPS
        result["shapes"][name] = res
        print(json.dumps({name: res}), flush=True)
        ds.close()
    sh = result["shapes"]
    if "f32" in sh:
        for b in ("bf16", "bf16w"):
            if b in sh:
                sh[b]["evaluate_GBps_over_f32"] = sh[b]["evaluate_GBps"] / sh["f32"]["evaluate_GBps"]
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
