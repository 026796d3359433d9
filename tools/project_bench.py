"""RowMatrix.multiply on resident shards: call time, kernel time and share of the hardware bound of agd_project.

  python tools/project_bench.py [--reps 5] [--shapes f32,bf16,csr] [--ks 16,64,256] [--out result.json] [--no-profile]

Shards are generated in place (agd_generate / agd_generate_csr).  For each shape and k, a projection into an fp32 dataset
(DeviceDataset.project, which opens, fills and synchronises a new dataset; it is closed after each call) is alternated with
`evaluate` on the same shard, the yardstick for one read of X; both are timed by a host clock around the call and reported
as median and min-max after a warm-up of each.  Kernel times come from a separate torch.profiler run (CUDA activities).
The bound is the larger of the HBM term (bytes read and written over 3.35 TB/s) and the compute term: 2 n d k flops over the
67 TFLOP/s fp64 tensor-core rate of the dense kernel, or 2 nnz k flops over the 34 TFLOP/s fp64 CUDA-core rate of the CSR
kernel (H100 SXM data sheet).  The card name and power limit are read in the same run."""
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
HBM = 3.35e12
DMMA = 67e12
FP64 = 34e12
EB = {"f32": 4, "f64": 8, "bf16": 2}


def bound_ms(rows, d, store, nnz, k):
    out_bytes = rows * (k * 4 + 8)                               # fp32 destination rows and labels
    if nnz:
        in_bytes = rows * (nnz * (4 + EB[store]) + 16)           # idx + value per entry, rowptr + label per row
        flops, rate = 2.0 * rows * nnz * k, FP64
    else:
        in_bytes = rows * (d * EB[store] + 8)
        flops, rate = 2.0 * rows * d * k, DMMA
    hbm, comp = (in_bytes + out_bytes) / HBM * 1e3, flops / rate * 1e3
    return {"hbm_ms": hbm, "compute_ms": comp, "bound_ms": max(hbm, comp), "bound_by": "HBM" if hbm >= comp else "compute",
            "flops": flops}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--ks", default="16,64,256")
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
            B = np.random.default_rng(k).standard_normal((d, k)) / np.sqrt(d)
            proj = lambda: ds.project(B, store="f32").close()      # noqa: E731
            proj()
            ev()
            tp, te = [], []
            for _ in range(args.reps):
                tp.append(timed(proj))
                te.append(timed(ev))
            res = {"rows": rows, "d": d, "store": store, "nnz_per_row": nnz, "k": k, "multiply": spread(tp),
                   "evaluate": spread(te), **bound_ms(rows, d, store, nnz, k)}
            if not args.no_profile:
                kt = kernel_ms(proj)
                pk = pick(kt, r"project_(dense|csr)_kernel")
                res["kernel_ms"] = {"project": pk, "scan_and_copies": pick(kt, r"project_scan|[Mm]emcpy|[Mm]emset"),
                                    "all": sum(kt.values())}
                res["evaluate_kernel_ms"] = pick(kernel_ms(ev), r"score_")
                if pk > 0:
                    res["share_of_bound"] = res["bound_ms"] / pk
                    res["TFLOPs"] = res["flops"] / (pk * 1e-3) / 1e12
            key = f"{name}_k{k}"
            result["runs"][key] = res
            print(json.dumps({key: res}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
