"""RowMatrix.computeCovariance on resident shards: call time, kernel split and the fp64 tensor-core rate of the Gramian kernel.

  python tools/gramian_bench.py [--reps 7] [--shapes f32,bf16,bf16w,f32x,csr] [--out result.json] [--no-profile]

Shards are generated in place (agd_generate / agd_generate_csr).  Each shape is warmed up, then computeCovariance is timed by
a host clock around one call (it ends in a device synchronise and includes the O(d^2) host derivation); reported are the
median and the min-max.  The kernel split -- the mu pass (colStats pass 1 and its slab reduce), the Gramian kernel, the slab
reduce and the copy back -- comes from a separate torch.profiler run (CUDA activities) of a few calls after the timed ones.
The rate counts the flops of the blocks the dense kernel computes: 2 x 128^2 per row and block pair I <= J.  The card name
and power limit are read in the same run."""
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
    "f32x": (1_000_000, 8192, "f32", None),
    "csr": (1_000_000, 4096, "f32", 64),
}
BLK = 128   # the dense kernel's block width (csrc/gramian.cu)


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


def kernel_ms(fn, calls=2):
    """Mean device time per call of each kernel (by name) over `calls` calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
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
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if args.reps < 5:
        ap.error("--reps must be at least 5")
    import spark_agd_b200 as S
    ctx = S.Context(devices=[0])
    result = {"card": card(), "reps": args.reps, "shapes": {}}
    print(json.dumps({"card": result["card"]}), flush=True)
    for name in args.shapes.split(","):
        rows, d, store, k = SHAPES[name]
        if k:
            ds = S.optimization._synthetic_csr(ctx, rows, d, k, S.HingeGradient(), seed=42, store=store)
        else:
            ds = ctx.synthetic(rows, d, S.LogisticGradient(), seed=42, store=store)
        rm = S.RowMatrix(ds)
        cov = rm.computeCovariance                                        # warm-up
        cov()
        t = [timed(cov) for _ in range(args.reps)]
        res = {"rows": rows, "d": d, "store": store, "nnz_per_row": k, "computeCovariance": spread(t)}
        nb = (d + BLK - 1) // BLK
        flops = 2.0 * BLK * BLK * (nb * (nb + 1) // 2) * rows
        if not args.no_profile:
            kt = kernel_ms(cov)
            gk = pick(kt, r"gramian_(dense|csr)_kernel")
            res["kernel_ms"] = {"mu_pass": pick(kt, r"colstats_(dense|csr)_kernel|colstats_mu"),
                                "gramian": gk,
                                "reduce_center_copy": pick(kt, r"k1_reduce|gramian_center|[Mm]emcpy|[Mm]emset"),
                                "all": sum(kt.values())}
            if not k and gk > 0:
                res["gramian_fp64_TFLOPs"] = flops / (gk * 1e-3) / 1e12
            res["kernels"] = {kk: v for kk, v in sorted(kt.items(), key=lambda x: -x[1])[:10]}
        result["shapes"][name] = res
        print(json.dumps({name: res}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
