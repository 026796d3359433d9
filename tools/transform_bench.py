"""What a feature transform costs: one gradient sweep (agd_smooth) on a generated shard without a transform, with the
intercept only, with scaling only and with both (agd_set_feature_transform).

  python tools/transform_bench.py [--reps 7] [--shapes f32,bf16,bf16w,csr] [--out result.json]

The transform is installed on the handle once per form through the C-ABI, so a timed call is the sweep and nothing else of
the view machinery: agd_smooth at a point, timed by a host clock around the call (it ends in a device synchronise), the forms
alternating within every repetition.  With scaling the call adds one small kernel that writes w_eff = (s o v, b) before K1 and,
on CSR shards, one that scales the gradient columns after it; dense shards scale in the slab reduction.  The card name and
power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SHAPES = {  # name: (rows, d, store, nnz per row or None)
    "f32": (10_000_000, 1024, "f32", None),          # ring, the headline shape
    "bf16": (10_000_000, 1024, "bf16", None),        # wgmma
    "bf16w": (2_500_000, 4096, "bf16", None),        # wgmma, the widest rows it takes
    "csr": (20_000_000, 1_000_000, "f32", 64),       # the configuration of tools/csr_bench.py
}
FORMS = {"none": (False, 0), "bias": (False, 1), "scale": (True, 0), "both": (True, 1)}


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
    L = S._native.lib()
    ctx = S.Context(devices=[0])
    result = {"card": card(), "reps": args.reps, "shapes": {}}
    for name in args.shapes.split(","):
        rows, d, store, k = SHAPES[name]
        g = S.HingeGradient() if k else S.LogisticGradient()
        ds = ctx.synthetic_csr(rows, d, k, g, seed=42, store=store) if k else ctx.synthetic(rows, d, g, seed=42, store=store)
        rng = np.random.default_rng(1)
        w = np.append(rng.standard_normal(d) / np.sqrt(k or d), 0.25)
        s = rng.uniform(0.5, 2.0, d)
        grad = np.empty(d + 1)
        loss, cnt = C.c_double(), C.c_int64()

        def sweep(form):
            scaled, bias = FORMS[form]
            S._native.check(L.agd_set_feature_transform(ds.h, s.ctypes.data_as(C.c_void_p) if scaled else None, bias), ds.h)
            t0 = time.perf_counter()
            S._native.check(L.agd_smooth(ds.h, g.kind, w.ctypes.data_as(C.c_void_p), C.byref(loss),
                                         grad.ctypes.data_as(C.c_void_p), C.byref(cnt)), ds.h)
            ms = (time.perf_counter() - t0) * 1e3
            S._native.check(L.agd_set_feature_transform(ds.h, None, 0), ds.h)
            return ms

        for f in FORMS:   # warm-up
            sweep(f)
        t = {f: [] for f in FORMS}
        for _ in range(args.reps):
            for f in FORMS:
                t[f].append(sweep(f))
        res = {"rows": rows, "d": d, "store": store, "nnz_per_row": k, "kernel": ds.kernel_name(0),
               "smooth": {f: spread(v) for f, v in t.items()}}
        base = res["smooth"]["none"]["median_ms"]
        res["over_none"] = {f: res["smooth"][f]["median_ms"] / base for f in FORMS}
        result["shapes"][name] = res
        print(json.dumps({name: res}), flush=True)
        ds.close()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
