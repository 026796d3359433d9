"""Times the bf16 gradient kernels (wgmma vs CUDA-core ring) on a config-4-shaped shard."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import spark_agd_b200 as S
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 6_250_000
d = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
ds = S.Context(devices=[0]).synthetic(rows, d, S.LeastSquaresGradient(), seed=42, store="bf16")
w0 = np.zeros(d)
bytes_pass = rows * (d * 2 + 8)
def t(label, grad, **opts):
    for k, v in opts.items():
        ds.set_option(k, v)
    S.run_with_stats(ds, grad, S.SimpleUpdater(), 0.0, 1, 0.0, w0, 8.0, 8.0, 1.0, 0.9, False)
    _, h, st = S.run_with_stats(ds, grad, S.SimpleUpdater(), 0.0, 5, 0.0, w0, 8.0, 8.0, 1.0, 0.9, False)
    ms = st.k1_ms_total / st.k1_launches
    print(json.dumps(dict(label=label, rows=rows, d=d, **opts, k1_ms=round(ms, 3), gbs=round(bytes_pass / ms / 1e6, 1),
                          frac_of_datasheet=round(bytes_pass / ms / 1e6 / 3350.0, 4), loss=h[-1])), flush=True)
LS = S.LeastSquaresGradient()
t("tc LS (default: 2 rows/thread, one 3-D copy per group)", LS, k1_variant="tc", ring_rows=0, ring_ctas=0, k1_diag=0)
t("tc logistic", S.LogisticGradient())
t("tc LS, 4 rows/thread", LS, ring_rows=4)
t("tc LS, row per lane", LS, ring_rows=1)
t("tc LS, 2-D copies", LS, ring_rows=0, ring_ctas=2)
t("diag: no consumer arithmetic", LS, ring_ctas=0, k1_diag=100)
t("diag: no MMAs", LS, k1_diag=101)
if len(sys.argv) > 3:
    t("ring LS (CUDA cores)", LS, k1_variant="ring", k1_diag=0)
