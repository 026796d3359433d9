"""CPU self-test of tests/k1_reference.py: the emulated wgmma kernel passes every bound the GPU tests hold the real kernel to
(tests/test_k1_exact.py, tests/test_gpu_parity.py), and each deliberate defect fails the threshold listed next to it.  So
the GPU tests can find these errors before any GPU time is spent."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import k1_reference as R  # noqa: E402

GRAD_NORMWISE, LOSS_NORMWISE = 3e-7, 1.5e-7       # fp32-margin limits of test_bf16_storage_matches_oracle / test_tc_kernel_forms


def _dense(rng, n, d, kind):
    X = R.bf16_to_f32(R.f32_to_bf16_bits(rng.standard_normal((n, d)).astype(np.float32)))
    m = X.astype(np.float64) @ (rng.standard_normal(d) / np.sqrt(d))
    y = m + 0.1 * rng.standard_normal(n) if kind.startswith("least") else (m + rng.logistic(size=n) > 0).astype(float)
    return X, y, rng.standard_normal(d) * 1.2 / np.sqrt(d)


def emulate(X, y, w, kind, defect=None, mask=None):
    """(loss, gradient, count) of one applySmooth on the emulated wgmma kernel, default mapping."""
    kw2 = {"drop_lo": {"drop_lo": True}, "swap_mid_lo": {"swap_mid_lo": True}, "row_xor": {"row_xor": 1},
           "rows128": {"rows": 128}}.get(defect, {})
    kw1 = {"w_bf16": {"w_bf16": True}, "no_flush": {"flush": False}}.get(defect, {})
    m = R.tc_margins_f32(X, w, **kw1)
    r, loss = R.row_terms(kind, m, y)
    sel = np.ones(len(y), bool) if mask is None else mask
    r = np.where(sel, r, 0.0)
    cnt = int(sel.sum())
    return float(loss[sel].sum() / cnt), R.tc_gradient_sum(X, r, **kw2) / cnt, cnt


def checks(defect):
    """Every threshold as value / limit (<= 1 passes)."""
    out = {}
    rng = np.random.default_rng(7)
    # one-hot designs, least squares at w = 0: r = -2y exactly
    for d in (128, 640):
        n = 2113
        X, col = R.one_hot_design(n, d, rng)
        y = R.full_labels(n, rng)
        _, g, cnt = emulate(X, y, np.zeros(d), "least_squares", defect)
        e1, e2 = R.one_hot_check(g, X[np.arange(n), col], col, -2.0 * y, cnt)
        out[f"one-hot d={d}: 2^-40 against the pieces"] = e1
        out[f"one-hot d={d}: 2^-22 against r"] = e2
    # dense shards: element-wise bounds and the norm-wise limits
    for kind in ("logistic", "least_squares", "hinge"):
        X, y, w = _dense(rng, 1000, 512, kind)
        loss, g, cnt = emulate(X, y, w, kind, defect)
        gb, lb, (rl, rg, _) = R.dense_bounds(kind, X, y, w)
        out[f"dense {kind}: element-wise gradient"] = np.max(np.abs(g - rg) / gb)
        out[f"dense {kind}: loss bound"] = abs(loss - rl) / lb
        out[f"dense {kind}: norm-wise gradient"] = np.linalg.norm(g - rg) / np.linalg.norm(rg) / GRAD_NORMWISE
        out[f"dense {kind}: norm-wise loss"] = abs(loss - rl) / abs(rl) / LOSS_NORMWISE
    # zero-residual least-squares probe: the loss is the mean squared margin error, within 1% of the emulator's
    X, _, w = _dense(rng, 400, 3200, "least_squares")      # 25 ring groups per row: 13 flushes
    y = R.exact_margins(X, w)
    mse = np.mean((R.tc_margins_f32(X, w) - y) ** 2)
    loss, _, _ = emulate(X, y, w, "least_squares", defect)
    out["zero-residual probe: within 1% of the phase-1 emulator"] = abs(loss / mse - 1.0) / 0.01
    # the mini-batch mask (fraction 0.25, the seed of iteration 1), on a shard of rank 0 and of rank 1 (row_base = 2^40)
    X, y, w = _dense(rng, 700, 256, "logistic")
    thresh = int(0.25 * 2.0 ** 64)
    for rank in (0, 1):
        rows = (rank << 40) + np.arange(700)
        truth = R.row_selected(43, thresh, rows)
        used = {"mask_ignored": np.ones(700, bool), "row_base_ignored": R.row_selected(43, thresh, np.arange(700))}.get(defect, truth)
        loss, g, cnt = emulate(X, y, w, "logistic", None, used)
        gb, lb, (rl, rg, rc) = R.dense_bounds("logistic", X, y, w, mask=truth)
        out[f"mini-batch rank {rank}: element-wise gradient"] = max(np.max(np.abs(g - rg) / gb), float(cnt != rc) * 2)
    return out


# defect -> the threshold that rejects it (a key of checks())
DEFECTS = {
    "drop_lo": "one-hot d=128: 2^-40 against the pieces",
    "row_xor": "one-hot d=128: 2^-22 against r",
    "rows128": "one-hot d=128: 2^-40 against the pieces",
    "w_bf16": "zero-residual probe: within 1% of the phase-1 emulator",
    "no_flush": "zero-residual probe: within 1% of the phase-1 emulator",
    "mask_ignored": "mini-batch rank 0: element-wise gradient",
    "row_base_ignored": "mini-batch rank 1: element-wise gradient",
}


def test_emulated_kernel_meets_every_bound():
    res = checks(None)
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_each_defect_fails_its_threshold(defect):
    res = checks(defect)
    assert res[DEFECTS[defect]] > 1.0, (defect, DEFECTS[defect], res[DEFECTS[defect]])


def test_swapped_mid_and_lo_columns_are_the_same_arithmetic():
    """mid and lo in each other's B columns: every lane still reads all three pieces of its own rows, and the fp64 sum of the
    three fp32 partials is exact either way, so the result is bit-identical and no numerical test can (or needs to) see it.
    That exactness needs the three fp32 partials of a tile to span at most 53 bits (from the top bit of the largest to the
    last bit of the smallest); the shards here do, and where a tile does not, the two orders differ in the last fp64 bit."""
    rng = np.random.default_rng(3)
    X, y, w = _dense(rng, 300, 256, "logistic")
    r, _ = R.row_terms("logistic", R.tc_margins_f32(X, w), y)
    assert np.array_equal(R.tc_gradient_sum(X, r), R.tc_gradient_sum(X, r, swap_mid_lo=True))


def test_reference_pieces_and_margins():
    rng = np.random.default_rng(5)
    r = rng.standard_normal(1000) * np.ldexp(1.0, rng.integers(-30, 30, 1000))
    hi, mid, lo = R.split3(r)
    assert np.all(np.abs(r - (hi + mid + lo)) <= 2.0 ** -24 * np.abs(r))
    assert np.array_equal(R.bf16_rne(hi), hi) and np.array_equal(R.bf16_rne(lo), lo)
    f = rng.standard_normal(1000).astype(np.float32)
    assert np.array_equal(R.bf16_rne(f.astype(np.float64)), R.bf16_to_f32(R.f32_to_bf16_bits(f)).astype(np.float64))
    assert R.bf16_rne(np.array([2.0 ** -140]))[0] == 0.0 and R.bf16_rne(np.array([3 * 2.0 ** -134]))[0] == 2.0 ** -132
    X = R.bf16_to_f32(R.f32_to_bf16_bits(rng.standard_normal((20, 64)).astype(np.float32)))
    w = rng.standard_normal(64)
    from fractions import Fraction
    exact = [float(sum(Fraction(float(a)) * Fraction(float(b)) for a, b in zip(X[i], w))) for i in range(20)]
    assert np.array_equal(R.exact_margins(X, w), exact)
