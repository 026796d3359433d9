"""Plain high-precision references for the gradient kernels (numpy and the standard library only; not a test module).

- exact bf16 decoding and double -> bf16 rounding to nearest-even; the hi / mid / lo split of r in k1_tc.cu;
- per-row fp64 margins, multipliers and losses of the four gradients (Gradient.scala of spark-mllib 1.3.0);
- correctly rounded margins: w split into two 26-bit halves (every x . w part of a bf16 or fp32 x is then an exact
  double) and math.fsum per row;
- the counter-based mini-batch row mask (Philox4x32-10, k1_device.cuh);
- an emulator of the wgmma kernel's arithmetic: phase 1 in fp32 (w rounded to fp32, two accumulators per thread holding
  features 0,2,4,6 and 1,3,5,7 of its 8-feature chunk, flushed to fp64 every two ring groups) and phase 2 (r of each
  16-row tile scaled by 2^-s, split into three bf16 pieces, fp32 sums over the tile's rows, fp64 across tiles);
- the element-wise error bounds the GPU tests hold the kernels to.
The emulator takes the defects that tests/test_k1_reference.py injects to show that those bounds catch them."""
import math

import numpy as np

KINDS = ("logistic", "least_squares", "least_squares_half", "hinge")
# d r / d m for the bound on how a margin error moves r: max sigmoid' = 1/4, least squares 2, halved 1, hinge 0
LAMBDA = {"logistic": 0.25, "least_squares": 2.0, "least_squares_half": 1.0, "hinge": 0.0}
EPS_F32_MARGIN = 2.0 ** -20      # margin error of the fp32 phase 1, relative to sum_j |x_ij w_j|
EPS_PIECES = 2.0 ** -20          # gradient error of the bf16 x 3 split + fp32 tile sums, relative to sum_i |x_ij r_i|
ONE_HOT_EXACT = 2.0 ** -40       # one-hot designs: gradient against sum x (hi + mid + lo), relative to sum |x r|
ONE_HOT_R = 2.0 ** -22           # ... and against the exact r


def bf16_to_f32(raw):
    """Exact widening of raw bf16 bit patterns (uint16) to float32."""
    return (np.asarray(raw).astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16_bits(x):
    """float32 -> bf16 bit patterns, round to nearest-even (what a bf16 load stores)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_rne(x):
    """double -> the nearest bf16 value (ties to even), as float64, subnormals included; one rounding."""
    x = np.asarray(x, dtype=np.float64)
    _, e = np.frexp(x)                                   # |x| = m 2^e, 0.5 <= m < 1
    q = np.maximum(e - 8, -133).astype(np.float64)       # 8 significant bits; bf16 quantum bottoms out at 2^-133
    return np.ldexp(np.rint(np.ldexp(x, (-q).astype(np.int64))), q.astype(np.int64))


def split3(r):
    """The hi / mid / lo pieces of k1_tc.cu (each a bf16 value, as float64)."""
    hi = bf16_rne(r)
    r1 = r - hi
    mid = bf16_rne(r1)
    lo = bf16_rne(r1 - mid)
    return hi, mid, lo


def row_terms(kind, m, y):
    """Per-row fp64 multiplier loss'(m) and loss."""
    m = np.asarray(m, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    if kind == "logistic":
        with np.errstate(over="ignore"):
            mult = 1.0 / (1.0 + np.exp(-m)) - y
        loss = np.logaddexp(0.0, -m) + np.where(y > 0, 0.0, m)
    elif kind == "least_squares":
        mult, loss = 2.0 * (m - y), (m - y) ** 2
    elif kind == "least_squares_half":
        mult, loss = m - y, (m - y) ** 2 / 2.0
    else:
        s = 2.0 * y - 1.0
        act = 1.0 > s * m
        mult, loss = np.where(act, -s, 0.0), np.where(act, 1.0 - s * m, 0.0)
    return mult, loss


def exact_margins(X, w):
    """Correctly rounded x_i . w for X holding bf16 or fp32 values (24 significant bits at most)."""
    w = np.asarray(w, dtype=np.float64)
    t = w * 134217729.0                                  # Veltkamp: 2^27 + 1
    wh = t - (t - w)
    wl = w - wh                                          # wh, wl: at most 26 significant bits each
    Xd = np.asarray(X, dtype=np.float64)
    P, Q = Xd * wh, Xd * wl                              # exact products
    return np.array([math.fsum(np.concatenate([P[i], Q[i]])) for i in range(Xd.shape[0])])


def row_selected(seed, thresh, rows):
    """The mini-batch mask: Philox4x32-10 keyed by `seed`, counter (row, 0, 6); kept iff the 64-bit draw < thresh."""
    M = np.uint64(0xFFFFFFFF)
    g = np.asarray(rows, dtype=np.uint64)
    c0, c1 = g & M, g >> np.uint64(32)
    c2, c3 = np.zeros_like(g), np.full_like(g, 6)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & M, p1 >> np.uint64(32), p1 & M
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return ((c0 << np.uint64(32)) | c1) < np.uint64(thresh)


def group_blocks(d):
    """64-feature blocks per ring group: the largest even divisor of d / 64 that is <= 8."""
    gb = 8
    while (d // 64) % gb:
        gb -= 2
    return gb


def _fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def tc_margins_f32(X, w, w_bf16=False, flush=True):
    """Phase 1 of the default mapping.  X: (n, d) bf16 values; per thread (chunk vv of every group) two fp32 accumulators
    (features 0,2,4,6 and 1,3,5,7 of the chunk), their fp32 sum added into fp64 every two ring groups.
    Defects: w_bf16 rounds w to bf16 instead of fp32; flush=False keeps the fp32 accumulators for the whole row."""
    n, d = X.shape
    gb = group_blocks(d)
    ngt = d // (64 * gb)
    wf = (bf16_rne(w) if w_bf16 else np.asarray(w, dtype=np.float64)).astype(np.float32)
    Xc = np.asarray(X, dtype=np.float32).reshape(n, ngt, gb * 8, 8)
    Wc = wf.reshape(ngt, gb * 8, 8)
    pd = np.zeros((n, gb * 8))
    ae = np.zeros((n, gb * 8), np.float32)
    ao = np.zeros((n, gb * 8), np.float32)
    for gi in range(ngt):
        for q in range(4):
            ae = _fma32(Xc[:, gi, :, 2 * q], Wc[gi, :, 2 * q], ae)
            ao = _fma32(Xc[:, gi, :, 2 * q + 1], Wc[gi, :, 2 * q + 1], ao)
        if (flush and (gi & 1)) or gi + 1 == ngt:
            pd += (ae + ao).astype(np.float64)
            ae[:] = 0
            ao[:] = 0
    return pd.sum(axis=1)


def tc_gradient_sum(X, r, rows=16, drop_lo=False, swap_mid_lo=False, row_xor=0, scale=True):
    """Phase 2: sum_i x_i r_i (not yet divided by the count).  X: (n, d) bf16 values; r: per-row multipliers (0 for rows the
    mask drops).  Defects: drop_lo, swap_mid_lo (mid and lo in each other's B columns: the lane adds lo before mid),
    row_xor = 1 (row p's pieces land on row p ^ 1 of its tile), rows = 128 (fp32 sums over 128 rows), scale=False (no
    power-of-two scaling of the tile)."""
    X = np.asarray(X, dtype=np.float32)
    n, d = X.shape
    T = -(-n // rows)
    Xp = np.zeros((T * rows, d), np.float32)
    Xp[:n] = X
    rp = np.zeros(T * rows)
    rp[:n] = r
    if row_xor:
        rp = rp.reshape(T, rows)[:, np.arange(rows) ^ row_xor].ravel()
    s16 = np.repeat(tile_scales(rp), 16) if (scale and rows == 16) else np.zeros(T * rows, np.int64)
    pieces = split3(np.ldexp(rp, -s16))
    if drop_lo:
        pieces = (pieces[0], pieces[1], np.zeros_like(pieces[2]))
    Xt = Xp.reshape(T, rows, d)
    sums = [np.add.reduce(Xt * p.astype(np.float32).reshape(T, rows, 1), axis=1, dtype=np.float32).astype(np.float64)
            for p in pieces]
    tile = (sums[0] + sums[2]) + sums[1] if swap_mid_lo else (sums[0] + sums[1]) + sums[2]
    if rows == 16:
        tile = np.ldexp(tile, s16[::16, None])
    return tile.sum(axis=0)


def tile_scales(r):
    """s per 16-row tile: the exponent of max |r| over the tile (max |r| = m 2^s, 0.5 <= m < 1); 0 for an all-zero tile."""
    rp = np.zeros(-(-len(r) // 16) * 16)
    rp[:len(r)] = r
    amax = np.abs(rp).reshape(-1, 16).max(axis=1)
    _, s = np.frexp(amax)
    return np.where((amax > 0) & np.isfinite(amax), s, 0).astype(np.int64)


def one_hot_design(n, d, rng, exp_range=4):
    """Row i = 16 t + p has one nonzero, at feature (t + 131 p) mod d: every per-tile fp32 sum then holds one product.
    x: random bf16 values of magnitude 2^(+-exp_range), random signs.  Returns (X as float32, feature of each row)."""
    i = np.arange(n)
    col = (i // 16 + 131 * (i % 16)) % d
    mag = np.ldexp(1.0 + rng.integers(0, 128, n) / 128.0, rng.integers(-exp_range, exp_range, n))
    x = (mag * rng.choice([-1.0, 1.0], n)).astype(np.float32)
    X = np.zeros((n, d), np.float32)
    X[i, col] = x
    return X, col


def full_labels(n, rng, lo=-21, hi=19):
    """Labels with full 53-bit significands, |y| over 2^[lo, hi]: with w = 0, r = -2 y exactly (least squares)."""
    return rng.choice([-1.0, 1.0], n) * np.ldexp(1.0 + rng.random(n), rng.integers(lo, hi + 1, n))


def one_hot_check(g, x, col, r, cnt):
    """The one-hot bounds for row i = (x_i at feature col_i, multiplier r_i): the largest error against
    sum x 2^s (hi + mid + lo) of the scaled split, and against the exact r, both in units of sum |x r| / cnt and divided
    by their limits (ONE_HOT_EXACT, ONE_HOT_R): <= 1 passes."""
    x = np.asarray(x, dtype=np.float64)
    d = g.shape[0]
    s = np.repeat(tile_scales(r), 16)[:len(r)]
    hi, mid, lo = split3(np.ldexp(r, -s))
    pred, exact, S = np.zeros(d), np.zeros(d), np.zeros(d)
    np.add.at(pred, col, np.ldexp(x * hi + x * mid + x * lo, s))
    np.add.at(exact, col, x * r)
    np.add.at(S, col, np.abs(x * r))
    unit = S / cnt                                       # features no row touches must come out exactly 0

    def ratio(ref):
        err = np.abs(g - ref / cnt)
        return np.max(np.where(unit > 0, err / np.where(unit > 0, unit, 1.0), np.where(err == 0, 0.0, np.inf)))
    return ratio(pred) / ONE_HOT_EXACT, ratio(exact) / ONE_HOT_R


def dense_bounds(kind, X, y, w, f32_margins=True, mask=None):
    """Element-wise bounds for a dense shard against the fp64 reference.  Returns (gradient bound per feature, loss bound),
    both already divided by the row count, and the reference (loss, gradient, count) they apply to.
      margin error  eps_i = 2^-20 sum_j |x_ij w_j|   (fp32 margins; 2^-45 of it for fp64 margins)
      |dg_j| <= [sum_i |x_ij| (lambda eps_i + 2^-20 |r_i|) + sum_{i near the hinge kink} |x_ij|] / n
      |dloss| <= sum_i (|r_i| eps_i + lambda eps_i^2 / 2 + [near the kink] eps_i) / n
    Two slack terms cover the fp64 rounding of the reference itself (its margins and its loss sum), not the kernel:
    2^-50 |m_i| is added to eps_i, and 2^-45 sum_i |loss_i| / n to the loss bound."""
    Xd = np.asarray(X, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    sel = np.ones(Xd.shape[0], bool) if mask is None else mask
    Xd, y = Xd[sel], np.asarray(y, dtype=np.float64)[sel]
    m = Xd @ w
    r, loss = row_terms(kind, m, y)
    cnt = Xd.shape[0]
    eps = (EPS_F32_MARGIN if f32_margins else 2.0 ** -45) * (np.abs(Xd) @ np.abs(w)) + 2.0 ** -50 * np.abs(m)
    lam = LAMBDA[kind]
    kink = np.abs(1.0 - (2.0 * y - 1.0) * m) <= eps if kind == "hinge" else np.zeros(cnt, bool)
    A = np.abs(Xd)
    gb = (A.T @ (lam * eps + EPS_PIECES * np.abs(r)) + A[kink].sum(axis=0)) / cnt
    lb = np.sum(np.abs(r) * eps + lam * eps ** 2 / 2 + kink * eps) / cnt + 2.0 ** -45 * np.sum(np.abs(loss)) / cnt
    return gb, lb, (loss.sum() / cnt, Xd.T @ r / cnt, cnt)


def _exp(x):
    try:
        return math.exp(x)
    except OverflowError:
        return math.inf


def _log1p_exp(x):                                       # MLUtils.log1pExp [mllib-1.3.0]
    return x + math.log1p(_exp(-x)) if x > 0 else math.log1p(_exp(x))


def fold_shard(kind, y, w, X=None, csr=None, sample=None):
    """The seqOp fold of applySmooth over one shard as the reference performs it, in fp64 with the oracle's order of
    operations (sequential dot per row, rows folded in order, no FMA): returns (loss sum, row count, gradient sum).
    X: the stored dense rows (fp32, fp64 or bf16 values); csr: (rowptr, idx, val) as stored.  sample: optional
    (seed, thresh, global row ids) for the mini-batch mask; rows it drops are never touched.
    Which rows reach the gradient:
      dense: the axpy is netlib DAXPY, which returns when the multiplier is exactly 0, so such a row adds nothing whatever
             its features are (a hinge row outside the margin has multiplier 0 too);
      CSR:   the sparse axpy has no zero test, so every sampled row adds mult * x (0 * inf = NaN) except a hinge row outside
             the margin, for which HingeGradient never calls axpy."""
    w = np.asarray(w, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    n, d = len(y), len(w)
    if X is not None:
        Xd = np.asarray(X, dtype=np.float64)
        m = np.zeros(n)
        with np.errstate(invalid="ignore", over="ignore"):
            for j in range(d):                           # per row: s += x_j w_j, j ascending
                m = m + Xd[:, j] * w[j]
    else:
        rowptr, idx, val = csr
        val = np.asarray(val, dtype=np.float64)
        m = np.zeros(n)
        for i in range(n):
            s = 0.0
            for k in range(int(rowptr[i]), int(rowptr[i + 1])):
                s += float(val[k]) * float(w[idx[k]])
            m[i] = s
    sel = np.ones(n, bool) if sample is None else row_selected(sample[0], sample[1], sample[2])
    g = np.zeros(d)
    loss, cnt = 0.0, 0
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(n):
            if not sel[i]:
                continue
            mi, yi = float(m[i]), float(y[i])
            call = True
            if kind == "logistic":
                margin = -1.0 * mi
                mult = (1.0 / (1.0 + _exp(margin))) - yi
                li = _log1p_exp(margin) if yi > 0 else _log1p_exp(margin) - margin
            elif kind in ("least_squares", "least_squares_half"):
                diff = mi - yi
                mult, li = (2.0 * diff, diff * diff) if kind == "least_squares" else (diff, diff * diff / 2.0)
            else:
                s = 2 * yi - 1.0
                call = 1.0 > s * mi
                mult, li = (-s, 1.0 - s * mi) if call else (0.0, 0.0)
            if call and X is not None and mult != 0.0:
                g += mult * Xd[i]
            elif call and X is None:
                for k in range(int(rowptr[i]), int(rowptr[i + 1])):
                    g[idx[k]] += mult * float(val[k])
            loss = loss + li
            cnt += 1
    return loss, cnt, g
