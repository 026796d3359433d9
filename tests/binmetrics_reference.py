"""An independent numpy restatement of BinaryClassificationMetrics' curve (not a test module itself): the descending-order
key of a margin, the curve of distinct margins with cumulative counts, and the trapezoid areas summed with math.fsum."""
import math

import numpy as np

SIGN = np.uint64(1 << 63)


def margin_key(m):
    """Unsigned keys whose ascending order is the descending order of the (non-NaN) margins; -0 and +0 share a key."""
    m = np.asarray(m, dtype=np.float64)
    u = np.where(m == 0.0, 0.0, m).view(np.uint64)
    asc = np.where((u >> np.uint64(63)) == 1, ~u, u | SIGN)
    return ~asc


def margin_of_key(k):
    asc = ~np.asarray(k, dtype=np.uint64)
    u = np.where((asc >> np.uint64(63)) == 1, asc & ~SIGN, ~asc)
    return u.view(np.float64)


def curve(m, y):
    """(margins descending, cumulative tp, cumulative fp, NaN count) of the rows with margins m and labels y."""
    m = np.asarray(m, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    nan = np.isnan(m)
    k = margin_key(m[~nan])
    pos = (y[~nan] > 0.5).astype(np.int64)
    order = np.argsort(k, kind="stable")
    ks, ps = k[order], pos[order]
    uniq, start = np.unique(ks, return_index=True)
    ends = np.append(start[1:], ks.shape[0]).astype(np.int64)
    ctp = np.cumsum(ps)[ends - 1] if ks.shape[0] else np.zeros(0, dtype=np.int64)
    cfp = ends - ctp
    return margin_of_key(uniq), ctp.astype(np.int64), cfp.astype(np.int64), int(nan.sum())


def _trapezoid_fsum(x, y):
    return math.fsum(((x[i + 1] - x[i]) * (y[i + 1] + y[i]) / 2.0) for i in range(len(x) - 1))


def areas(tp, fp):
    """(areaUnderROC, areaUnderPR) of a curve, fsum over the same points: ROC (0,0) .. (1,1), PR from (0,1)."""
    if len(tp) == 0:
        return float("nan"), float("nan")
    P, N = float(tp[-1]), float(fp[-1])
    tpd, fpd = np.asarray(tp, dtype=np.float64), np.asarray(fp, dtype=np.float64)
    auroc = float("nan")
    if P > 0 and N > 0:
        auroc = _trapezoid_fsum([0.0] + list(fpd / N) + [1.0], [0.0] + list(tpd / P) + [1.0])
    aupr = float("nan")
    if P > 0:
        aupr = _trapezoid_fsum([0.0] + list(tpd / P), [1.0] + list(tpd / (tpd + fpd)))
    return auroc, aupr
