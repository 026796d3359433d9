"""Pure-Python restatement of views (include/agd_b200.h, agd_set_row_filter): the per-row draw, the bound mapping and the
predicate, for the tests to check the device's mask and the views' rows against.  Standard library and numpy only."""
import math
from fractions import Fraction

import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF
VIEW_STREAM = 7


def philox4x32_10(ctr, key):
    c, k = list(ctr), list(key)
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & MASK, p1 & MASK, ((p0 >> 32) ^ c[3] ^ k[1]) & MASK, p0 & MASK]
        k = [(k[0] + W0) & MASK, (k[1] + W1) & MASK]
    return c


def row_draw(seed: int, grow: int, stream: int = VIEW_STREAM) -> int:
    """u(seed, grow): Philox4x32-10, key = seed, counter (grow lo, grow hi, 0, stream); words 0 and 1 as one 64-bit value."""
    c = philox4x32_10([grow & MASK, (grow >> 32) & MASK, 0, stream], [seed & MASK, (seed >> 32) & MASK])
    return (c[0] << 32) | c[1]


def bound(c: float) -> int:
    """b = floor(c * 2^64), exactly (c = 1 gives 2^64: 'to the end')."""
    return math.floor(Fraction(c) * (1 << 64))


def predicate(u: int, seed_lo_hi_comp) -> bool:
    _, lo, hi, comp = seed_lo_hi_comp
    inside = bound(lo) <= u < bound(hi)
    return inside != bool(comp)


def view_mask(preds, row_base: int, rows: int) -> np.ndarray:
    """Which rows row_base + [0, rows) every predicate (seed, lo, hi, complement) keeps."""
    out = np.ones(rows, dtype=bool)
    for p in preds:
        out &= np.array([predicate(row_draw(p[0], row_base + r), p) for r in range(rows)], dtype=bool)
    return out
