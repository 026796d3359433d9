"""Views without a GPU: the pure-Python restatement of the per-row draw is pinned to the Random123 known answers, the bound
mapping is checked at its edges, and the Python layer's split arithmetic and argument checks are exercised (views are
created on the host; nothing here runs a kernel)."""
import math
from fractions import Fraction

import numpy as np
import pytest

from view_reference import bound, philox4x32_10, predicate, row_draw


def test_philox_known_answers():
    # Random123 kat_vectors, philox4x32 with 10 rounds
    M = 0xFFFFFFFF
    assert philox4x32_10([0, 0, 0, 0], [0, 0]) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert philox4x32_10([M] * 4, [M] * 2) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert philox4x32_10([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0]) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_draw_layout():
    """The draw is words 0 and 1 of the block at counter (grow lo, grow hi, 0, 7) under key (seed lo, seed hi)."""
    seed, grow = 0x0123456789ABCDEF, (5 << 40) + 17
    c = philox4x32_10([grow & 0xFFFFFFFF, grow >> 32, 0, 7], [seed & 0xFFFFFFFF, seed >> 32])
    assert row_draw(seed, grow) == (c[0] << 32) | c[1]
    assert row_draw(seed, grow) != row_draw(seed, grow, stream=6)    # not the mini-batch mask's stream


def test_bound_mapping_edges():
    assert bound(0.0) == 0
    assert bound(1.0) == 1 << 64                                     # "to the end": above every 64-bit draw
    below_one = math.nextafter(1.0, 0.0)                             # 1 - 2^-53
    assert bound(below_one) == (1 << 64) - (1 << 11)
    assert predicate((1 << 64) - 1, (0, 0.0, 1.0, False))            # the largest draw is inside [0, 1)
    assert not predicate((1 << 64) - 1, (0, 0.0, below_one, False))
    assert not predicate(0, (0, 1.0, 1.0, False)) and predicate(0, (0, 1.0, 1.0, True))
    for c in (0.1, 0.2, 1.0 / 3.0, 0.6, 5e-324, 1e-300, 2.0 ** -70 * 3):
        b = bound(c)
        exact = Fraction(c) * (1 << 64)
        assert b <= exact < b + 1                                    # floor, also where c 2^64 is not an integer
        assert b == int(np.ldexp(c, 64)) if c >= 2.0 ** -11 else True  # ldexp is exact where the product is an integer
    assert bound(5e-324) == 0 and bound(2.0 ** -70 * 3) == 0


def test_split_bounds(agd):
    b = agd.split_bounds([0.6, 0.3, 0.1])
    assert b[0] == 0.0 and b[-1] == 1.0 and len(b) == 4
    assert b[1] == 0.6 / 1.0 and b[2] == 0.6 + 0.3                    # scanLeft in fp64
    assert agd.split_bounds([2, 2]) == [0.0, 0.5, 1.0]
    assert agd.split_bounds([1, 0, 1]) == [0.0, 0.5, 0.5, 1.0]         # a zero weight is an empty split
    b = agd.split_bounds([1e-300, 3.0, 7.0])
    assert all(x <= y for x, y in zip(b, b[1:])) and b[-1] == 1.0
    for bad in ([], [-1.0, 2.0], [0.0, 0.0], [float("nan"), 1.0], [float("inf"), 1.0]):
        with pytest.raises(ValueError):
            agd.split_bounds(bad)


def _host_view(agd):
    """A DeviceDataset shell with no handle: enough for the view arithmetic, which never reaches the library."""
    ds = object.__new__(agd.DeviceDataset)
    ds.ctx, ds.h, ds.total_rows, ds._xchg_d, ds._base, ds._preds = None, None, 7, 0, None, ()
    return ds


def test_random_split_structure(agd):
    ds = _host_view(agd)
    parts = ds.randomSplit([0.6, 0.3, 0.1], seed=9)
    assert [p._preds for p in parts] == [((9, 0.0, 0.6, False),), ((9, 0.6, 0.8999999999999999, False),),
                                         ((9, 0.8999999999999999, 1.0, False),)]
    assert all(p.is_view and p._base is ds and p.total_rows == 7 for p in parts)
    assert ds.randomSplit([1, 1])[0]._preds[0][0] == agd.DEFAULT_SPLIT_SEED
    with pytest.raises(ValueError):
        ds.randomSplit([0.0])


def test_sample_and_kfold_structure(agd):
    ds = _host_view(agd)
    assert ds.sample(False, 0.25, seed=3)._preds == ((3, 0.0, 0.25, False),)
    with pytest.raises(NotImplementedError):
        ds.sample(True, 0.5)
    with pytest.raises(ValueError):
        ds.sample(False, 1.5)
    folds = agd.MLUtils.kFold(ds, 3, seed=11)
    assert len(folds) == 3
    for i, (train, valid) in enumerate(folds):
        assert valid._preds == ((11, i / 3, (i + 1) / 3, False),)
        assert train._preds == ((11, i / 3, (i + 1) / 3, True),)
    assert folds[-1][1]._preds[0][2] == 1.0
    for k in (1, 0, -2):
        with pytest.raises(ValueError):
            agd.MLUtils.kFold(ds, k)


def test_views_compose_up_to_four(agd):
    ds = _host_view(agd)
    v = ds
    for level in range(4):
        v = v.sample(False, 0.9, seed=level)
        assert len(v._preds) == level + 1 and v._base is ds      # every level keeps the owner of the shards alive
    with pytest.raises(ValueError, match="at most 4"):
        v.sample(False, 0.5)
    with pytest.raises(ValueError, match="at most 4"):
        agd.MLUtils.kFold(v, 2)
    train, _ = agd.MLUtils.kFold(ds.randomSplit([0.8, 0.2])[0], 5)[0]
    assert len(train._preds) == 2


def test_view_close_frees_nothing_and_refuses_loads(agd):
    ds = _host_view(agd)
    v = ds.sample(False, 0.5)
    v.close()
    assert v.h is None and ds.h is None       # the shell has no handle; close() on the view did not touch the parent
    with pytest.raises(ValueError, match="view"):
        v.load_dense([0.0], [[1.0]])
    with pytest.raises(ValueError, match="view"):
        v.unpersist()
