"""CPU: the SortTopK restatement the GPU ORDER BY tests compare against (tests/sort_topk_ref.py), with the oracle's
Number::cmp, equals a plain sort by (Number::cmp key, scan position) -- reversed key for DESC -- on values with ties,
+-0.0, +-inf and NaNs of both signs and several payloads."""
import functools
import struct

import numpy as np
import pytest

from oracle import pyoracle as O
from sort_topk_ref import key_cmp, num_key, sort_keyed, sort_topk


def _nan(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


SPECIALS = [0.0, -0.0, np.inf, -np.inf, _nan(0x7FF8000000000000), _nan(0xFFF8000000000000), _nan(0x7FF0000000000001),
            _nan(0xFFFFFFFFFFFFFFFF), 1.0, -1.0, 5e-324, -5e-324]


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("k", [0, 1, 3, 7, 40, 200])
def test_sort_topk_equals_plain_sort(desc, k):
    rng = np.random.default_rng(7 + k)
    vals = list(rng.choice(np.array([0.25, 0.5, 0.75, 1.0, 2.0]), 120))  # many ties
    vals += SPECIALS * 2
    rng.shuffle(vals)
    passes = rng.random(len(vals)) < 0.8
    for p in (None, passes):
        rows, got = sort_topk(vals, k, desc, p)
        er, ev = sort_keyed(vals, k, desc, p)
        assert np.array_equal(rows, er)
        assert np.array_equal(_bits(got), _bits(ev))


def test_num_cmp_agrees_with_the_key():
    for a in SPECIALS:
        for b in SPECIALS:
            assert O.num_cmp(a, b) == key_cmp(a, b), (a, b)


@pytest.mark.parametrize("desc", [False, True])
def test_equal_value_after_a_full_heap_does_not_replace(desc):
    # the heap is full of 1.0s after three rows; later rows equal to the worst kept one must not enter
    vals = [1.0, 1.0, 1.0, 1.0, -0.0, 0.0, 1.0]
    rows, got = sort_topk(vals, 3, desc)
    if desc:
        assert rows.tolist() == [0, 1, 2]
    else:
        assert rows.tolist() == [4, 5, 0]  # -0.0 == 0.0: scan order decides
        assert _bits(got[:1]).tolist() == _bits([-0.0]).tolist()  # the value is the one computed, sign kept


def test_nan_order_reverses_as_a_whole():
    pos, neg = _nan(0x7FF8000000000000), _nan(0xFFF8000000000000)
    vals = [1.0, pos, neg, -1.0]
    asc, _ = sort_topk(vals, 4, False)
    desc, _ = sort_topk(vals, 4, True)
    assert asc.tolist() == [2, 3, 0, 1]   # negative NaN first, positive NaN last
    assert desc.tolist() == [1, 0, 3, 2]  # reversed
    assert functools.cmp_to_key(key_cmp)(neg) < functools.cmp_to_key(key_cmp)(-np.inf)
