"""pack_row_filter: the bitmap layout of the filtered KNN calls (bit r = bit r % 32 of word r // 32), checked against
numpy's little-endian bit packing.  No GPU needed."""
import numpy as np
import pytest

from surrealdb_b200.engine import pack_row_filter


def reference(mask):
    n = mask.shape[-1]
    words = (n + 31) // 32
    padded = np.zeros(mask.shape[:-1] + (words * 32,), bool)
    padded[..., :n] = mask
    return np.packbits(padded, axis=-1, bitorder="little").view(np.uint32)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 1000, 4097])
def test_single_mask_matches_packbits(n):
    rng = np.random.default_rng(n)
    m = rng.random(n) < 0.37
    got = pack_row_filter(m)
    assert got.dtype == np.uint32 and got.shape == ((n + 31) // 32,)
    assert np.array_equal(got, reference(m))
    for r in rng.integers(0, n, 20):  # the documented bit position of every row
        assert bool((got[r // 32] >> (r % 32)) & 1) == bool(m[r])


def test_stack_of_masks_and_edges():
    rng = np.random.default_rng(5)
    m = rng.random((7, 301)) < 0.5
    got = pack_row_filter(m)
    assert got.shape == (7, 10) and np.array_equal(got, reference(m))
    assert not pack_row_filter(np.zeros(70, bool)).any()
    full = pack_row_filter(np.ones(70, bool))
    assert list(full) == [0xFFFFFFFF, 0xFFFFFFFF, 0x3F]  # padding bits of the last word stay clear
    assert pack_row_filter([True, False, True]).tolist() == [5]
