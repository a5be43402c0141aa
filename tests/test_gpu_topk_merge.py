"""sdb_topk_merge_device against tests/select_ref.merge, bit for bit: the k-way merge (one warp per query, <= 32 lists)
and the shared-memory sorter (> 32 lists), on per-shard lists built on the host as production builds them -- rows
unique across lists, each list sorted by (Number::cmp key, row) -- with distances that repeat across lists and include
+-0, +-inf and both NaN signs, counts of 0, short, exactly k and above k, and the strides of the all-gather buffer as
well as the packed default."""
import numpy as np
import pytest

import select_ref as R

pytestmark = pytest.mark.gpu

GEN_NAN = np.uint64(0xFFF8000000000000).view(np.float64)
DATA_NAN = np.uint64(0x7FF8000000000000).view(np.float64)
POOL = np.array([GEN_NAN, -np.inf, -2.5, -1.0, -0.0, 0.0, 5e-324, 1.0, 2.5, np.inf, DATA_NAN])
SORTER_LIMIT = 8192  # n_lists * k entries: 24 bytes each in the sorter's shared memory, at most 200 KB


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_lists(rng, n_lists, nq, k):
    """-> rows (n_lists, nq, k) u64, dist (n_lists, nq, k) f64, counts (n_lists, nq) u32"""
    dist = POOL[rng.integers(0, POOL.size, (n_lists, nq, k))]
    rows = np.empty((n_lists, nq, k), np.uint64)
    for q in range(nq):  # disjoint shards: a row appears in one list only
        rows[:, q, :] = rng.permutation(4 * n_lists * k)[: n_lists * k].reshape(n_lists, k)
    o = np.argsort(rows, axis=-1, kind="stable")  # each list in (key, row) order
    rows, dist = np.take_along_axis(rows, o, -1), np.take_along_axis(dist, o, -1)
    o = np.argsort(R.num_key(dist.ravel()).reshape(dist.shape), axis=-1, kind="stable")
    rows, dist = np.take_along_axis(rows, o, -1), np.take_along_axis(dist, o, -1)
    kind = rng.integers(0, 4, (n_lists, nq))  # 0, short, exactly k, above k
    counts = np.where(kind == 0, 0, np.where(kind == 1, rng.integers(0, k + 1, (n_lists, nq)),
                                             np.where(kind == 2, k, k + rng.integers(1, 5, (n_lists, nq)))))
    counts[:, 0] = rng.integers(0, 2, n_lists)  # fewer than k entries in all (n_lists < k), or none
    if nq > 1:
        counts[:, 1] = 0
    return rows, dist, counts.astype(np.uint32)


def run_merge(ctx, rows, dist, counts, k, gathered):
    """the lists packed (default strides) or laid out as the all-gather buffer (shard_block_layout strides)"""
    import torch
    from surrealdb_b200.engine import shard_block_layout, topk_merge_device
    n_lists, nq = counts.shape
    dev = torch.device("cuda", 0)
    if gathered:
        off_rows, off_dist, off_cnt, blk = shard_block_layout(nq, k)
        buf = np.zeros((n_lists, blk), np.uint8)
        for l in range(n_lists):
            buf[l, off_rows:off_dist] = rows[l].reshape(-1).view(np.uint8)
            buf[l, off_dist:off_cnt] = dist[l].reshape(-1).view(np.uint8)
            buf[l, off_cnt:off_cnt + 4 * nq] = counts[l].view(np.uint8)
        g = torch.from_numpy(buf.reshape(-1)).to(dev)
        p = g.data_ptr()
        args = (p + off_rows, p + off_dist, p + off_cnt)
        strides = dict(stride_rows=blk // 8, stride_dist=blk // 8, stride_counts=blk // 4)
        keep = [g]
    else:
        tr = torch.from_numpy(rows.view(np.int64).copy()).to(dev)
        td = torch.from_numpy(dist.copy()).to(dev)
        tc = torch.from_numpy(counts.view(np.int32).copy()).to(dev)
        args = (tr.data_ptr(), td.data_ptr(), tc.data_ptr())
        strides = {}
        keep = [tr, td, tc]
    o_rows = torch.full((nq, k), -1, dtype=torch.int64, device=dev)
    o_dist = torch.full((nq, k), -7.0, dtype=torch.float64, device=dev)
    o_cnt = torch.full((nq,), -1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()  # torch's stream and the library's are not ordered with each other
    topk_merge_device(ctx, n_lists, nq, k, *args, o_rows.data_ptr(), o_dist.data_ptr(), o_cnt.data_ptr(), **strides)
    del keep
    return o_rows.cpu().numpy().view(np.uint64), o_dist.cpu().numpy(), o_cnt.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("k", [1, 7, 100, 256])
@pytest.mark.parametrize("n_lists", [1, 2, 31, 32, 33, 64, 100])
def test_merge_matches_reference(ctx, n_lists, k):
    from surrealdb_b200._lib import SDB_EUNSUPPORTED, SdbError
    rng = np.random.default_rng(n_lists * 1000 + k)
    for nq in (1, 5, 1027):
        rows, dist, counts = make_lists(rng, n_lists, nq, k)
        if n_lists > 32 and n_lists * k > SORTER_LIMIT:
            for gathered in (False, True):
                with pytest.raises(SdbError) as e:
                    run_merge(ctx, rows, dist, counts, k, gathered)
                assert e.value.status == SDB_EUNSUPPORTED
            continue
        want_rows, want_dist, want_cnt = R.merge(rows, dist, counts, k)
        for gathered in (False, True):
            got_rows, got_dist, got_cnt = run_merge(ctx, rows, dist, counts, k, gathered)
            assert got_cnt.tolist() == want_cnt.tolist(), (nq, gathered)
            for q in range(nq):
                c = int(want_cnt[q])
                assert got_rows[q, :c].tolist() == want_rows[q, :c].tolist(), (nq, gathered, q)
                assert got_dist[q, :c].view(np.uint64).tolist() == want_dist[q, :c].view(np.uint64).tolist(), \
                    (nq, gathered, q)

