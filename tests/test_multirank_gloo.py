"""N>1 host-side protocol on CPU (gloo, world_size 2): row sharding, the single packed all-gather of the
per-shard top-k blocks, and the (distance, global row) merge rule must reproduce the unsharded oracle result.
The CUDA side of the same protocol (sdb_topk_merge_device) is covered by tests/test_gpu_multi.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import pyoracle as O
from select_ref import merge
from surrealdb_b200.engine import shard_block_layout
from surrealdb_b200.sharding import shard_range
from surrealdb_b200.synthetic import gen_f32

ROWS, DIM, NQ, K = 3000, 24, 5, 7


def merge_reference(blocks, nq, k):
    """sdb_topk_merge_device over the gathered blocks (tests/select_ref.merge): order by (Number::cmp key, global
    row), first k"""
    off_rows, off_dist, off_cnt, blk = shard_block_layout(nq, k)
    rows = np.stack([b[off_rows:off_dist].view(np.uint64).reshape(nq, k) for b in blocks])
    dst = np.stack([b[off_dist:off_cnt].view(np.float64).reshape(nq, k) for b in blocks])
    cnt = np.stack([b[off_cnt:off_cnt + 4 * nq].view(np.uint32) for b in blocks])
    r, d, c = merge(rows, dst, cnt, k)
    return [[(float(d[q, j]), int(r[q, j])) for j in range(int(c[q]))] for q in range(nq)]


def worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    corpus = gen_f32(5, 0, ROWS * DIM).reshape(ROWS, DIM)
    queries = gen_f32(6, 0, NQ * DIM).reshape(NQ, DIM).astype(np.float64)
    base, n_local = shard_range(ROWS, world, rank)
    off_rows, off_dist, off_cnt, blk = shard_block_layout(NQ, K)
    block = np.zeros(blk, np.uint8)
    for i in range(NQ):  # the per-shard exact top-k (what sdb_knn_bruteforce_device(row_base=base) produces)
        r, d = O.knn_topk(corpus[base:base + n_local], queries[i], "cosine", K)
        block[off_rows:off_dist].view(np.uint64).reshape(NQ, K)[i, : r.size] = r + base
        block[off_dist:off_cnt].view(np.float64).reshape(NQ, K)[i, : r.size] = d
        block[off_cnt:off_cnt + 4 * NQ].view(np.uint32)[i] = r.size
    gathered = torch.zeros(world * blk, dtype=torch.uint8)
    dist.all_gather_into_tensor(gathered, torch.from_numpy(block))  # ONE collective
    merged = merge_reference([gathered.numpy()[i * blk:(i + 1) * blk] for i in range(world)], NQ, K)
    if rank == 0:
        q.put(merged)
    dist.barrier()
    dist.destroy_process_group()


def test_shard_ranges_partition_the_corpus():
    for rows in (0, 1, 255, 256, 257, 3000, 10_000_000):
        for world in (1, 2, 3, 4, 8):
            cover = []
            for r in range(world):
                b, n = shard_range(rows, world, r)
                assert b % 256 == 0 or n == 0
                cover.append((b, n))
            assert sum(n for _, n in cover) == rows
            pos = 0
            for b, n in cover:
                if n:
                    assert b == pos
                    pos += n


def test_two_rank_allgather_merge_equals_unsharded_oracle():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    merged = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    corpus = gen_f32(5, 0, ROWS * DIM).reshape(ROWS, DIM)
    queries = gen_f32(6, 0, NQ * DIM).reshape(NQ, DIM).astype(np.float64)
    for i in range(NQ):
        r, d = O.knn_topk(corpus, queries[i], "cosine", K)
        assert [e[1] for e in merged[i]] == list(r)
        assert [e[0] for e in merged[i]] == list(d)


def test_numpy_generator_matches_oracle_generator():
    a = O.gen_f32(0x5DB00002, 123456789012, 50000)
    b = gen_f32(0x5DB00002, 123456789012, 50000)
    assert a.tobytes() == b.tobytes()


# ---- sharded graph expansion (graph.cu, round 2): the collective protocol of one hop, restated with gloo ---------------
G_NODES, G_EDGES, G_LIMIT = 400, 3000, 5


def _rmat_csr(seed):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, G_NODES, G_EDGES)
    dst = rng.integers(0, G_NODES, G_EDGES)
    key = np.unique(src.astype(np.int64) * G_NODES + dst)  # (src, dst) order = edge-key order of the KV range
    src, dst = key // G_NODES, key % G_NODES
    row_ptr = np.zeros(G_NODES + 1, np.uint64)
    row_ptr[1:] = np.cumsum(np.bincount(src, minlength=G_NODES))
    return row_ptr, dst.astype(np.uint32)


def graph_worker(rank, world, port, q):
    """One hop as hop_device does it on a 1-D source-range shard: (1) degree of every frontier element this rank owns
    (0 for the others), all-reduce(sum) -> the global degree array; (2) exclusive scan -> the position of every source's
    neighbours in the level; (3) this rank writes its sources' neighbours into a ZERO-filled level; (4) all-reduce(sum)
    assembles the level.  Order and duplicates must equal the unsharded per-source scans."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    row_ptr, col_idx = _rmat_csr(11)
    lo, hi = (0, G_NODES // 3) if rank == 0 else (G_NODES // 3, G_NODES)  # deliberately uneven ranges
    rp_local = row_ptr[lo:hi + 1] - row_ptr[lo]
    ci_local = col_idx[int(row_ptr[lo]):int(row_ptr[hi])]
    rng = np.random.default_rng(5)
    frontier = rng.integers(0, G_NODES, 64).astype(np.uint32)  # duplicates on purpose: LookupPart keeps them
    levels = []
    for _hop in range(3):
        deg = np.zeros(frontier.size, np.int64)
        mine = (frontier >= lo) & (frontier < hi)
        d = (rp_local[frontier[mine] - lo + 1] - rp_local[frontier[mine] - lo]).astype(np.int64)
        deg[mine] = np.minimum(d, G_LIMIT) if G_LIMIT else d
        t = torch.from_numpy(deg)
        dist.all_reduce(t)  # (1)
        offs = np.concatenate([[0], np.cumsum(t.numpy())])  # (2)
        level = np.zeros(int(offs[-1]), np.int64)
        for i in np.nonzero(mine)[0]:  # (3)
            s = int(frontier[i]) - lo
            nb = ci_local[int(rp_local[s]):int(rp_local[s]) + int(deg[i])]
            level[offs[i]:offs[i] + nb.size] = nb
        t2 = torch.from_numpy(level)
        dist.all_reduce(t2)  # (4)
        frontier = t2.numpy().astype(np.uint32)
        levels.append(frontier.copy())
    if rank == 0:
        q.put(levels)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_graph_hop_protocol_equals_unsharded_oracle():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=graph_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    levels = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    row_ptr, col_idx = _rmat_csr(11)
    frontier = np.random.default_rng(5).integers(0, G_NODES, 64).astype(np.uint32)
    for h in range(3):
        frontier = O.graph_hop(row_ptr, col_idx, frontier, G_LIMIT)
        assert levels[h].tolist() == frontier.tolist(), h
