"""The GPU HNSW builder's three kernels at production shapes, each against a CPU reference on sampled elements of a
full-size launch (more elements or queries than the device holds warps, so that warps loop):

  sdb_hnsw_select_device (hnsw_select_typed_kernel)   vs tests/hnsw_select_ref.select, restated on precomputed
                                                       distances: kc past 32 (a second e_dist chunk, a visiting-order
                                                       rank over more than 32 entries), more than 32 accepted
                                                       neighbours, the element absent / first / inside / twice,
                                                       duplicate ids and rows, both addressings
  sdb_hnsw_knn_exact_device (hnsw_knn_exact_kernel)    vs hnsw_select_ref.knn: wide rows, k around 32 and 256, member
                                                       sets around 32 and 10^4, a crowd of equal rows cut at the k-th
                                                       place by id
  sdb_hnsw_select_neighbors[_ids] (hnsw_select_kernel) vs tests/select_f32_ref.select (the kernel's own f32
                                                       arithmetic), with zero, NaN, infinite, overflowing and duplicate
                                                       rows; picks are compared where every comparison was decided
                                                       within rsqrtf's error

plus the shared-memory limits of the three launches and both F32 builders on degenerate data."""
import ctypes as C

import numpy as np
import pytest

import hnsw_select_ref as S
import hnsw_types_ref as R
import select_f32_ref as F
from test_gpu_hnsw_build import TYPES, METRICS, check_structure, clustered, dev, index, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def gen(rng, metric, vt, shape):
    """spread data: normal floats; integers in [-60, 60] (I16: [-6, 6], so that its cosine dot does not wrap); Hamming
    and Jaccard small alphabets"""
    if metric == "hamming":
        v = rng.integers(0, 3, shape).astype(np.float64)
    elif metric == "jaccard":
        v = rng.integers(0, 40, shape).astype(np.float64)
    elif vt[0] == "I":
        v = rng.integers(-6 if vt == "I16" else -60, 7 if vt == "I16" else 61, shape).astype(np.float64)
    else:
        v = rng.normal(0, 1, shape)
    return v.astype(R.DTYPES[vt])


# ---- a. sdb_hnsw_select_device --------------------------------------------------------------------------------------

def ref_select(metric, vt, X, elem, cand, m_max, presorted):
    """hnsw_select_ref.select with the distances of one call per visited candidate (every metric but JACCARD is
    symmetric in the reference's arithmetic, bit for bit)"""
    cand = [int(c) for c in cand]
    real = [j for j, c in enumerate(cand) if c != elem]
    take_all = len(real) <= m_max
    rows = np.array(cand, np.int64)
    e_dist = {}
    if not (presorted and take_all) and real:
        if presorted or metric != "jaccard":
            d = S.distances(metric, X[rows], X[elem], 2.5, vt)
        else:
            d = np.array([R.distance(metric, X[elem], X[c], 2.5, vt) for c in cand])
        e_dist = {j: d[j] for j in real}
    visit = real if presorted else sorted(real, key=lambda j: (S.key(e_dist[j]), j))
    acc = []
    for j in visit:
        if len(acc) >= m_max:
            break
        e = cand[j]
        if not take_all and acc:
            rd = S.distances(metric, X[np.array(acc)], X[e], 2.5, vt)
            if any(e_dist[j] > r for r in rd):
                continue
        acc.append(e)
    return acc


def cand_lists(rng, n_rows, elems, kc):
    """kc-wide lists: full or short, the element absent, first, inside or twice; a duplicate id in every fifth"""
    n = elems.size
    cand = rng.integers(0, n_rows, (n, kc)).astype(np.int64)
    cnt = np.where(rng.random(n) < 0.7, kc, rng.integers(1, kc + 1, n)).astype(np.int32)
    where = np.arange(n) % 4
    for i in range(n):
        c = int(cnt[i])
        if where[i] == 1:
            cand[i, 0] = elems[i]
        elif where[i] == 2:
            cand[i, c // 2] = elems[i]
        elif where[i] == 3 and c >= 3:
            cand[i, 1], cand[i, c - 1] = elems[i], elems[i]
        if i % 5 == 0 and c >= 4:
            cand[i, c - 2] = cand[i, 2]
    return cand, cnt


def run_select(ctx, metric, vt, dim, kc, m_max, n, samples, seed):
    import torch
    from surrealdb_b200.hnsw_build import select
    rng = np.random.default_rng(seed)
    n_rows = n + 64
    X = gen(rng, metric, vt, (n_rows, dim))
    X[n_rows - 8 : n_rows] = X[n_rows - 16 : n_rows - 8]  # duplicate rows: exact ties
    elems = rng.permutation(n_rows)[:n]
    cand, cnt = cand_lists(rng, n_rows, elems, kc)
    cand[: n // 8, -16:] = np.arange(n_rows - 16, n_rows)  # the twins in the same list
    # hubs: an element at the mean of its candidates lies nearer to each of them than they lie to each other, so
    # its selection accepts up to m_max of them (the acceptance loop then runs over more than 32 neighbours)
    hubs = np.arange(n // 2, n // 2 + 64)
    if kc >= 48:  # a twin pair at positions 36 and 45: the second can only be rejected by the 37th accepted neighbour
        cnt[hubs] = kc
        cand[hubs, 36] = n_rows - 16 + hubs % 8
        cand[hubs, 45] = n_rows - 8 + hubs % 8
    mean = np.stack([X[cand[i, : cnt[i]]].astype(np.float64).mean(0) for i in hubs])
    if vt[0] == "I":  # rounded and scaled up, and never a zero row (a NaN cosine distance has no pinned rank)
        mean = np.rint(4 * mean)
        mean[:, 0] += (mean == 0).all(1)
    X[elems[hubs]] = mean.astype(X.dtype)
    pick = np.concatenate([rng.choice(n, samples, replace=False), hubs[:2]])
    idx = index(ctx, X, metric, vt, 2.5)
    try:
        most = 0
        for presorted in (1, 0):
            out, oc = select(idx.h, dev(cand), dev(cnt), m_max, presorted, elem_ids=dev(elems.astype(np.int32)))
            out, oc = out.cpu().numpy(), oc.cpu().numpy()
            most = max(most, int(oc.max()))
            for i in pick:
                want = ref_select(metric, vt, X, int(elems[i]), cand[i, : cnt[i]], m_max, presorted)
                assert list(out[i, : oc[i]]) == want, (metric, vt, dim, kc, m_max, presorted, int(i))
        # row0 addressing picks what the explicit ids pick
        o1, c1 = select(idx.h, dev(cand), dev(cnt), m_max, 0, row0=64)
        o2, c2 = select(idx.h, dev(cand), dev(cnt), m_max, 0, elem_ids=dev(np.arange(64, 64 + n, dtype=np.int32)))
        assert torch.equal(c1, c2) and torch.equal(o1, o2)
        return most
    finally:
        idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vt", TYPES)
def test_select_typed_production_shape(ctx, vt, metric):
    dim = 256 if vt == "I16" else 768
    kc, m_max = (64, 33) if metric == "jaccard" else (151, 64)
    samples = 2 if metric == "jaccard" else 5
    # 17000 elements: more than 4x the resident warps of every cell (at most 32 warps on each of 132 SMs)
    most = run_select(ctx, metric, vt, dim, kc, m_max, 17000, samples, 300 + 7 * METRICS.index(metric) + TYPES.index(vt))
    if metric in ("cosine", "euclidean", "manhattan", "minkowski"):
        assert most > 32, most  # the acceptance test ran against more than 32 accepted neighbours


@pytest.mark.parametrize("kc,m_max", [(33, 32), (64, 33), (128, 64), (256, 32)])
@pytest.mark.parametrize("metric", ["euclidean", "cosine", "jaccard"])
@pytest.mark.parametrize("vt", ["F32", "F64"])
def test_select_typed_dimension_ladder(ctx, vt, metric, kc, m_max):
    cw = 256 // np.dtype(R.DTYPES[vt]).itemsize  # the column step of the type
    dims = [cw - 1, cw, cw + 1, 2 * cw - 1, 2 * cw, 2 * cw + 1]
    for d, dim in enumerate(dims):
        samples = 1 if metric == "jaccard" else 3
        run_select(ctx, metric, vt, dim, min(kc, 40) if metric == "jaccard" else kc, m_max, 9000, samples,
                   900 + d + 11 * kc + m_max)


# ---- b. sdb_hnsw_knn_exact_device -----------------------------------------------------------------------------------

def ref_knn(metric, vt, X, q, k, members, d_all=None):
    """hnsw_select_ref.knn, vectorised: lexsort on (NaN last, total-order key, id); d_all: the distances of q to every
    row, when known"""
    ids = np.sort(np.asarray(members, np.int64))
    d = S.distances(metric, X[ids], q, 2.5, vt) if d_all is None else d_all[ids]
    b = d.view(np.int64)
    key = np.where(b < 0, ~b, b | np.int64(-0x8000000000000000))  # walk_key as a signed order
    key = key ^ np.int64(-0x8000000000000000)
    o = np.lexsort((ids, key, np.isnan(d)))[:k]
    return ids[o], d[o]


@pytest.mark.parametrize("vt,dim", [("F32", 768), ("F32", 1536), ("F64", 768), ("F64", 1536), ("I16", 2048)])
def test_knn_exact_production_shape(ctx, vt, dim):
    from surrealdb_b200.hnsw_build import knn_exact
    metric = "euclidean"
    rng = np.random.default_rng(40 + dim + len(vt))
    n, nq = 12000, 6000
    X = gen(rng, metric, vt, (n, dim))
    crowd = rng.choice(n, 40, replace=False)  # equal rows with scattered ids
    X[crowd] = X[crowd[0]]
    Q = gen(rng, metric, vt, (nq, dim))
    Q[::3] = X[crowd[0]]  # the crowd at distance 0: ranks 0..39, cut at k = 31, 32, 33 by id
    Q[1::3] = X[rng.integers(0, n, Q[1::3].shape[0])]
    idx = index(ctx, X, metric, vt)
    try:
        big = rng.permutation(n)[:10007]
        big = np.unique(np.concatenate([big, crowd]))
        rng.shuffle(big)
        sets = [None, big, rng.permutation(n)[:1]] + [np.concatenate([crowd[:s // 2], rng.permutation(n)[: s - s // 2]])
                                                    for s in (31, 32, 33)]
        pick = np.concatenate([rng.choice(nq, 4, replace=False), [0, 3]])
        d_all = {int(q): S.distances(metric, X, Q[q], 2.5, vt) for q in pick}
        for mem in sets:
            if mem is not None:
                mem = np.unique(mem)
                rng.shuffle(mem)
            for k in (1, 31, 32, 33, 255, 256):
                if mem is not None and mem.size < 100 and k not in (1, 32, 33, 256):
                    continue
                ids, dist, cnt = knn_exact(idx.h, dev(Q), k, None if mem is None else dev(mem.astype(np.int32)))
                ids, dist, cnt = ids.cpu().numpy(), dist.cpu().numpy(), cnt.cpu().numpy()
                members = np.arange(n) if mem is None else mem
                for q in pick:
                    wi, wd = ref_knn(metric, vt, X, Q[q], k, members, d_all[int(q)])
                    assert cnt[q] == wi.size, (vt, dim, k, q)
                    assert list(ids[q, : cnt[q]]) == list(wi), (vt, dim, k, q, None if mem is None else mem.size)
                    assert all(same(metric, a, b) for a, b in zip(dist[q, : cnt[q]], wd)), (vt, dim, k, q)
    finally:
        idx.close()


# ---- c. sdb_hnsw_select_neighbors[_ids] -----------------------------------------------------------------------------

def f32_data(rng, n, dim, cosine, equal_norms=False):
    """normal rows with degenerate ones: zero rows, NaN and +-inf elements, values whose squared distance overflows,
    duplicate rows.  equal_norms: every row is one vector with random signs, so that every norm, every product under
    the rsqrtf and so every r is the same and the long lists stay decidable (one-dimensional cosine rows: +-1)"""
    X = rng.normal(0, 1, (n, dim)).astype(np.float32)
    if dim == 1 and cosine:
        X = np.where(X < 0, -1.0, 1.0).astype(np.float32)  # dot * r exact: the fused and unfused distances agree
    elif equal_norms:
        X = (X[0] * np.where(rng.random((n, dim)) < 0.5, -1, 1)).astype(np.float32)
    X[:6] = 0.0
    X[6:9, 0] = np.nan
    X[9, -1] = np.inf
    X[10, 0] = -np.inf
    if not cosine:
        X[11:14] *= np.float32(3e19)  # (3e19)^2 overflows f32
    X[20:40] = X[40:60]
    return X


def f32_select(ctx, X, metric, cand, cnt, kc, m_max, presorted, elems=None, row0=0):
    import torch
    from surrealdb_b200 import _lib as L
    n = cand.shape[0]
    x = dev(X)
    cd, cn = dev(cand.astype(np.int64)), dev(cnt.astype(np.int32))
    out = torch.zeros((n, m_max), dtype=torch.int32, device="cuda")
    oc = torch.zeros((n,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    args = (C.c_void_p(cd.data_ptr()), C.c_void_p(cn.data_ptr()), kc, m_max, presorted, C.c_void_p(out.data_ptr()),
            C.c_void_p(oc.data_ptr()))
    if elems is None:
        rc = L.lib().sdb_hnsw_select_neighbors(ctx.h, C.c_void_p(x.data_ptr()), X.shape[1], L.METRIC[metric], row0, n,
                                               *args)
    else:
        ids = dev(elems.astype(np.int32))
        rc = L.lib().sdb_hnsw_select_neighbors_ids(ctx.h, C.c_void_p(x.data_ptr()), X.shape[1], L.METRIC[metric],
                                                   C.c_void_p(ids.data_ptr()), n, *args)
    L.check(rc)
    return out.cpu().numpy(), oc.cpu().numpy()


F32_CASES = [(1, 7, 3), (1, 64, 6), (31, 256, 64), (31, 33, 32), (32, 128, 1), (32, 200, 33), (33, 256, 64),
             (33, 1, 1), (768, 151, 32), (1536, 64, 40)]


@pytest.mark.parametrize("metric", ["COSINE", "EUCLIDEAN"])
def test_select_f32(ctx, metric):
    cosine = metric == "COSINE"
    decided = total = 0
    undecided = []
    for c, (dim, kc, m_max) in enumerate(F32_CASES):
        rng = np.random.default_rng(70 + c + 100 * cosine)
        n = 2048
        X = f32_data(rng, n + 128, dim, cosine, equal_norms=cosine and kc > 64)
        elems = rng.permutation(n + 128)[:n]
        cand, cnt = cand_lists(rng, n + 128, elems, kc)
        cand[:200, : min(kc, 8)] = rng.integers(0, 14, (200, min(kc, 8)))  # the degenerate rows in many lists
        # the twins 20..39 / 40..59 inside one list (equal distances: list order decides), and, euclidean, elements
        # whose own twin is a candidate (e_dist then equals r_dist exactly for every later candidate; under cosine the
        # two differ by the rounding of the unfused e_dist, which the reference cannot decide)
        if kc >= 48:
            cand[200:216, 8:48] = rng.permutation(np.arange(20, 60))
            cnt[200:216] = np.maximum(cnt[200:216], 48)
        tw = np.nonzero((elems >= 20) & (elems < 40))[0][: 0 if cosine else 4]
        cand[tw, 0] = elems[tw] + 20
        pick = np.concatenate([np.nonzero(elems < 14)[0][:4], [200, 201], tw,
                               rng.choice(n, 20 if dim < 768 else 6, replace=False)])
        for presorted in (1, 0):
            out, oc = f32_select(ctx, X, metric, cand, cnt, kc, m_max, presorted, elems=elems)
            for i in pick:
                want, ok = F.select(X, int(elems[i]), cand[i, : cnt[i]], m_max, presorted, cosine)
                total += 1
                if not ok:
                    undecided.append((dim, kc, m_max, presorted, int(i)))
                    continue
                decided += 1
                assert list(out[i, : oc[i]]) == want, (metric, dim, kc, m_max, presorted, int(i))
        # row0 addressing selects what the explicit ids select
        o1, c1 = f32_select(ctx, X, metric, cand, cnt, kc, m_max, 0, row0=100)
        o2, c2 = f32_select(ctx, X, metric, cand, cnt, kc, m_max, 0, elems=np.arange(100, 100 + n))
        assert (c1 == c2).all() and all((o1[i, : c1[i]] == o2[i, : c2[i]]).all() for i in range(n))
    print(f"F32 {metric}: {decided} of {total} sampled selections decided; undecided {undecided}")
    assert decided >= 0.95 * total, (decided, total, undecided)


# ---- d. limits ------------------------------------------------------------------------------------------------------
# typed kernels: 4 warps x per_warp (rounded to 16 bytes) <= 220 KB.  F64 EUCLIDEAN per_warp = 8 dim (rounded to 16)
# + 4224 (tile) + 64, plus 12 kc + 4 m_max (select) or 12 (k + 1) (kNN): kc 256, m_max 32 fits dim 6104, not 6105;
# k 256 fits dim 6118, not 6119.  The f32 selection: 16 (2 dim + 2 kc) bytes <= 227 KB, i.e. dim + kc <= 7264.

def test_typed_shared_memory_limits(ctx):
    from surrealdb_b200 import _lib as L
    from surrealdb_b200.hnsw_build import knn_exact, select
    rng = np.random.default_rng(8)
    for dim_in, dim_out, what in ((6104, 6105, "select"), (6118, 6119, "knn")):
        X = rng.normal(0, 1, (600, dim_out)).astype(np.float64)
        inside = index(ctx, np.ascontiguousarray(X[:, :dim_in]), "euclidean", "F64")
        outside = index(ctx, X, "euclidean", "F64")
        try:
            Xi = np.ascontiguousarray(X[:, :dim_in])
            if what == "select":
                elems = np.arange(600)
                cand, cnt = cand_lists(rng, 600, elems, 256)
                out, oc = select(inside.h, dev(cand), dev(cnt), 32, 0, row0=0)
                out, oc = out.cpu().numpy(), oc.cpu().numpy()
                for i in (0, 1, 2, 599):
                    assert list(out[i, : oc[i]]) == ref_select("euclidean", "F64", Xi, i, cand[i, : cnt[i]], 32, 0)
                with pytest.raises(L.SdbError, match="SDB_EUNSUPPORTED"):
                    select(outside.h, dev(cand), dev(cnt), 32, 0, row0=0)
                c64, n64 = cand[:, :64].copy(), np.minimum(cnt, 64)  # the handle keeps answering
                o2, c2 = select(outside.h, dev(c64), dev(n64), 32, 0, row0=0)
                o2, c2 = o2.cpu().numpy(), c2.cpu().numpy()
                for i in (0, 1, 599):
                    assert list(o2[i, : c2[i]]) == ref_select("euclidean", "F64", X, i, c64[i, : n64[i]], 32, 0)
            else:
                ids, dist, cnt = knn_exact(inside.h, dev(Xi[:100]), 256)
                ids, cnt = ids.cpu().numpy(), cnt.cpu().numpy()
                for q in (0, 50, 99):
                    wi, _ = ref_knn("euclidean", "F64", Xi, Xi[q], 256, np.arange(600))
                    assert cnt[q] == 256 and list(ids[q]) == list(wi)
                with pytest.raises(L.SdbError, match="SDB_EUNSUPPORTED"):
                    knn_exact(outside.h, dev(X[:10]), 256)
                ids, _, cnt = knn_exact(outside.h, dev(X[:10]), 8)
                assert (cnt.cpu().numpy() == 8).all() and (ids.cpu().numpy()[:, 0] == np.arange(10)).all()
        finally:
            inside.close()
            outside.close()


def test_f32_select_shared_memory_limit(ctx):
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(9)
    kc, n = 256, 300
    X = rng.normal(0, 1, (n, 7009)).astype(np.float32)
    elems = np.arange(n)
    cand, cnt = cand_lists(rng, n, elems, kc)
    cnt[:2] = 40  # the sampled elements: a short list keeps the reference quick at this width
    for metric in ("COSINE", "EUCLIDEAN"):
        Xi = np.ascontiguousarray(X[:, :7008])  # dim + kc = 7264: fits
        out, oc = f32_select(ctx, Xi, metric, cand, cnt, kc, 32, 0, row0=0)
        for i in (0, 1):
            want, ok = F.select(Xi, i, cand[i, : cnt[i]], 32, 0, metric == "COSINE")
            if ok:
                assert list(out[i, : oc[i]]) == want, (metric, i)
        with pytest.raises(L.SdbError, match="SDB_EUNSUPPORTED"):  # 7265
            f32_select(ctx, X, metric, cand, cnt, kc, 32, 0, row0=0)
        out2, oc2 = f32_select(ctx, Xi, metric, cand, cnt, kc, 32, 0, row0=0)
        assert (oc2 == oc).all()


# ---- e. both F32 builders on degenerate data ------------------------------------------------------------------------

def build(ctx, data, metric, builder):
    from surrealdb_b200.hnsw_build import build_incremental, build_layers
    n, dim = data.shape
    if builder == "layers":
        layers, entry, levels = build_layers(ctx, dev(data), n, dim, metric.upper(), m=8, m0=16, seed=5)
        return data, layers, entry, levels
    res = build_incremental(ctx, dev(data), metric.upper(), m=8, m0=16, efc=64, seed=5, boot_min=1000)
    layers = [(rp.cpu().numpy().astype(np.uint64), ci.cpu().numpy().astype(np.uint32)) for rp, ci in res["layers_dev"]]
    return res["x"].cpu().numpy(), layers, res["entry"], res["levels"]


def recall(ctx, x, layers, entry, metric, queries, k=10, ef=64):
    """recall@k at ef against the exact kNN over the rows whose distances are numbers (a NaN distance may rank first)"""
    from surrealdb_b200.hnsw import HnswIndex
    from surrealdb_b200.hnsw_build import knn_exact
    idx = HnswIndex(ctx, x, layers, entry, metric)
    ids, dist, cnt = idx.search_graph(queries, k, ef)
    ok = np.isfinite(x).all(1) & ((x != 0).any(1) if metric == "cosine" else True)
    tids, _, tcnt = knn_exact(idx.h, dev(queries), k, dev(np.nonzero(ok)[0].astype(np.int32)))
    tids, tcnt = tids.cpu().numpy(), tcnt.cpu().numpy()
    r = float(np.mean([len(set(ids[q, : cnt[q]].tolist()) & set(tids[q, : tcnt[q]].tolist())) / k
                       for q in range(queries.shape[0])]))
    return r, idx, (ids, dist, cnt)


@pytest.mark.parametrize("builder", ["layers", "incremental"])
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_builders_on_degenerate_rows(ctx, metric, builder):
    from oracle import pyoracle as O
    rng = np.random.default_rng(13)
    n, dim = 3000, 16
    bad = clustered(rng, metric, "F32", n + 100, dim)
    bad, queries = bad[:n], bad[n:]
    where = rng.choice(n, 40, replace=False)
    bad[where[:10]] = 0.0  # zero rows: NaN cosine distances
    bad[where[10:30]] = bad[where[30:40]].repeat(2, 0)  # duplicate rows
    if metric == "euclidean":
        bad[where[0], 3] = np.nan  # a NaN row
    clean = np.delete(bad, where[:30], axis=0)  # the same data without the zero, NaN and repeated rows
    rs = {}
    for name, data in (("clean", clean), ("degenerate", bad)):
        x, layers, entry, levels = build(ctx, data, metric, builder)
        check_structure(layers, levels, data.shape[0], 8, 16)
        r, idx, (ids, dist, cnt) = recall(ctx, x, layers, entry, metric, queries)
        rs[name] = r
        g = {"vectors": x, "layers": layers, "entry_point": entry}
        for q in range(8):
            oi, od, _ = O.hnsw_search_csr(dict(g, metric=metric), queries[q], 10, 64)
            assert list(ids[q, : cnt[q]]) == list(oi), (name, q)
            assert all(same(metric, a, b) for a, b in zip(dist[q, : cnt[q]], od)), (name, q)
        idx.close()
    print(f"RECALL {builder} {metric} clean {rs['clean']:.3f} degenerate {rs['degenerate']:.3f}")
    assert rs["degenerate"] >= rs["clean"] - 0.05, rs
