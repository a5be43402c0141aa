"""Brute-force KNN of PEARSON columns through the cosine tensor-core screens on the centred rows, the f32 re-score, the
proof (with eps_ref) and the exact re-rank.  Every answer is compared bit for bit (rows, f64 distances, counts) with the
CPU oracle; the screen's premises (centred copies, residual figures, scores within the bound of -pearson, kept sets,
every excluded row beyond the proof's bound) are held against tests/pearson_screen_ref.py through the debug calls."""
import ctypes as C
import zlib

import numpy as np
import pytest

import pearson_screen_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SIMT_F32, TC_BF16, NONE_EXACT, TC_INT8 = 1, 2, 3, 4
SCREEN = {"AUTO": None, "TC_INT8": TC_INT8, "TC_BF16": TC_BF16, "SIMT_F32": NONE_EXACT, "NONE_EXACT": NONE_EXACT}


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def make_col(ctx, corpus, skip=None, screen=None):
    from surrealdb_b200 import VectorColumn
    dt = "F32" if corpus.dtype == np.float32 else "F64"
    col = VectorColumn(ctx, corpus.shape[1], "PEARSON", dt, capacity=max(1, corpus.shape[0]))
    col.append(corpus)
    if skip is not None:
        col.set_skip(skip)
    col.finalize()
    if screen:
        col.set_screen(screen)
    return col


def check(corpus, queries, k, rows, dist, cnt, qs=None, skip=None):
    qs = range(queries.shape[0]) if qs is None else qs
    for q in qs:
        r, d = O.knn_topk(corpus, queries[q], "pearson", k, skip=skip)
        assert cnt[q] == r.size, (q, int(cnt[q]), r.size)
        assert rows[q, : cnt[q]].tolist() == r.tolist(), (q, rows[q, : cnt[q]], r)
        assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, dist[q, : cnt[q]], d)


def sample(nq):
    return sorted(set(list(range(0, nq, max(1, nq // 16))) + [nq - 1]))


def expected_screen(screen, k, dim):
    if k > 256 or dim == 1 or SCREEN[screen] == NONE_EXACT:
        return NONE_EXACT
    return SCREEN[screen]


# ---- 1. parity matrix ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [2, 7, 100, 768, 1025, 4100])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_parity_matrix(ctx, dtype, dim):
    rng = np.random.default_rng(zlib.crc32(f"pearson{dtype}{dim}".encode()))
    n = 6000 if dim <= 1025 else 2500
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    col = make_col(ctx, corpus)
    nqs = (1, 3, 17, 64, 1024, 2100) if dim <= 768 else (1, 17, 64)
    runs = [(nq, "AUTO") for nq in nqs] + [(17, s) for s in ("TC_INT8", "TC_BF16", "SIMT_F32", "NONE_EXACT")]
    for nq, screen in runs:
        col.set_screen(screen)
        queries = rng.uniform(-1, 1, (nq, dim))
        for k in (1, 10, 100, 256, 257):
            if nq > 64 and k not in (10, 257):
                continue
            rows, dist, cnt = col.knn(queries, k)
            st = col.stats()
            want = expected_screen(screen, k, dim)
            if want is None:  # AUTO: int8 when the quantisation is fine enough, else bf16
                assert st["screen_used"] in (TC_INT8, TC_BF16) and st["n_passes"] > 0, (nq, k, st)
                if dim > 2:
                    assert st["n_fallback"] <= 2 + nq // 64, (nq, k, st)
            else:
                assert st["screen_used"] == want, (screen, nq, k, st)
            check(corpus, queries, k, rows, dist, cnt, qs=sample(nq))


# ---- 2. data shapes ---------------------------------------------------------------------------------------------------
DATA = {
    "uniform20": lambda rng, n, d: rng.uniform(-20, 20, (n, d)),
    "offset1000": lambda rng, n, d: 1000.0 + rng.uniform(-1e-3, 1e-3, (n, d)),
    "clustered": lambda rng, n, d: rng.normal(0, 1, (32, d))[rng.integers(0, 32, n)] + rng.normal(0, 1e-2, (n, d)),
    "scaled_small": lambda rng, n, d: rng.uniform(-1, 1, (n, d)) * 1e-30,
    "scaled_large": lambda rng, n, d: rng.uniform(-1, 1, (n, d)) * 1e30,
}


@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("case", list(DATA))
def test_data_shapes(ctx, case, dtype):
    if case.startswith("scaled") and dtype == "F32":
        pytest.skip("f64 magnitudes")
    rng = np.random.default_rng(zlib.crc32(f"{case}{dtype}".encode()))
    n, dim = 8000, 96
    corpus = DATA[case](rng, n, dim).astype(np.float32 if dtype == "F32" else np.float64)
    queries = DATA[case](rng, 40, dim)
    queries[:5] = corpus[rng.integers(0, n, 5)].astype(np.float64)
    col = make_col(ctx, corpus)
    for k in (1, 10, 200):
        rows, dist, cnt = col.knn(queries, k)
        assert col.stats()["screen_used"] in (TC_INT8, TC_BF16)
        check(corpus, queries, k, rows, dist, cnt)


# ---- 3. near-ties, special rows and queries ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_near_ties_special_rows_and_queries(ctx, dtype):
    rng = np.random.default_rng(zlib.crc32(f"adv{dtype}".encode()))
    fdt = np.float32 if dtype == "F32" else np.float64
    n, dim = 6000, 64
    corpus = rng.uniform(-1, 1, (n, dim)).astype(fdt)
    queries = rng.uniform(-1, 1, (14, dim))
    base = corpus[40].astype(np.float64)
    for i, (a, b) in enumerate([(2.0, 0.5), (3.0, -7.0), (0.3, 100.0), (1.0, 1e-3)]):  # affine copies: equal in theory
        corpus[41 + i] = (a * base + b).astype(fdt)
    corpus[50] = -corpus[40]                              # a row and its negation
    corpus[51] = np.nextafter(corpus[40], fdt(np.inf))    # one-ulp neighbours
    corpus[52] = np.nextafter(corpus[40], fdt(-np.inf))
    corpus[100] = 0.0                                     # constant rows: 0/0, a generated NaN that sorts first
    corpus[101] = -0.0
    corpus[102] = 5.0
    corpus[103, 3] = np.nan                               # data NaN: sorts last
    corpus[104, 0] = np.inf
    corpus[105, 1] = -np.inf
    corpus[106, 0], corpus[106, 1] = np.inf, -np.inf       # +inf and -inf: a generated NaN mean
    corpus[107] = 1.0
    corpus[107, 9] = 1.0 + 1e3                            # one dominant component: an int8 outlier
    if dtype == "F64":
        corpus[108, 2] = 1e39                             # beyond f32 range
        corpus[109] = 7.0 + rng.uniform(-1, 1, dim) * 1e-32  # centred norm below 2^-100
    queries[0] = base                                     # equal to a row
    queries[1] = -base                                    # a negated row: pearson exactly -1
    queries[2] = 3.0                                      # constant query: the exact kernel
    queries[3, 7] = 1e300                                 # beyond f32 range
    queries[4] = 2.0 * base - 1.0
    col = make_col(ctx, corpus)
    for k in (1, 10, 100, 256):
        rows, dist, cnt = col.knn(queries, k)
        assert col.stats()["screen_used"] in (TC_INT8, TC_BF16)
        check(corpus, queries, k, rows, dist, cnt)
    assert col.stats()["n_special_rows"] >= (8 if dtype == "F32" else 10)


def test_nan_query(ctx):
    # a query with a NaN element takes the exact kernel: every distance is a positive NaN, ties by scan position.
    # (Against rows whose own arithmetic generates a NaN -- an infinite element -- the NaN sign is unpinned, DESIGN.md
    # section 3, so this corpus holds a data NaN row only.)
    rng = np.random.default_rng(31)
    corpus = rng.uniform(-1, 1, (5000, 24)).astype(np.float32)
    corpus[9, 2] = np.nan
    queries = rng.uniform(-1, 1, (3, 24))
    queries[1, 5] = np.nan
    col = make_col(ctx, corpus)
    rows, dist, cnt = col.knn(queries, 10)
    assert col.stats()["n_fallback"] == 1
    check(corpus, queries, 10, rows, dist, cnt)


@pytest.mark.parametrize("n_special", [1024, 1025])
def test_special_list_capacity(ctx, n_special):
    rng = np.random.default_rng(n_special)
    corpus = rng.uniform(-1, 1, (6000, 16)).astype(np.float32)
    corpus[rng.choice(6000, n_special, replace=False)] = 2.5  # constant rows
    queries = rng.uniform(-1, 1, (5, 16))
    col = make_col(ctx, corpus)
    rows, dist, cnt = col.knn(queries, 10)
    assert col.stats()["screen_used"] == (NONE_EXACT if n_special > 1024 else TC_INT8)
    check(corpus, queries, 10, rows, dist, cnt)


# ---- 4. mutations and filters ------------------------------------------------------------------------------------------
def test_skip_remove_and_refinalize(ctx):
    from surrealdb_b200 import VectorColumn
    rng = np.random.default_rng(5)
    n, dim = 8000, 40
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = corpus[rng.integers(0, n, 8)].astype(np.float64) + rng.normal(0, 1e-3, (8, dim))
    skip = (rng.random(n) < 0.2).astype(np.uint8)
    dead = np.unique(rng.integers(0, n, 200)).astype(np.uint64)
    col = VectorColumn(ctx, dim, "PEARSON", "F32", capacity=n)
    col.append(corpus)
    col.set_skip(skip)
    col.remove(dead[:100])
    col.finalize()
    col.remove(dead[100:])
    eff = skip.copy()
    eff[dead.astype(np.int64)] = 1
    rows, dist, cnt = col.knn(queries, 10)
    assert col.stats()["screen_used"] in (TC_INT8, TC_BF16)
    check(corpus, queries, 10, rows, dist, cnt, skip=eff)
    skip2 = (rng.random(n) < 0.5).astype(np.uint8)
    col.set_skip(skip2)
    col.finalize()
    eff = skip2.copy()
    eff[dead.astype(np.int64)] = 1
    rows, dist, cnt = col.knn(queries, 10)
    check(corpus, queries, 10, rows, dist, cnt, skip=eff)


def pack(masks):
    from surrealdb_b200.engine import pack_row_filter
    return pack_row_filter(np.asarray(masks, bool))


@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_filters(ctx, dtype):
    import torch
    rng = np.random.default_rng(zlib.crc32(f"filt{dtype}".encode()))
    n, dim = 40000 + 11, 48
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32 if dtype == "F32" else np.float64)
    corpus[17] = 1.0  # a constant (special) row passes every filter below that keeps it
    col = make_col(ctx, corpus)
    masks = np.stack([np.ones(n, bool), rng.random(n) < 0.1, rng.random(n) < 0.01, rng.random(n) < 3000 / n])

    def run(queries, qf, k=10, device=False):
        if device:  # device bitmaps, queries and outputs
            dev = torch.device("cuda", 0)
            bits = torch.from_numpy(pack(masks).view(np.int32)).to(dev)
            qd = torch.from_numpy(np.ascontiguousarray(queries)).to(dev)
            nq = queries.shape[0]
            o = (torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64,
                 device=dev), torch.zeros(nq, dtype=torch.int32, device=dev))
            torch.cuda.synchronize()
            col.knn_device_filtered(qd.data_ptr(), nq, k, bits.data_ptr(), masks.shape[0], qf, 0, o[0].data_ptr(),
                                    o[1].data_ptr(), o[2].data_ptr())
            torch.cuda.synchronize()
            rows, dist, cnt = (t.cpu().numpy() for t in o)
            rows, cnt = rows.astype(np.uint64), cnt.astype(np.uint32)
        else:
            rows, dist, cnt = col.knn(queries, k, filters=pack(masks), query_filter=qf)
        for q in sample(queries.shape[0]):
            sk = (~masks[qf[q]]).astype(np.uint8)
            r, d = O.knn_topk(corpus, queries[q], "pearson", k, skip=sk)
            assert cnt[q] == r.size and rows[q, : cnt[q]].tolist() == r.tolist(), (q, qf[q])
            assert dist[q, : cnt[q]].tobytes() == d.tobytes(), (q, qf[q])
        return col.stats()

    qs = rng.uniform(-1, 1, (6, dim))
    st = run(qs, np.array([0, 1, 2, 0, 1, 2], np.uint32))  # 100 %, 10 %, 1 %
    assert st["screen_used"] in (TC_INT8, TC_BF16) and st["n_passes"] > 0
    st = run(qs, np.full(6, 3, np.uint32))                  # <= 4096 rows: the direct regime, no screen
    assert st["n_passes"] == 0, st
    run(qs, np.array([3, 0, 3, 2, 3, 1], np.uint32))        # mixed direct / screened batch
    qb = rng.uniform(-1, 1, (300, dim))
    run(qb, rng.integers(0, 4, 300).astype(np.uint32))
    run(qs, np.array([0, 1, 2, 3, 3, 1], np.uint32), device=True)


# ---- 5. tickets, cancellation, shards ----------------------------------------------------------------------------------
def test_async_tickets_and_cancellation(ctx):
    import torch
    from surrealdb_b200 import SdbError
    from surrealdb_b200 import _lib as L
    rng = np.random.default_rng(4)
    n, dim, nq, k = 20000, 64, 70, 10
    corpus = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    col = make_col(ctx, corpus)
    dev = torch.device("cuda", 0)
    batches = [rng.uniform(-1, 1, (nq, dim)) for _ in range(4)]
    qd = [torch.from_numpy(b).to(dev) for b in batches]
    outs = [(torch.zeros((nq, k), dtype=torch.int64, device=dev), torch.zeros((nq, k), dtype=torch.float64, device=dev),
             torch.zeros(nq, dtype=torch.int32, device=dev)) for _ in range(4)]
    torch.cuda.synchronize()
    tickets = [col.submit_device(qd[i].data_ptr(), nq, k, 0, outs[i][0].data_ptr(), outs[i][1].data_ptr(),
                                 outs[i][2].data_ptr()) for i in range(4)]
    for t in tickets:
        col.wait(t)
    torch.cuda.synchronize()
    for i in range(4):
        rows, dist, cnt = (o.cpu().numpy() for o in outs[i])
        check(corpus, batches[i], k, rows.astype(np.uint64), dist, cnt.astype(np.uint32), qs=sample(nq))
    flag = np.ones(1, np.int32)
    with pytest.raises(SdbError) as e:
        col.knn(batches[0][:4], 10, cancel_flag=flag)
    assert e.value.status == L.SDB_ECANCELLED
    rows, dist, cnt = col.knn(batches[0][:4], 10)
    check(corpus, batches[0][:4], 10, rows, dist, cnt)


@pytest.mark.parametrize("dtype", ["F32", "F64"])
def test_two_shards_merged(ctx, dtype):
    import torch
    from surrealdb_b200 import VectorColumn
    from surrealdb_b200.engine import shard_block_layout, topk_merge_device
    rng = np.random.default_rng(2)
    rows_n, dim, nq, k, world = 20000, 64, 40, 10, 2
    fdt = np.float32 if dtype == "F32" else np.float64
    corpus = rng.uniform(-1, 1, (rows_n, dim)).astype(fdt)
    corpus[15000:15004] = corpus[100:104]  # exact ties across the shards resolve by global row
    queries = rng.uniform(-1, 1, (nq, dim))
    queries[0] = corpus[100]
    dev = torch.device("cuda", 0)
    qd = torch.from_numpy(queries).to(dev)
    torch.cuda.synchronize()
    off_rows, off_dist, off_cnt, blk = shard_block_layout(nq, k)
    gathered = torch.zeros(world * blk, dtype=torch.uint8, device=dev)
    for r in range(world):
        base, n_local = r * rows_n // world, rows_n // world
        col = VectorColumn(ctx, dim, "PEARSON", dtype, capacity=n_local)
        col.append(corpus[base:base + n_local])
        col.finalize()
        p = gathered.data_ptr() + r * blk
        col.knn_device(qd.data_ptr(), nq, k, base, p + off_rows, p + off_dist, p + off_cnt)
        assert col.stats()["screen_used"] in (TC_INT8, TC_BF16)
    f_rows = torch.zeros((nq, k), dtype=torch.int64, device=dev)
    f_dist = torch.zeros((nq, k), dtype=torch.float64, device=dev)
    f_cnt = torch.zeros((nq,), dtype=torch.int32, device=dev)
    gp = gathered.data_ptr()
    topk_merge_device(ctx, world, nq, k, gp + off_rows, gp + off_dist, gp + off_cnt, f_rows.data_ptr(),
                      f_dist.data_ptr(), f_cnt.data_ptr(), stride_rows=blk // 8, stride_dist=blk // 8,
                      stride_counts=blk // 4)
    torch.cuda.synchronize()
    check(corpus, queries, k, f_rows.cpu().numpy().astype(np.uint64), f_dist.cpu().numpy(),
          f_cnt.cpu().numpy().astype(np.uint32))


# ---- 6. the proof's premises -------------------------------------------------------------------------------------------
def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def corpus_state(col, n):
    from surrealdb_b200 import _lib as L
    f, u = np.zeros(4, np.float32), np.zeros(5, np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, _p(f), _p(u), None, None, None, None))
    n_special, dim_pad, dim_pad8, n_pad = int(u[0]), int(u[2]), int(u[3]), int(u[4])
    i8 = np.zeros((n_pad, dim_pad8), np.int8)
    bf = np.zeros((n_pad, dim_pad), np.uint16)
    snorm = np.zeros(n_pad, np.float32)
    special = np.zeros(max(n_special, 1), np.uint32)
    L.check(L.lib().sdb_debug_corpus_state(col.h, None, None, _p(i8), _p(bf), _p(snorm), _p(special)))
    return dict(scale=f[0], qerr=f[1], bf_err=f[2], n_pad=n_pad, i8=i8, bf=bf, snorm=snorm,
                special=set(special[:n_special].tolist()))


def debug_batch(col, Q, k, screen, score_all, n_pad, cap=4096):
    from surrealdb_b200 import _lib as L
    nq = Q.shape[0]
    capq = max(cap, n_pad) if score_all else cap
    o = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
             a=np.zeros((nq, capq, 3), np.uint32))
    if not score_all:
        o["b"] = np.zeros((nq, capq, 2), np.uint32)
        o["rr"] = np.zeros((nq, capq + 1024), np.uint32)
    L.check(L.lib().sdb_debug_screen_batch(col.h, _p(Q), nq, k, screen, 0, cap, int(score_all), _p(o["qf"]),
                                           _p(o["qmag"]), _p(o["qu"]), None, None, _p(o["a"]), _p(o.get("b")),
                                           _p(o.get("rr"))))
    o["tau"], o["margin"], o["bscale"], o["beps"] = (o["qf"][:, j] for j in (0, 1, 2, 3))
    o["tau2"], o["beps2"] = o["qf"][:, 4], o["qf"][:, 5]
    o["flags"], o["qflags"], o["n_a"], o["n_b"], o["n_e"] = (o["qu"][:, j].astype(np.int64) for j in (0, 1, 3, 4, 5))
    return o


PREMISE_CASES = {
    "uniform_d100": lambda rng: rng.uniform(-1, 1, (3000, 100)),
    "offset_d257": lambda rng: 1e6 + rng.uniform(-1, 1, (2000, 257)),
    "special_d33": lambda rng: np.where(rng.random((2500, 33)) < 0.002, np.nan, rng.uniform(-20, 20, (2500, 33))),
}


@pytest.mark.parametrize("screen", [TC_INT8, TC_BF16])
@pytest.mark.parametrize("dtype", ["F32", "F64"])
@pytest.mark.parametrize("case", list(PREMISE_CASES))
def test_proof_premises(ctx, case, dtype, screen):
    rng = np.random.default_rng(zlib.crc32(f"pearson{case}{dtype}".encode()))
    X = PREMISE_CASES[case](rng).astype(np.float32 if dtype == "F32" else np.float64)
    n, dim = X.shape
    k = 10
    col = make_col(ctx, X)
    s = corpus_state(col, n)
    # (1) the copies: snorm = fl32(1/|dx|), bf16(dx), the int8 copy of dx/|dx|, specials, residual figures
    special = R.is_special(X)
    assert s["special"] >= set(np.flatnonzero(special).tolist())  # (plus the int8 outliers, if any)
    valid = ~np.isnan(s["snorm"][:n])
    assert not (valid & special).any() and np.isnan(s["snorm"][n:]).all()
    _, s1, dx = R.moments(X)
    assert np.array_equal(s["snorm"][:n][valid], (1.0 / np.sqrt(s1[valid])).astype(np.float32))
    bf = (s["bf"][:n, :dim].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    assert np.array_equal(bf[valid], R.bf16_rn(dx[valid]))
    assert s["bf_err"] >= R.bf16_residual(X[valid]) * (1 - 1e-6)
    q8, res = R.int8_copy(X[valid], s["scale"])
    assert np.array_equal(s["i8"][:n, :dim][valid], q8)
    assert s["qerr"] >= res.max() * (1 - 1e-6)
    # (2) score_all: every valid pair scores within beps (+ eps_ref) of -pearson
    Q = X[rng.integers(0, n, 12)].astype(np.float64)
    Q = np.where(np.isfinite(Q), Q, 0.25) + rng.normal(0, 1e-2, Q.shape) * np.nanstd(X)
    Q = np.ascontiguousarray(Q)
    o = debug_batch(col, Q, k, screen, True, s["n_pad"])
    P = np.stack([R.pearson(X, q) for q in Q])
    ok_q = (o["qflags"] & 1) == 0
    for q in np.flatnonzero(ok_q):
        rws = o["a"][q, : o["n_a"][q], 0]
        sc = o["a"][q, : o["n_a"][q], 1].view(np.float32).astype(np.float64)
        keep = (rws < n) & ~np.isnan(sc)
        if screen == TC_INT8:
            keep &= valid[np.minimum(rws, n - 1)]
        rws, sc = rws[keep], sc[keep]
        assert set(rws.tolist()) >= set(np.flatnonzero(valid).tolist())
        sim = sc * np.float64(o["bscale"][q]) / o["qmag"][q]
        dev = np.abs(sim + P[q, rws])
        assert (dev <= np.float64(o["beps"][q]) + R.eps_ref(dim)).all(), (q, dev.max(), o["beps"][q])
    # (3) the production sequence: kept set, tau, stage B, and an audit of the proof
    o = debug_batch(col, Q, k, screen, False, s["n_pad"])
    for q in np.flatnonzero(ok_q):
        if o["flags"][q] & 2:
            continue
        in_a = np.zeros(n, bool)
        in_a[o["a"][q, : o["n_a"][q], 0].astype(np.int64)] = True
        tau = np.float64(o["tau"][q])
        if tau > -np.inf:  # stage A left out every other valid row: each lies beyond the proof's bound
            bound = R.proof_bound(o["tau"][q], o["bscale"][q], o["qmag"][q], o["beps"][q], dim)
            assert not (valid & ~in_a & (P[q] < bound)).any(), q
        t2 = np.float64(o["tau2"][q])
        if t2 > -np.inf:  # stage B kept exactly the rows reaching tau2; the ones it dropped lie beyond its bound
            b_rows = o["b"][q, : o["n_b"][q], 0].astype(np.int64)
            b_sc = o["b"][q, : o["n_b"][q], 1].view(np.float32)
            r_sc = o["a"][q, : o["n_a"][q], 2].view(np.float32)
            assert (b_sc >= np.float32(t2)).all()
            assert np.array_equal(np.sort(b_rows), np.sort(o["a"][q, : o["n_a"][q], 0][r_sc >= np.float32(t2)]))
            in_b = np.zeros(n, bool)
            in_b[b_rows] = True
            bound2 = R.proof_bound(o["tau2"][q], 1.0, o["qmag"][q], o["beps2"][q], dim)
            assert not (in_a & ~in_b & (P[q] < bound2)).any(), q
