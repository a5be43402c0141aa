"""Invariants of the filtered brute-force screens (per-query row bitmaps), each held against the unfiltered screen and
a plain reference, through the test-only entry point sdb_debug_screen_batch_filtered.

DESIGN.md section 2, "Filtered rows and the proof": a row the query's filter rejects counts nowhere -- not in the
probe's chunk maxima, not in the refiners' histograms, not in a list.  End-to-end parity cannot see a rejected row that
raises tau (the proof fails, the query is repaired, the answer stays right), and sees a dropped passing row only when
it was a true neighbour.  So every link is checked directly, per query of every batch:

  a  pass 0        the filtered score list holds every valid passing row with its unfiltered score, bit for bit;
                   the tensor-core screens NaN the rejected rows, SIMT_F32 never appends them
  b  stage A       kept set = {valid, passing, score >= tau} (int8: integer dot >= ceil(tau)), unfiltered scores,
                   overflow flag iff more were gathered than the list holds
  c  threshold     tau <= (k-th best score over the valid PASSING rows) - margin; the leak detector (a filter rejecting
                   the query's ~2000 best rows) fails here if rejected rows reach the probe or the histograms
  d  stage B       f32 re-scores within beps2, kept set = the stage-A rows reaching tau2
  e  re-rank set   the stage-B rows plus exactly the special rows the query's filter passes
  f  proof audit   every valid passing row outside the re-rank set of a proven query is beyond the proof's bound
  g  mask_hits     the int8 consumers' hit-mask filtering is a speed switch: off, on and the production rule give the
                   same tau and stage-A sets in the multi-pass schedule, and each holds (b) and (c) when streaming
  h  direct        filters of at most DIRECT_MAX_ROWS set bits skip the screen: the list is exactly the passing rows
                   that are below n, unskipped and not removed (special rows included, padding bits ignored)
"""
import ctypes as C
import zlib

import numpy as np
import pytest

import lp_screen_ref as LR
import pearson_screen_ref as PR
import screen_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

SCREEN_CODE = {"SIMT_F32": 1, "TC_BF16": 2, "TC_INT8": 4}
SPECIAL_CAP = 1024
DIRECT_MAX_ROWS = 4096  # csrc/internal.cuh
K = 10
LEAK_ROWS = 2000


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


# ------------------------------------------------------------------------------------------------------------ corpora
# name: metric, dtype, n, dim, share of skipped rows.  Row counts are multiples of neither 32 nor 256.  On the small
# corpora the filters also set the bits of every skipped and removed row: these count towards the filter's set bits
# (the direct / screened split) but pass nothing, so the screened filters can pass as few rows as the direct ones.
CORPORA = {
    "cos_f32_d64": ("COSINE", "F32", 20011, 64, 0.25),
    "cos_f32_d33": ("COSINE", "F32", 20011, 33, 0.25),
    "euc_f32_d64": ("EUCLIDEAN", "F32", 20011, 64, 0.25),
    "cos_f64_d64": ("COSINE", "F64", 20011, 64, 0.25),
    "pea_f32_d48": ("PEARSON", "F32", 20011, 48, 0.25),
    "man_f32_d36": ("MANHATTAN", "F32", 20011, 36, 0.25),
    "man_f64_d36": ("MANHATTAN", "F64", 20011, 36, 0.25),
    "che_f32_d35": ("CHEBYSHEV", "F32", 20011, 35, 0.25),
    "che_f64_d36": ("CHEBYSHEV", "F64", 20011, 36, 0.25),
    "cos_f32_fits": ("COSINE", "F32", 12007, 64, 0.4),  # fits a 16384-slot list: the streaming pass-0 path
    "cos_f32_big": ("COSINE", "F32", 100003, 32, 0.001),  # a 4500-row filter is < n / 20: mask_hits on by the rule
}
ZERO, NAN, INF = 3, 11, 12
OUTLIERS = (4000, 9000, 15000)


class Corpus:
    def __init__(self, ctx, name):
        from surrealdb_b200 import VectorColumn
        from surrealdb_b200 import _lib as L
        metric, dtype, n, dim, skip_share = CORPORA[name]
        rng = np.random.default_rng(zlib.crc32(name.encode()))
        self.name, self.metric, self.dtype, self.n, self.dim, self.L = name, metric, dtype, n, dim, L
        X = rng.uniform(-1, 1, (n, dim))
        X[ZERO] = 0.0
        X[NAN, 5] = np.nan
        X[INF, 0] = np.inf
        for i, r in enumerate(OUTLIERS):
            if r < n:  # one dominant component: an int8 outlier of the cosine corpora
                X[r] = rng.uniform(-1e-3, 1e-3, dim)
                X[r, i] = 40.0
        self.X = np.ascontiguousarray(X.astype(np.float32 if dtype == "F32" else np.float64))
        keep = np.array([ZERO, NAN, INF] + [r for r in OUTLIERS if r < n])
        self.skip = (rng.random(n) < skip_share).astype(np.uint8)
        self.skip[keep] = 0
        self.col = VectorColumn(ctx, dim, metric, dtype, capacity=n)
        self.col.append(self.X)
        self.col.set_skip(self.skip)
        self.col.finalize()
        dead = np.setdiff1d(np.unique(rng.integers(0, n, 200)), keep)
        self.col.remove(dead)  # tombstones after finalize: NaN screening norm, all-zero int8 row
        self.removed = np.zeros(n, bool)
        self.removed[dead] = True
        self.gone = (self.skip != 0) | self.removed  # rows no search ranks
        lib = L.lib()
        f, u = np.zeros(4, np.float32), np.zeros(5, np.uint32)
        L.check(lib.sdb_debug_corpus_state(self.col.h, _p(f), _p(u), None, None, None, None))
        self.n_special, self.dim_pad, self.dim_pad8, self.n_pad = int(u[0]), int(u[2]), int(u[3]), int(u[4])
        self.snorm = np.zeros(self.n_pad, np.float32)
        special = np.zeros(max(self.n_special, 1), np.uint32)
        L.check(lib.sdb_debug_corpus_state(self.col.h, None, None, None, None, _p(self.snorm), _p(special)))
        self.special = np.sort(special[: self.n_special].astype(np.int64))
        self.valid = ~np.isnan(self.snorm[:n])
        assert self.special.size >= 2 and not self.valid[self.special].any()
        assert not (self.valid & self.gone).any()
        self.words = (n + 31) // 32
        self.rng = rng

    def queries(self, nq):
        rng = np.random.default_rng(zlib.crc32(f"{self.name}/{nq}".encode()))
        base = np.flatnonzero(self.valid)[rng.integers(0, int(self.valid.sum()), nq)]
        Q = self.X[base].astype(np.float64) * rng.uniform(0.5, 2.0, (nq, 1))
        Q += rng.normal(0, 1e-2, Q.shape)
        Q[::3] = rng.uniform(-1, 1, Q[::3].shape)
        return np.ascontiguousarray(Q)

    def pack(self, masks):
        """bool masks (n_filters, n) -> bitmaps; the last word's bits past n are set (they must be ignored)"""
        from surrealdb_b200.engine import pack_row_filter
        bits = np.atleast_2d(pack_row_filter(np.asarray(masks, bool))).copy()
        if self.n % 32:
            bits[:, -1] |= np.uint32((0xFFFFFFFF << (self.n % 32)) & 0xFFFFFFFF)
        return np.ascontiguousarray(bits, np.uint32)

    def batch(self, Q, screen, streaming=False, score_all=False, cap=4096, filters=None, qf=None, mask_hits=-1):
        nq = Q.shape[0]
        capq = max(cap, self.n_pad) if score_all else cap
        o = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
                 a=np.zeros((nq, capq, 3), np.uint32))
        if not score_all:
            o["b"] = np.zeros((nq, capq, 2), np.uint32)
            o["rr"] = np.zeros((nq, capq + SPECIAL_CAP), np.uint32)
        qf = None if qf is None else np.ascontiguousarray(qf, np.uint32)
        self.L.check(self.L.lib().sdb_debug_screen_batch_filtered(
            self.col.h, _p(Q), nq, K, SCREEN_CODE[screen], int(streaming), cap, int(score_all), _p(o["qf"]),
            _p(o["qmag"]), _p(o["qu"]), None, None, _p(o["a"]), _p(o.get("b")), _p(o.get("rr")), _p(filters),
            0 if filters is None else filters.shape[0], _p(qf), mask_hits))
        for j, nm in enumerate(("tau", "margin", "bscale", "beps", "tau2", "beps2")):
            o[nm] = o["qf"][:, j]
        for j, nm in enumerate(("flags", "qflags", "gathered", "n_a", "n_b", "n_e")):
            o[nm] = o["qu"][:, j].astype(np.int64)
        return o

    def score_matrix(self, Q, screen):
        """[nq][n] unfiltered pass-0 scores (NaN: not a screen candidate); tests/test_gpu_screen_invariants.py and the
        premise tests hold them against the exact references"""
        o = self.batch(Q, screen, score_all=True)
        S = np.full((Q.shape[0], self.n), np.nan, np.float32)
        for q in range(Q.shape[0]):
            rows = o["a"][q, : o["n_a"][q], 0]
            keep = rows < self.n
            S[q, rows[keep]] = o["a"][q, : o["n_a"][q], 1][keep].view(np.float32)
        S[:, ~self.valid] = np.nan
        return S

    def exact_distance(self, Q):
        """[nq][n] what the proof bounds: the oracle's distance (cosine, euclidean), pearson, the reference's L1 / L-inf"""
        if self.metric == "PEARSON":
            return np.stack([PR.pearson(self.X, q) for q in Q])
        if self.metric in ("MANHATTAN", "CHEBYSHEV"):
            return LR.reference(Q, self.X, self.metric)
        rows, dist = O.knn_topk_batch(self.X, Q, self.metric.lower(), self.n, 16)
        D = np.full((Q.shape[0], self.n), np.nan)
        for q in range(Q.shape[0]):  # (reversed: a row's ranked entry wins over unused trailing entries)
            D[q, rows[q, ::-1].astype(np.int64)] = dist[q, ::-1]
        return D

    def proof_bounds(self, o, q):
        """(stage-A bound, stage-B bound) of proven query q's excluded rows, in exact_distance's units"""
        tau, tau2 = o["tau"][q], o["tau2"][q]
        if self.metric == "COSINE":
            return (R.proof_bound_cosine(tau, o["bscale"][q], o["qmag"][q], o["beps"][q]),
                    R.proof_bound_cosine(tau2, 1.0, o["qmag"][q], o["beps2"][q]))
        if self.metric == "EUCLIDEAN":
            return R.proof_bound_euclid(tau, o["qmag"][q], o["beps"][q]), R.proof_bound_euclid(tau2, o["qmag"][q], o["beps2"][q])
        if self.metric == "PEARSON":
            return (PR.proof_bound(tau, o["bscale"][q], o["qmag"][q], o["beps"][q], self.dim),
                    PR.proof_bound(tau2, 1.0, o["qmag"][q], o["beps2"][q], self.dim))
        return -np.float64(tau) - np.float64(o["beps"][q]), -np.inf

    def stage_b_deviation(self, Q, q, rows, r_a, o):
        """|f32 re-score - exact| of stage B and the bound it must respect"""
        x = self.X[rows]
        if self.metric == "COSINE":
            return np.abs(r_a / o["qmag"][q] - R.cosine_sim(Q[q: q + 1], x)[0]), np.float64(o["beps2"][q])
        if self.metric == "EUCLIDEAN":
            return np.abs(r_a.astype(np.float64) - R.euclid_score(Q[q: q + 1], x)[0]), np.float64(o["beps2"][q])
        return np.abs(r_a.astype(np.float64) + PR.pearson(x, Q[q])), np.float64(o["beps2"][q]) + PR.eps_ref(self.dim)


_CACHE = {}


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def get_corpus(ctx, name):
    if name not in _CACHE:
        _CACHE.clear()  # one corpus alive at a time
        _CACHE[name] = Corpus(ctx, name)
    return _CACHE[name]


# ------------------------------------------------------------------------------------------------------------ filters
def screened_filters(c, S):
    """masks (n_filters, n) and the filter of each query; every filter has more than DIRECT_MAX_ROWS set bits.
    Each filter passes a different half of the special rows; the small corpora's filters set every skipped and removed
    row's bit."""
    rng = np.random.default_rng(zlib.crc32(f"filters/{c.name}/{S.shape[0]}".encode()))
    n, nq = c.n, S.shape[0]
    valid = c.valid
    dead_bits = c.gone if c.n < 50000 else np.zeros(n, bool)
    base = [np.ones(n, bool), rng.random(n) < 0.5]
    if c.n < 50000:
        base += [rng.random(n) < 0.05, rng.random(n) < 0.005]
        rng_mask = np.zeros(n, bool)
        rng_mask[n // 3: n // 3 + 3000] = True
        base.append(rng_mask)
        few = np.zeros(n, bool)  # fewer than k valid rows pass
        few[rng.choice(np.flatnonzero(valid), K // 2, replace=False)] = True
        base += [few, np.zeros(n, bool)]  # ... and none
    else:
        exact = np.zeros(n, bool)  # 4500 set bits: screened, and under n / 20 (the production rule's mask_hits)
        exact[rng.choice(n, 4500, replace=False)] = True
        rng_mask = np.zeros(n, bool)
        rng_mask[n // 3: n // 3 + 30000] = True
        base += [exact, rng_mask]
    masks = []
    for i, m in enumerate(base):
        m = m | dead_bits
        m[c.special] = (np.arange(c.special.size) + i) % 2 == 0
        masks.append(m)
    # the leak detector: every third query gets a filter that rejects its LEAK_ROWS best rows
    qf = np.zeros(nq, np.uint32)
    for q in range(nq):
        if q % 3 == 1:
            s = np.where(valid, S[q], -np.inf)
            m = np.ones(n, bool)
            m[np.argsort(-s, kind="stable")[:LEAK_ROWS]] = False
            m |= dead_bits
            m[c.special] = (np.arange(c.special.size) + q) % 2 == 0
            qf[q] = len(masks)
            masks.append(m)
        else:
            qf[q] = (q + q // 3) % len(base)  # neighbouring queries use different filters
    masks = np.stack(masks)
    bits = c.pack(masks)
    set_bits = np.array([int(np.unpackbits(b.view(np.uint8)).sum()) for b in bits])
    assert (set_bits > DIRECT_MAX_ROWS).all(), set_bits
    return masks, bits, qf


# ------------------------------------------------------------------------------------------------------------ checks
def check_score_all(c, S, o, passing, tc):
    """(a) every valid passing row with its unfiltered score; rejected rows NaN (tensor cores) or absent (SIMT)"""
    n = c.n
    for q in range(S.shape[0]):
        m = o["n_a"][q]
        rows = o["a"][q, :m, 0].astype(np.int64)
        sc = o["a"][q, :m, 1].view(np.float32)
        keep = rows < n
        rows, sc = rows[keep], sc[keep]
        assert rows.size == np.unique(rows).size, (q, "a row twice in the pass-0 list")
        ps = passing[q][rows]
        if tc:
            assert rows.size == n, (q, "pass 0 wrote", rows.size, "of", n, "rows")
            assert np.isnan(sc[~ps]).all(), (q, "a rejected row kept its score", rows[~ps & ~np.isnan(sc)][:5])
        else:
            assert ps.all(), (q, "SIMT appended a rejected row", rows[~ps][:5])
        want = np.flatnonzero(c.valid & passing[q])
        got = rows[ps & c.valid[rows]]
        assert np.array_equal(np.sort(got), want), (q, "valid passing rows missing", np.setdiff1d(want, got)[:5])
        sel = ps & c.valid[rows]
        assert np.array_equal(sc[sel].view(np.uint32), S[q, rows[sel]].view(np.uint32)), (q, "score differs")


def check_production(c, Q, S, o, passing, screen, cap, audit_rows=None, stage="production"):
    """(b)-(f) for every query of one production batch; returns the proven queries kept for the audit"""
    n = c.n
    int8 = screen == "TC_INT8"
    refined = screen != "SIMT_F32"
    audit = []
    for q in range(Q.shape[0]):
        if o["qflags"][q] & 1:  # zero / non-finite query norm: the exact kernel ranks it
            continue
        ok = c.valid & passing[q]
        tau = np.float32(o["tau"][q])
        n_a = o["n_a"][q]
        rows_a = o["a"][q, :n_a, 0].astype(np.int64)
        sc_a = o["a"][q, :n_a, 1].view(np.float32)
        ctx_ = (stage, screen, q, float(tau))
        # (b) stage A
        assert rows_a.size == np.unique(rows_a).size, (ctx_, "duplicate candidates")
        assert (rows_a < n).all() and ok[rows_a].all(), (ctx_, "a rejected, skipped, removed or special row kept",
                                                         rows_a[~ok[np.minimum(rows_a, n - 1)]][:5])
        assert np.array_equal(sc_a.view(np.uint32), S[q, rows_a].view(np.uint32)), (ctx_, "kept score differs")
        overflow = o["gathered"][q] > cap
        assert bool(o["flags"][q] & 1) == overflow, (ctx_, o["flags"][q], o["gathered"][q])
        sq = S[q, ok].astype(np.float64)
        if not overflow:
            thr = np.ceil(np.float64(tau)) if int8 else np.float64(tau)
            want = np.flatnonzero(ok)[sq >= thr]
            assert np.array_equal(np.sort(rows_a), want), (ctx_, "kept set", rows_a.size, want.size,
                                                           np.setdiff1d(want, rows_a)[:5], np.setdiff1d(rows_a, want)[:5])
        # (c) the threshold against the k-th best PASSING score
        if sq.size >= K:
            if tau > -np.inf:
                s_k = np.sort(sq)[::-1][K - 1]
                lim = np.nextafter(s_k - np.float64(o["margin"][q]), np.inf)
                assert np.float64(tau) <= lim, (ctx_, "tau above the k-th best passing score - margin", float(s_k),
                                                float(o["margin"][q]))
        elif not overflow:
            assert np.array_equal(np.sort(rows_a), np.flatnonzero(ok)), (ctx_, "fewer than k pass: all are kept")
        # (d) stage B
        n_b = o["n_b"][q]
        rows_b = o["b"][q, :n_b, 0].astype(np.int64)
        sc_b = o["b"][q, :n_b, 1].view(np.float32)
        spec_q = c.special[passing[q][c.special]]
        is_sp = np.isin(rows_b, c.special)
        assert (sc_b[is_sp] == np.inf).all(), (ctx_, "a special row without its +inf score")
        scr_b = rows_b[~is_sp]
        if refined:
            r_a = o["a"][q, :n_a, 2].view(np.float32)
            if n_a:
                dev, lim = c.stage_b_deviation(Q, q, rows_a, r_a, o)
                assert (dev <= lim).all(), (ctx_, "stage B error above beps2", dev.max(), lim)
            tau2 = np.float32(o["tau2"][q])
            assert np.array_equal(np.sort(scr_b), np.sort(rows_a[r_a >= tau2])), (ctx_, "stage-B kept set")
            order = {r: i for i, r in enumerate(rows_a.tolist())}
            assert np.array_equal(sc_b[~is_sp], r_a[[order[r] for r in scr_b.tolist()]]), (ctx_, "stage-B scores")
        else:
            tau2 = np.float32(-np.inf)
            assert np.array_equal(np.sort(scr_b), np.sort(rows_a)), (ctx_, "SIMT: stage B = stage A")
        # (e) the re-rank set: stage B plus exactly the query's passing special rows
        assert np.array_equal(np.sort(rows_b[is_sp]), spec_q), (ctx_, "special rows", rows_b[is_sp], spec_q)
        rr = o["rr"][q, : o["n_e"][q]].astype(np.int64)
        assert o["n_e"][q] == n_b and np.array_equal(np.sort(rr), np.sort(rows_b)), (ctx_, "re-ranked rows")
        if not (o["flags"][q] & 2) and tau > -np.inf and len(audit) < 6:
            audit.append((q, rows_a, rr, tau, tau2))
    # (f) proof audit against exact distances
    if audit:
        D = c.exact_distance(Q[[a[0] for a in audit]])
        for (q, rows_a, rr, tau, tau2), d in zip(audit, D):
            bound_a, bound_b = c.proof_bounds(o, q)
            in_a = np.zeros(n, bool)
            in_a[rows_a] = True
            out = c.valid & passing[q]
            out[rr] = False
            bound = np.where(in_a, bound_b if tau2 > -np.inf else -np.inf, bound_a)
            with np.errstate(invalid="ignore"):
                bad = np.flatnonzero(out & (d < bound))
            assert bad.size == 0, (stage, screen, q, "excluded row inside the proof's bound", bad[:5].tolist(),
                                   d[bad[:5]].tolist(), np.broadcast_to(bound, (n,))[bad[:5]].tolist())


# ------------------------------------------------------------------------------------------------------------ cases
# (corpus, screen, streaming, nq, cand_cap)
CASES = [
    ("cos_f32_d64", "TC_INT8", True, 5, 4096),
    ("cos_f32_d64", "TC_INT8", True, 65, 4096),     # one 128-query block: the one-CTA int8 launch
    ("cos_f32_d64", "TC_INT8", True, 256, 4096),    # two blocks: the 2-CTA cluster streaming launch
    ("cos_f32_d64", "TC_INT8", False, 20, 16384),
    ("cos_f32_d64", "TC_INT8", True, 2100, 4096),   # three query chunks: the qf offset, the drain ring's query tag
    ("cos_f32_d64", "TC_BF16", True, 65, 4096),
    ("cos_f32_d64", "TC_BF16", False, 3, 4096),
    ("cos_f32_d64", "TC_BF16", False, 2100, 4096),
    ("cos_f32_d64", "SIMT_F32", False, 1, 4096),    # ring kernel, QB 1, 4, 8
    ("cos_f32_d64", "SIMT_F32", False, 3, 4096),
    ("cos_f32_d64", "SIMT_F32", False, 20, 4096),
    ("cos_f32_d33", "SIMT_F32", False, 5, 4096),    # odd dim: the generic kernel
    ("cos_f32_d33", "TC_INT8", True, 65, 4096),
    ("euc_f32_d64", "TC_BF16", True, 65, 4096),
    ("euc_f32_d64", "TC_BF16", False, 20, 4096),
    ("euc_f32_d64", "SIMT_F32", False, 5, 4096),
    ("cos_f64_d64", "TC_INT8", True, 65, 4096),
    ("cos_f64_d64", "TC_BF16", False, 20, 4096),
    ("pea_f32_d48", "TC_INT8", True, 65, 4096),
    ("pea_f32_d48", "TC_INT8", False, 20, 4096),
    ("pea_f32_d48", "TC_BF16", True, 5, 4096),
    ("man_f32_d36", "SIMT_F32", False, 5, 4096),    # Lp query blocks 8, 32, 64
    ("man_f32_d36", "SIMT_F32", False, 65, 4096),
    ("man_f64_d36", "SIMT_F32", False, 20, 4096),
    ("che_f32_d35", "SIMT_F32", False, 20, 4096),
    ("che_f64_d36", "SIMT_F32", False, 5, 16384),
    ("cos_f32_fits", "TC_INT8", True, 65, 16384),
    ("cos_f32_fits", "TC_BF16", True, 5, 16384),
    ("cos_f32_big", "TC_INT8", False, 20, 4096),
    ("cos_f32_big", "TC_INT8", True, 65, 4096),
]


def _id(case):
    corpus, screen, streaming, nq, cap = case
    return f"{corpus}-{screen}-{'stream' if streaming else 'multi'}-nq{nq}-cap{cap}"


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_filtered_screen(ctx, case):
    name, screen, streaming, nq, cap = case
    c = get_corpus(ctx, name)
    Q = c.queries(nq)
    S = c.score_matrix(Q, screen)
    masks, bits, qf = screened_filters(c, S)
    passing = masks[qf]
    tc = screen != "SIMT_F32"
    # (a) the filtered pass 0
    o = c.batch(Q, screen, score_all=True, filters=bits, qf=qf)
    check_score_all(c, S, o, passing, tc)
    # (b)-(f) the production sequence; (g) every mask_hits setting of the int8 consumers
    runs = (-1, 0, 1) if screen == "TC_INT8" else (-1,)
    outs = {}
    for mh in runs:
        o = c.batch(Q, screen, streaming=streaming, cap=cap, filters=bits, qf=qf, mask_hits=mh)
        check_production(c, Q, S, o, passing, screen, cap, stage=f"mask_hits={mh}")
        outs[mh] = o
    if not streaming and len(runs) > 1:  # deterministic schedule: the switch changes nothing
        ref = outs[-1]
        for mh in (0, 1):
            o = outs[mh]
            assert np.array_equal(o["tau"].view(np.uint32), ref["tau"].view(np.uint32)), (mh, "tau differs")
            for q in range(nq):
                a = np.sort(o["a"][q, : o["n_a"][q], 0])
                b = np.sort(ref["a"][q, : ref["n_a"][q], 0])
                assert np.array_equal(a, b), (mh, q, "stage-A set differs")


# ------------------------------------------------------------------------------------------------------------ direct
@pytest.mark.parametrize("name,screen", [("cos_f32_d64", "TC_INT8"), ("pea_f32_d48", "TC_BF16"),
                                         ("man_f64_d36", "SIMT_F32"), ("euc_f32_d64", "TC_BF16")])
def test_direct_regime(ctx, name, screen):
    c = get_corpus(ctx, name)
    n = c.n
    rng = np.random.default_rng(zlib.crc32(f"direct/{name}".encode()))
    pad_bits = (32 - n % 32) % 32
    ms = []
    m = rng.random(n) < 0.005
    ms.append(m)
    m = np.zeros(n, bool)  # a row range
    m[n // 2: n // 2 + 2000] = True
    ms.append(m)
    m = np.zeros(n, bool)  # fewer than k rows
    m[rng.choice(n, 3, replace=False)] = True
    ms.append(m)
    ms.append(np.zeros(n, bool))  # none
    m = np.zeros(n, bool)  # exactly DIRECT_MAX_ROWS set bits, counting the skipped and removed rows and the padding
    dead = np.flatnonzero(c.gone)[:1000]
    m[dead] = True
    live = np.setdiff1d(np.arange(n), np.concatenate([dead, c.special]))
    m[rng.choice(live, DIRECT_MAX_ROWS - pad_bits - dead.size - c.special.size // 2, replace=False)] = True
    ms.append(m)
    for i, m in enumerate(ms):
        m[c.special] = (np.arange(c.special.size) + i) % 2 == 0
    masks = np.stack(ms)
    bits = c.pack(masks)
    set_bits = np.array([int(np.unpackbits(b.view(np.uint8)).sum()) for b in bits])
    assert set_bits.max() == DIRECT_MAX_ROWS, set_bits
    nq = 12
    Q = c.queries(nq)
    qf = (np.arange(nq) % masks.shape[0]).astype(np.uint32)
    o = c.batch(Q, screen, streaming=True, filters=bits, qf=qf)
    for q in range(nq):
        want = np.flatnonzero(masks[qf[q]] & ~c.gone)
        rows = o["a"][q, : o["n_a"][q], 0].astype(np.int64)
        assert rows.size == np.unique(rows).size, (q, "a row twice")
        assert np.array_equal(np.sort(rows), want), (q, "direct list", np.setdiff1d(want, rows)[:5],
                                                     np.setdiff1d(rows, want)[:5])
        assert (o["a"][q, : o["n_a"][q], 1].view(np.float32) == np.inf).all()
        assert o["tau"][q] == -np.inf and o["gathered"][q] == 0 and not (o["flags"][q] & 1), q
        assert o["n_b"][q] == o["n_a"][q] and o["n_e"][q] == o["n_a"][q], q
        assert np.array_equal(np.sort(o["rr"][q, : o["n_e"][q]].astype(np.int64)), want), q
    # the same batch through the production call: no screen pass, and the answers of the direct lists
    rows, dist, cnt = c.col.knn(Q, K, filters=bits, query_filter=qf)
    st = c.col.stats()
    assert st["n_passes"] == 0 and st["screen_used"] == 3, st  # SDB_SCREEN_NONE_EXACT
    for q in range(0, nq, 5):
        r, d = O.knn_topk(c.X, Q[q], c.metric.lower(), K, skip=(~masks[qf[q]] | c.gone).astype(np.uint8))
        assert cnt[q] == r.size and rows[q, : cnt[q]].tolist() == r.tolist(), q


def test_mixed_batch_is_refused(ctx):
    from surrealdb_b200 import _lib as L
    c = get_corpus(ctx, "cos_f32_d64")
    masks = np.stack([np.ones(c.n, bool), np.zeros(c.n, bool)])
    Q = c.queries(4)
    qf = np.array([0, 1, 0, 1], np.uint32)
    with pytest.raises(L.SdbError) as e:
        c.batch(Q, "TC_INT8", filters=c.pack(masks), qf=qf)
    assert e.value.status == L.SDB_EUNSUPPORTED
    o = c.batch(Q, "TC_INT8", score_all=True, filters=c.pack(masks), qf=qf)  # pass 0 has no lists to mix
    assert (o["n_a"] > 0).all()
