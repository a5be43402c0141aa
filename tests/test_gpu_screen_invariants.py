"""Invariants of the brute-force screens, each held against a plain reference (tests/screen_ref.py), through the
test-only entry points sdb_debug_corpus_state / sdb_debug_screen_batch.

The exactness proof of cand_final_kernel is sound only if (1) every valid row whose screen score reaches the query's
final tau is a candidate, (2) every screened score is within beps of the exact one, and (3) tau never exceeds
(k-th best score) - margin.  The end-to-end parity tests see a broken link only when it happens to move a true
neighbour; these tests look at each link directly:

  operand copies   the int8 / bf16 copies of rows and queries equal the restatement bit for bit; their measured residuals
                   stay within the figures the bounds use
  score matrix     one pass-0 launch over every tile: int8 scores are the exact integer dot products, bf16 and f32 scores
                   stay within their accumulation terms (the largest bf16 ratio to D * 2^-21 * sum|q_i x_i| is printed)
  bounds           |screened - exact| <= beps for every valid (query, row) pair, and beps is at least cand_begin's formula
  stage A / B      kept sets, scores, overflow flags and thresholds of the production sequence (streaming and
                   multi-pass schedules) against the score matrix
  proof audit      every valid row outside the re-ranked set of a proven query is at least the proof's bound away
"""
import ctypes as C

import numpy as np
import pytest

import screen_ref as R
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

CAP = 4096
SPECIAL_CAP = 1024
SCREEN_CODE = {"SIMT_F32": 1, "TC_BF16": 2, "TC_INT8": 4}
F32_NAN = np.float32(np.nan)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


# ---------------------------------------------------------------------------------------------------------- data
def _uniform(rng, n, dim):
    return rng.uniform(-1, 1, (n, dim)).astype(np.float32)


def _clustered(rng, n, dim):
    # 40 tight clusters stored one after another: a CTA's tiles hold one cluster, so its private sub-lists spill
    centers = rng.uniform(-1, 1, (40, dim))
    lab = np.sort(rng.integers(0, 40, n))
    return (centers[lab] + rng.normal(0, 0.03, (n, dim))).astype(np.float32)


def _crowd(rng, n, dim):
    # 5000 near-duplicates of one row: more candidates than the lists hold
    x = _uniform(rng, n, dim)
    x[1000:6000] = x[0] + rng.normal(0, 1e-5, (5000, dim)).astype(np.float32)
    return x


def _midpoints(rng, n, dim):
    # every component exactly halfway between two bf16 values (odd and even low bits): ties to even in both directions
    hi = rng.integers(0x3C00, 0x4000, (n, dim)).astype(np.uint32) | (rng.integers(0, 2, (n, dim)).astype(np.uint32) << 15)
    return ((hi << 16) | 0x8000).view(np.float32)


def _binades(rng, n, dim):
    # magnitudes over 40 binades with alternating signs: the tensor cores align every product of a K-group to the
    # largest one, so the small ones lose their low bits
    mag = np.exp2(rng.uniform(-20, 20, (n, dim))) * rng.uniform(1, 2, (n, dim))
    sign = np.where(np.arange(dim) % 2 == 0, 1.0, -1.0)
    return (mag * sign).astype(np.float32)


def _positive(rng, n, dim):
    return rng.uniform(0, 1, (n, dim)).astype(np.float32)


INVALID_SPECIAL = [3, 500, 7001, 11, 12, 20, 4000, 9000, 15000, 19999]


def _invalid(rng, n, dim):
    # zero / NaN / inf rows are special; five rows with one dominant component are int8 outliers (gap rule)
    x = _uniform(rng, n, dim)
    x[INVALID_SPECIAL[:3]] = 0.0
    x[11, 5] = np.nan
    x[12, 0] = np.inf
    for i, r in enumerate(INVALID_SPECIAL[5:]):
        x[r] = rng.uniform(-1e-3, 1e-3, dim)
        x[r, i] = 40.0
    return x


# name: (generator, n, dim, nq, k, metric, queries near rows, screens)
CASES = {
    "d1_uniform": (_uniform, 257, 1, 65, 10, "COSINE", True, None),
    "d7_uniform_euclid": (_uniform, 255, 7, 1, 1, "EUCLIDEAN", True, None),
    "d127_midpoints": (_midpoints, 256, 127, 129, 100, "COSINE", True, None),
    "d128_clustered": (_clustered, 20000, 128, 300, 10, "COSINE", True, None),
    "d129_one_row_euclid": (_uniform, 1, 129, 65, 10, "EUCLIDEAN", False, None),
    "d768_invalid_rows": (_invalid, 20000, 768, 129, 256, "COSINE", True, None),
    "d768_negative_kth": (_positive, 6000, 768, 65, 10, "COSINE", False, None),
    "d1536_crowd_euclid": (_crowd, 8000, 1536, 65, 100, "EUCLIDEAN", True, None),
    "d4100_binades": (_binades, 2000, 4100, 1, 10, "COSINE", True, None),
    "d128_chunked": (_uniform, 20000, 128, 2100, 10, "COSINE", True, ("TC_INT8", "TC_BF16")),
}


def _screens(case):
    metric, screens = CASES[case][5], CASES[case][7]
    if screens:
        return screens
    return ("TC_INT8", "TC_BF16", "SIMT_F32") if metric == "COSINE" else ("TC_BF16", "SIMT_F32")


class Case:
    def __init__(self, ctx, name):
        from surrealdb_b200 import VectorColumn
        from surrealdb_b200 import _lib as L
        gen, n, dim, nq, k, metric, near, _ = CASES[name]
        rng = np.random.default_rng(sum(map(ord, name)))
        self.name, self.n, self.dim, self.k, self.metric = name, n, dim, k, metric
        self.X = gen(rng, n, dim)
        if name == "d768_negative_kth":
            Q = -rng.uniform(0, 1, (nq, dim))  # every similarity is negative
        elif near:
            Q = self.X[rng.integers(0, n, nq)].astype(np.float64) * rng.uniform(0.5, 2.0, (nq, 1))
            Q += rng.normal(0, 1e-3, Q.shape) * np.abs(Q).max(axis=1, keepdims=True)
            Q[::3] = rng.uniform(-1, 1, Q[::3].shape)
            Q[~np.isfinite(Q).all(axis=1)] = 0.5
        else:
            Q = rng.uniform(-1, 1, (nq, dim))
        self.Q = np.ascontiguousarray(Q, np.float64)
        self.col = VectorColumn(ctx, dim, metric, "F32", capacity=n)
        self.col.append(self.X)
        self.skip = np.zeros(n, np.uint8)
        if name == "d768_invalid_rows":  # (the special rows of _invalid stay unskipped)
            self.skip[rng.integers(0, n, n // 10)] = 1
            self.skip[INVALID_SPECIAL] = 0
            self.col.set_skip(self.skip)
        self.col.finalize()
        if name == "d768_invalid_rows":  # tombstones after finalize: NaN screening norm and an all-zero int8 row
            dead = np.setdiff1d(np.unique(rng.integers(0, n, 300)), INVALID_SPECIAL)
            self.col.remove(dead)
            self.skip[dead] = 1
        self.L = L
        lib = L.lib()
        f = np.zeros(4, np.float32)
        u = np.zeros(5, np.uint32)
        L.check(lib.sdb_debug_corpus_state(self.col.h, _p(f), _p(u), None, None, None, None))
        self.i8_scale, self.max_rel_qerr, self.bf16_rel_err, self.max_norm = (np.float32(v) for v in f)
        self.n_special, self.n_outliers, self.dim_pad, self.dim_pad8, self.n_pad = (int(v) for v in u)
        cos = metric == "COSINE"
        self.x8 = np.zeros((self.n_pad, self.dim_pad8), np.int8) if cos else None
        self.xbf = np.zeros((self.n_pad, self.dim_pad), np.uint16)
        self.snorm = np.zeros(self.n_pad, np.float32)
        self.special = np.zeros(max(self.n_special, 1), np.uint32)
        L.check(lib.sdb_debug_corpus_state(self.col.h, None, None, _p(self.x8), _p(self.xbf), _p(self.snorm),
                                           _p(self.special)))
        self.special = self.special[: self.n_special]
        self.valid = ~np.isnan(self.snorm[:n])
        self.mag = R.magnitude(self.X)
        self._all = {}

    def batch(self, screen, streaming=True, score_all=False, cap=CAP):
        nq = self.Q.shape[0]
        capq = max(cap, self.n_pad) if score_all else cap
        out = dict(qf=np.zeros((nq, 9), np.float32), qmag=np.zeros(nq), qu=np.zeros((nq, 6), np.uint32),
                   q8=np.zeros((nq, self.dim_pad8), np.int8), qbf=np.zeros((nq, self.dim_pad), np.uint16),
                   a=np.zeros((nq, capq, 3), np.uint32))
        if not score_all:
            out["b"] = np.zeros((nq, capq, 2), np.uint32)
            out["rr"] = np.zeros((nq, capq + SPECIAL_CAP), np.uint32)
        self.L.check(self.L.lib().sdb_debug_screen_batch(
            self.col.h, _p(self.Q), nq, self.k, SCREEN_CODE[screen], int(streaming), cap, int(score_all),
            _p(out["qf"]), _p(out["qmag"]), _p(out["qu"]), _p(out["q8"]), _p(out["qbf"]), _p(out["a"]),
            _p(out.get("b")), _p(out.get("rr"))))
        for j, name in enumerate(("tau", "margin", "bscale", "beps", "tau2", "beps2", "q8scale", "q8err", "qbferr")):
            out[name] = out["qf"][:, j]
        for j, name in enumerate(("flags", "qflags", "gathered", "n_a", "n_b", "n_e")):
            out[name] = out["qu"][:, j].astype(np.int64)
        return out

    def score_matrix(self, screen):
        """[nq][n] scores of one pass-0 launch of the screen (NaN: the row is not a screen candidate)."""
        if screen not in self._all:
            o = self.batch(screen, score_all=True)
            S = np.full((self.Q.shape[0], self.n), F32_NAN, np.float32)
            for q in range(S.shape[0]):
                m = o["n_a"][q]
                rows = o["a"][q, :m, 0]
                keep = rows < self.n
                S[q, rows[keep]] = o["a"][q, :m, 1][keep].view(np.float32)
            S[:, ~self.valid] = F32_NAN
            self._all[screen] = (S, o)
        return self._all[screen]

    def exact(self):
        """[nq][n] exact f64 similarity (cosine) or 2 q.x - |x|^2 (euclidean)."""
        if "exact" not in self._all:
            f = R.cosine_sim if self.metric == "COSINE" else R.euclid_score
            with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
                self._all["exact"] = f(self.Q, self.X)
        return self._all["exact"]


_CACHE = {}


@pytest.fixture(scope="module")
def ctx():
    from surrealdb_b200 import Context
    return Context(0)


def get_case(ctx, name):
    if name not in _CACHE:
        _CACHE.clear()  # one corpus (and its score matrices) alive at a time
        _CACHE[name] = Case(ctx, name)
    return _CACHE[name]


# ---------------------------------------------------------------------------------------------------- operand copies
@pytest.mark.parametrize("case", list(CASES))
def test_operand_copies(ctx, case):
    c = get_case(ctx, case)
    n, dim, v = c.n, c.dim, c.valid
    # validity: skipped / tombstoned / zero / non-finite rows and outliers are NaN in snorm, padding rows too
    finite = np.isfinite(c.X).all(axis=1) & (c.mag > 0) & np.isfinite(c.mag)
    if c.metric == "EUCLIDEAN":
        finite = np.isfinite(c.X).all(axis=1) & np.isfinite((c.mag * c.mag).astype(np.float32))
    assert not (v & (c.skip != 0)).any() and not (v & ~finite).any()
    assert np.isnan(c.snorm[n:]).all()
    special = set(c.special.tolist())
    assert special == set(np.flatnonzero(~v & (c.skip == 0)).tolist()), "special rows = invalid rows not skipped"
    if case == "d768_invalid_rows":
        assert c.n_outliers == 5 and c.n_special == 5 + 5
    with np.errstate(divide="ignore"):
        want_sn = (1.0 / c.mag).astype(np.float32) if c.metric == "COSINE" else (c.mag * c.mag).astype(np.float32)
    # (euclid snorm is (float)sum x^2: the square of the f64 magnitude can differ from the sum in the last f64 bit)
    if c.metric == "COSINE":
        assert np.array_equal(c.snorm[:n][v], want_sn[v])
    else:
        assert np.allclose(c.snorm[:n][v], want_sn[v], rtol=2**-23, atol=0)
    # bf16 copy: round to nearest even of every row (valid or not; a NaN stays a NaN), zero padding
    nan = np.isnan(c.X)
    assert np.array_equal(c.xbf[:n, :dim][~nan], R.bf16_rne(c.X[~nan]))
    assert np.isnan(R.bf16_to_f32(c.xbf[:n, :dim][nan])).all()
    assert not c.xbf[:, dim:].any() and not c.xbf[n:].any()
    xb = R.bf16_to_f32(c.xbf[:n, :dim]).astype(np.float64)
    res_bf = np.linalg.norm(c.X[v].astype(np.float64) - xb[v], axis=1) / c.mag[v]
    if v.any():
        assert res_bf.max() <= c.bf16_rel_err, (res_bf.max(), c.bf16_rel_err)
    # int8 copy: the restatement on valid rows, all-zero elsewhere (invalid, padding rows and columns)
    if c.x8 is not None:
        want8 = np.zeros((c.n_pad, c.dim_pad8), np.int8)
        if v.any():
            want8[:n][v, :dim] = R.quantize_rows(c.X[v], c.mag[v], c.i8_scale)
        bad = np.argwhere(c.x8 != want8)
        assert bad.size == 0, f"{bad.shape[0]} int8 elements differ, first {bad[:4].tolist()}"
        res8 = np.linalg.norm(c.X[v].astype(np.float64) / c.mag[v, None] - np.float64(c.i8_scale) * c.x8[:n][v, :dim],
                              axis=1)
        if v.any():
            assert res8.max() <= c.max_rel_qerr, (res8.max(), c.max_rel_qerr)
    # query copies and their residuals
    o = c.batch(_screens(case)[0], score_all=True)
    q32 = c.Q.astype(np.float32)
    assert np.array_equal(o["qbf"][:, :dim], R.bf16_rne(q32)) and not o["qbf"][:, dim:].any()
    qmag = R.magnitude(c.Q)
    assert np.array_equal(o["qmag"], qmag)
    qres = np.linalg.norm(c.Q - R.bf16_to_f32(o["qbf"][:, :dim]), axis=1) / qmag
    assert (qres <= o["qbferr"]).all(), np.max(qres - o["qbferr"])
    if c.x8 is not None:
        q8, s = R.quantize_queries(q32)
        assert np.array_equal(o["q8scale"], s)
        assert np.array_equal(o["q8"][:, :dim], q8) and not o["q8"][:, dim:].any()
        qres8 = np.linalg.norm(c.Q - s[:, None].astype(np.float64) * q8, axis=1) / qmag
        assert (qres8 <= o["q8err"]).all(), np.max(qres8 - o["q8err"])


# ----------------------------------------------------------------------------------------- score matrix and bounds
def _params(kind):
    out = []
    for case in CASES:
        for screen in _screens(case):
            if kind == "score":
                out.append((case, screen))
            else:
                for streaming in ((True, False) if screen != "SIMT_F32" else (False,)):
                    out.append((case, screen, streaming))
    return out


@pytest.mark.parametrize("case,screen", _params("score"))
def test_score_matrix_and_error_bounds(ctx, case, screen):
    c = get_case(ctx, case)
    S, o = c.score_matrix(screen)
    v = c.valid
    dim = c.dim
    Sv = S[:, v].astype(np.float64)
    assert not np.isnan(Sv).any(), "a valid row has no score"
    sn = c.snorm[: c.n][v].astype(np.float64)
    if screen == "TC_INT8":
        exact = o["q8"][:, :dim].astype(np.float64) @ c.x8[: c.n][v, :dim].astype(np.float64).T  # exact in f64
        assert np.array_equal(S[:, v], exact.astype(np.float32)), "int8 scores are not the integer dot products"
    else:
        if screen == "TC_BF16":
            qo = R.bf16_to_f32(o["qbf"][:, :dim]).astype(np.float64)
            xo = R.bf16_to_f32(c.xbf[: c.n][v, :dim]).astype(np.float64)
            term = dim * 2.0**-21
        else:
            qo = c.Q.astype(np.float32).astype(np.float64)
            xo = c.X[v].astype(np.float64)
            term = (dim / 16.0 + 16.0) * 2.0**-23
        dot, absdot = qo @ xo.T, np.abs(qo) @ np.abs(xo).T
        if c.metric == "COSINE":
            ref, scale = dot * sn[None, :], sn[None, :]
        else:
            ref, scale = 2.0 * dot - sn[None, :], 2.0
        err = np.abs(Sv - ref) - 2.0**-24 * np.abs(Sv)  # less the rounding of the epilogue's final multiply / fma
        allowed = term * absdot * scale
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(allowed > 0, np.maximum(err, 0.0) / allowed, np.where(err > 1e-30, np.inf, 0.0))
        worst = float(ratio.max()) if ratio.size else 0.0
        if screen == "TC_BF16":
            print(f"\n[bf16 accumulation] {case}: max |score - exact(bf16 operands)| / (D 2^-21 sum|q_i x_i|) = {worst:.4g}")
        assert worst <= 1.0, (screen, worst)
    # beps is at least cand_begin's documented bound, and that bound holds for every valid (query, row) pair
    if screen == "TC_INT8":
        eq, ex = o["q8err"], c.max_rel_qerr
    elif screen == "TC_BF16":
        eq, ex = o["qbferr"], c.bf16_rel_err
    else:
        eq, ex = np.zeros(c.Q.shape[0]), 0.0
    eps_rel = R.screen_eps_rel(screen, dim, eq.astype(np.float64), ex)
    want_beps = R.screen_beps(c.metric, eps_rel, o["qmag"], c.max_norm)
    ok_q = (o["qflags"] & 1) == 0
    assert (o["beps"][ok_q] >= want_beps[ok_q] * (1 - 1e-9)).all(), np.max(want_beps[ok_q] - o["beps"][ok_q])
    exact = c.exact()[:, v]
    if c.metric == "COSINE":
        dev = np.abs(Sv * o["bscale"][:, None].astype(np.float64) / o["qmag"][:, None] - exact)
    else:
        dev = np.abs(Sv - exact)
    dev = dev[ok_q]
    slack = dev - o["beps"][ok_q, None].astype(np.float64)
    assert (slack <= 0).all(), f"screen error above beps: {slack.max():.3g} at {np.unravel_index(slack.argmax(), slack.shape)}"


# -------------------------------------------------------------------------------------- stage A, stage B, proof
@pytest.mark.parametrize("case,screen,streaming", _params("batch"))
def test_candidates_and_proof(ctx, case, screen, streaming):
    c = get_case(ctx, case)
    S, _ = c.score_matrix(screen)
    o = c.batch(screen, streaming=streaming)
    nq, n, k = c.Q.shape[0], c.n, c.k
    v = c.valid
    if screen == "TC_INT8":  # the kernel compares the exact integer dot product with ceil(tau)
        V = o["q8"][:, : c.dim].astype(np.float64) @ c.x8[:n][v, : c.dim].astype(np.float64).T
    audit = []
    for q in range(nq):
        if o["qflags"][q] & 1:  # zero / non-finite query norm: the exact kernel ranks it, nothing to hold
            continue
        tau = np.float32(o["tau"][q])
        n_a = o["n_a"][q]
        rows_a = o["a"][q, :n_a, 0].astype(np.int64)
        sc_a = o["a"][q, :n_a, 1].view(np.float32)
        assert rows_a.size == np.unique(rows_a).size, (q, "duplicate candidates")
        assert (rows_a < n).all() and v[rows_a].all(), (q, "an invalid row is a candidate")
        assert np.array_equal(sc_a, S[q, rows_a]), (q, "kept score differs from the score matrix")
        overflow = o["gathered"][q] > CAP
        assert bool(o["flags"][q] & 1) == overflow, (q, o["flags"][q], o["gathered"][q])
        sq = S[q, v]
        if not overflow:
            if screen == "TC_INT8":
                want = np.flatnonzero(v)[V[q] >= np.ceil(np.float64(tau))]
            else:
                want = np.flatnonzero(v)[sq >= tau]
            assert np.array_equal(np.sort(rows_a), want), (q, "kept set", rows_a.size, want.size, float(tau))
        # tau never above (k-th best score) - margin
        if sq.size >= k and tau > -np.inf:
            s_k = np.sort(sq)[::-1][k - 1]
            lim = np.nextafter(np.float64(s_k) - np.float64(o["margin"][q]), np.inf)
            assert np.float64(tau) <= lim, (q, float(tau), float(s_k), float(o["margin"][q]))
        # stage B: f32 re-scores within beps2 of exact, kept set = stage-A rows whose f32 score reaches tau2
        n_b = o["n_b"][q]
        rows_b = o["b"][q, :n_b, 0].astype(np.int64)
        refined = screen != "SIMT_F32"
        if refined:
            r_a = o["a"][q, :n_a, 2].view(np.float32)
            ex = c.exact()[q, rows_a] if n_a else np.zeros(0)
            dev = np.abs(r_a / o["qmag"][q] - ex) if c.metric == "COSINE" else np.abs(r_a.astype(np.float64) - ex)
            assert (dev <= np.float64(o["beps2"][q])).all(), (q, "stage B error above beps2", dev.max())
            tau2 = np.float32(o["tau2"][q])
            want_b = rows_a[r_a >= tau2]
            assert np.array_equal(np.sort(rows_b), np.sort(want_b)), (q, "stage-B kept set")
            order = {r: i for i, r in enumerate(rows_a.tolist())}
            assert np.array_equal(o["b"][q, :n_b, 1].view(np.float32), r_a[[order[r] for r in rows_b.tolist()]])
        else:
            tau2 = np.float32(-np.inf)
            assert np.array_equal(np.sort(rows_b), np.sort(rows_a))
        rr = o["rr"][q, : o["n_e"][q]].astype(np.int64)
        assert sorted(rr.tolist()) == sorted(rows_b.tolist() + c.special.tolist()), (q, "re-ranked rows")
        if not (o["flags"][q] & 2) and tau > -np.inf and len(audit) < 8:
            audit.append((q, set(rows_a.tolist()), set(rr.tolist()), tau, tau2))
    # proof audit: a proven query's excluded rows are no closer than the bound the proof used
    if not audit:
        return
    qs = [a[0] for a in audit]
    rows, dist = O.knn_topk_batch(c.X, c.Q[qs], c.metric.lower(), n, 8)
    for (q, in_a, in_rr, tau, tau2), r, d in zip(audit, rows, dist):
        dq = np.empty(n)
        dq[r.astype(np.int64)] = d
        if c.metric == "COSINE":
            bound_a = R.proof_bound_cosine(tau, o["bscale"][q], o["qmag"][q], o["beps"][q])
            bound_b = R.proof_bound_cosine(tau2, 1.0, o["qmag"][q], o["beps2"][q])
        else:
            bound_a = R.proof_bound_euclid(tau, o["qmag"][q], o["beps"][q])
            bound_b = R.proof_bound_euclid(tau2, o["qmag"][q], o["beps2"][q])
        a_mask = np.zeros(n, bool)
        a_mask[list(in_a)] = True
        out = v.copy()
        out[list(in_rr)] = False
        # rows stage A excluded: screen score <= tau; rows stage B excluded: f32 score < tau2
        bound = np.where(a_mask, bound_b if tau2 > -np.inf else -np.inf, bound_a)
        bad = np.flatnonzero(out & (dq < bound))
        assert bad.size == 0, (q, bad[:5].tolist(), dq[bad[:5]].tolist(), bound[bad[:5]].tolist())
