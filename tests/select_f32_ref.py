"""CPU restatement of hnsw_select_kernel (surrealdb_b200/csrc/hnsw.cu), the F32 COSINE / EUCLIDEAN neighbour selection
of the GPU builder (sdb_hnsw_select_neighbors[_ids]), op for op:

  fmaf(a, b, c)                  RN_f32(a * b + c), exact: the f64 sum is rounded to odd before it is narrowed, so it is
                                 never rounded twice
  lane_sum / butterfly           warp_pair_dist: lane l folds columns l, l + 32, ... with fmaf; the lanes combine by the
                                 xor butterfly 16, 8, 4, 2, 1 (f32 adds, the same value in every lane)
  norms(X)                       qn2 / en2 / n2: the same fold of x * x
  Dist                           one distance: cosine 1 - dot * rsqrtf(a_n2 * n2), euclidean the squared distance
  select(X, elem, cand, ...)     the selection -> (picks, decided)

rsqrtf is not correctly rounded (CUDA C programming guide: 2 ulp).  A cosine distance is therefore held as the set of
values 1 - dot * r takes for every f32 r within 2 ulp of 1 / sqrt(p); two distances whose products p are bit-identical
share r.  A comparison whose outcome is not the same for every admissible r is undecided, and so is the selection
that made it: select() then returns decided = False.  Euclidean distances are exact.

Contraction, as nvcc 12.9 compiles hnsw.cu for sm_90a (cuobjdump -sass of hnsw_select_kernel<true>): the distances
of the visiting order (s_d) and every r_dist are one FFMA, 1 + (-dot) * r rounded once; the e_dist the acceptance
loop recomputes for each visited candidate is FMUL then FADD, 1 - RN(dot * r), rounded twice.  So with
presorted = 0 a candidate is ranked by one value and tested by another.  rsqrtf is MUFU.RSQ, with inputs below
2^-126 scaled by 2^24 first and the result by 2^12 after.

The visiting order with presorted = 0 is rank(j) = #{t : d_t before d_j} in the total order of the kernel: numbers by
value, equal numbers in list order, NaN after every number (the element's 3.0e38 marker and +inf included), NaNs in
list order.  rank_old() keeps the rule the kernel had before, under which a NaN gets rank 0 and no number counts it.
"""
import numpy as np

F32 = np.float32
F64 = np.float64
SELF_MARK = F32(3.0e38)
RSQRT_ULP = 2


def fmaf(a, b, c):
    """fmaf elementwise on f32 arrays, exactly: a * b is exact in f64 (24 + 24 bits); the f64 sum is made
    round-to-odd with its TwoSum error, and narrowing a round-to-odd value with more than 2 extra bits rounds once"""
    a, b, c = np.broadcast_arrays(np.asarray(a, F32), np.asarray(b, F32), np.asarray(c, F32))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a.astype(F64) * b.astype(F64)
        cd = c.astype(F64)
        s = p + cd
        bb = s - p
        e = (p - (s - bb)) + (cd - bb)
        even = (s.view(np.int64) & 1) == 0
        fix = np.isfinite(s) & (e != 0) & even
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


def lane_sums(A, B):
    """(n, dim) x (n, dim) f32 -> (n, 32): lane l's fmaf chain over columns l, l + 32, ..."""
    n, dim = A.shape
    acc = np.zeros((n, 32), F32)
    for c0 in range(0, dim, 32):
        w = min(32, dim - c0)
        acc[:, :w] = fmaf(A[:, c0 : c0 + w], B[:, c0 : c0 + w], acc[:, :w])
    return acc


_PARTNER = {o: np.arange(32) ^ o for o in (16, 8, 4, 2, 1)}


def butterfly(v):
    """(n, 32) -> (n,): v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1 (lane 0's value; every lane ends equal)"""
    v = np.asarray(v, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for o in (16, 8, 4, 2, 1):
            v = v + v[:, _PARTNER[o]]
    return v[:, 0]


def norms(X):
    """qn2 / en2 of every row"""
    X = np.atleast_2d(np.asarray(X, F32))
    return butterfly(lane_sums(X, X))


def ulp32(x):
    """the spacing of f32 values at |x| (normal range; the subnormal spacing below it)"""
    _, e = np.frexp(np.abs(np.asarray(x, F64)))
    return np.ldexp(1.0, np.maximum(e - 24, -149))


def rsqrt_window(p):
    """(m,) f32 products -> (m, 7) f32: every f32 r within RSQRT_ULP ulp of 1/sqrt(p) (rows padded with repeats);
    0, inf and NaN are exact (inf, 0, NaN)"""
    p = np.asarray(p, F32)
    pd = p.astype(F64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = 1.0 / np.sqrt(pd)  # f64: within 1 ulp of the exact value
    lo = r * (1 - 2.0 ** -51) - RSQRT_ULP * ulp32(r)
    hi = r * (1 + 2.0 ** -51) + RSQRT_ULP * ulp32(r)
    r0 = r.astype(F32)
    steps = [r0]
    up, dn = r0, r0
    for _ in range(3):
        up = np.nextafter(up, F32(np.inf))
        dn = np.nextafter(dn, F32(0))
        steps += [up, dn]
    W = np.stack(steps, 1)
    with np.errstate(invalid="ignore"):
        ok = (W.astype(F64) >= lo[:, None]) & (W.astype(F64) <= hi[:, None])
    ok[:, 0] |= ~ok.any(1)  # r0 itself is always admissible
    W = np.where(ok, W, r0[:, None])
    exact = ~np.isfinite(r) | (pd == 0) | ~np.isfinite(pd)
    return np.where(exact[:, None], r0[:, None], W)


class Dist:
    """distances from one staged vector a (the kernel's s_q or s_e, with its norm) to the rows B: vals (m, 7) are the
    values each can take (all equal when exact), p (m,) the f32 products under the rsqrtf (None: euclidean)"""

    def __init__(self, a, a_n2, B, cosine, fused=True):
        B = np.atleast_2d(np.asarray(B, F32))
        a = np.broadcast_to(np.asarray(a, F32), B.shape)
        if cosine:
            dot = butterfly(lane_sums(a, B))
            with np.errstate(over="ignore", invalid="ignore"):
                self.p = F32(a_n2) * norms(B)
                W = rsqrt_window(self.p)
                if fused:  # FFMA d, -dot, rsq, 1
                    self.vals = fmaf(-dot[:, None], W, F32(1.0))
                else:  # FMUL t, dot, rsq; FADD d, -t, 1
                    self.vals = F32(1.0) - dot[:, None] * W
        else:
            with np.errstate(over="ignore", invalid="ignore"):
                d = a - B
            self.p = None
            self.vals = np.repeat(butterfly(lane_sums(d, d))[:, None], 7, 1)


def gt(x, px, Y, pY):
    """x > Y[i] for every i, x (7,), Y (m, 7) -> (outcome at the first admissible values (m,) bool, decided (m,) bool):
    decided when every admissible pair of values gives the same outcome; a shared product shares r"""
    with np.errstate(invalid="ignore"):
        every = x[None, :, None] > Y[:, None, :]  # (m, 7, 7): every pair of admissible values
        diag = x[None, :] > Y  # the same r on both sides
    shared = np.zeros(Y.shape[0], bool) if px is None else (pY.view(np.int32) == px.view(np.int32))
    all_ = np.where(shared, diag.all(1), every.all((1, 2)))
    any_ = np.where(shared, diag.any(1), every.any((1, 2)))
    with np.errstate(invalid="ignore"):
        return x[0] > Y[:, 0], all_ == any_


def rank_fixed(d):
    """s_ord of the fixed kernel for distances d (f32, the element's slots holding SELF_MARK): rank(j) = #{t : d_t < d_j,
    or equal numbers with t < j, or d_t a number and d_j NaN, or both NaN with t < j}"""
    d = np.asarray(d, F32)
    nc = d.size
    ord_ = np.full(nc, -1, np.int64)
    nan = np.isnan(d)
    t = np.arange(nc)
    for j in range(nc):
        with np.errstate(invalid="ignore"):
            before = np.where(nan == nan[j], (d < d[j]) | (((d == d[j]) | nan[j]) & (t < j)), nan[j])
        ord_[before.sum()] = j
    return ord_


def rank_old(d):
    """s_ord of the kernel before the fix: rank(j) = #{t : d_t < d_j or (d_t == d_j and t < j)}; -1 marks a slot no
    entry wrote"""
    d = np.asarray(d, F32)
    nc = d.size
    ord_ = np.full(nc, -1, np.int64)
    t = np.arange(nc)
    for j in range(nc):
        with np.errstate(invalid="ignore"):
            ord_[((d < d[j]) | ((d == d[j]) & (t < j))).sum()] = j
    return ord_


def select(X, elem, cand, m_max, presorted, cosine):
    """hnsw_select_kernel for element `elem` (a row of X) over the candidate rows `cand` -> (picks, decided).
    decided = False when a comparison on the way could go either way within rsqrtf's error (the picks then follow
    the nearest f32 to 1 / sqrt(p))."""
    X = np.asarray(X, F32)
    cand = np.asarray(cand, np.int64)
    nc = cand.size
    q = X[elem]
    qn2 = norms(q[None, :])[0]
    real = cand != elem
    take_all = int(real.sum()) <= m_max
    decided = True
    # the distances of the visiting order (fused), and e_dist as the acceptance loop recomputes it (not fused)
    ed = Dist(q, qn2, X[cand], cosine) if nc else None
    ea = Dist(q, qn2, X[cand], cosine, fused=False) if nc else None
    if presorted:
        visit = [j for j in range(nc) if real[j]]
    else:
        v = np.where(real, ed.vals[:, 0], SELF_MARK)
        visit = [j for j in rank_fixed(v) if real[j]]
        # the order is decided iff no two numbers could swap: with one product (one r) the pair must compare alike at
        # every admissible r; with two, their value ranges must not overlap
        r = np.nonzero(real & ~np.isnan(ed.vals[:, 0]))[0]
        if cosine and r.size > 1:
            V = ed.vals[r]
            lo, hi = V.min(1), V.max(1)
            apart = (hi[:, None] < lo[None, :]) | (hi[None, :] < lo[:, None])
            lt, gt_, eq = V[:, None, :] < V[None, :, :], V[:, None, :] > V[None, :, :], V[:, None, :] == V[None, :, :]
            alike = lt.all(-1) | gt_.all(-1) | eq.all(-1)
            shared = ed.p[r].view(np.int32)[:, None] == ed.p[r].view(np.int32)[None, :]
            if not np.where(shared, alike, apart | alike & eq.all(-1)).all():
                decided = False
    acc = []
    for j in visit:
        if len(acc) >= m_max:
            break
        e = int(cand[j])
        if not take_all and acc:
            en2 = norms(X[e][None, :])[0]
            rd = Dist(X[e], en2, X[np.array(acc)], cosine)
            out, ok = gt(ea.vals[j], None if ea.p is None else ea.p[j], rd.vals, rd.p)
            if not (out & ok).any() and not ok.all():  # neither a sure rejection nor a sure acceptance
                decided = False
            if out.any():
                continue
        acc.append(e)
    return acc, decided
