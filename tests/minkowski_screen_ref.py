"""numpy restatement of the MINKOWSKI screen of integer order p (surrealdb_b200/csrc/screen_lp.cu: minkowski_fma,
minkowski_score) and of its error bound (cand_begin_minkowski_kernel in candidates.cu, DESIGN.md section 2).

  scale          s = 2^-e, e = the exponent of M + Qb (frexp: M + Qb < 2^e), at least -126; M = the largest |x^_i| of
                 a screened row, Qb = the largest |q^_i| of the batch
  screen         t_i = fl32(fl32(x^_i s) - fl32(q^_i s)); |t_i|^p by minkowski_fma's chain, the last product fused into
                 the accumulator (FFMA, computed exactly here); n~ = fl32(S~^(1/p) 2^e)
  reference      d = pow(sum_i pow(|x_i - q_i|, p), 1/p), sequential f64 over the f64 values (the exact kernel)
  bound          |n~ - d| <= beps(p, D, M, q^, e) for every screened row"""
import numpy as np

U = 2.0 ** -24
F32 = np.float32


def rounding_up_rows(n, dim):
    """rows whose f32 power sum rounds up at every step for p = 1: a first term of 1, then terms just above half an
    ulp of the accumulator (for order p the elements are the p-th roots of those terms)."""
    x = np.full((n, dim), 2.0 ** -24 * (1 + 2.0 ** -10), np.float32)
    x[:, 0] = 1.0
    return x


def max_abs(X):
    """finalize_lp_kernel's max_norm of a MINKOWSKI corpus: the largest |x^_i| (f32, exact)."""
    return F32(np.abs(np.asarray(X, np.float64).astype(F32)).max())


def batch_exponent(mnorm, q32):
    """e of the launch's scale s = 2^-e: M + Qb < 2^e over the queries whose f32 copy is finite, e >= -126."""
    q = np.abs(np.asarray(q32, F32))
    ok = np.isfinite(q).all(axis=-1)
    qb = float(q[ok].max()) if ok.any() else 0.0
    v = float(mnorm) + qb
    if v <= 0.0:
        return -126
    return max(int(np.frexp(v)[1]), -126)


def _fma32(a, b, c):
    """fl32(a * b + c) for f32 arrays, exactly rounded: a b is exact in f64 (48 bits), the f64 sum's error is
    recovered by TwoSum, and a sum that lands on an f32 midpoint is pushed the way of the error."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    r = (p - (s - bb)) + (c64 - bb)
    with np.errstate(over="ignore"):
        f = s.astype(F32)
    f64 = f.astype(np.float64)
    lo = np.where(f64 <= s, f, np.nextafter(f, F32(-np.inf)))
    hi = np.where(f64 >= s, f, np.nextafter(f, F32(np.inf)))
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) / 2
    at_mid = (s == mid) & (r != 0) & (lo != hi)
    return np.where(at_mid & (r > 0), hi, np.where(at_mid & (r < 0), lo, f))


def chain(t, p):
    """minkowski_fma's factors: |t|^p = a * b with a, b f32 (rounded products), the last product left to the FFMA."""
    t = np.asarray(t, F32)
    a = np.abs(t)
    if p == 1:
        return a, np.ones_like(a)
    if p == 2:
        return t, t
    t2 = t * t
    if p == 3:
        return t2, a
    if p == 4:
        return t2, t2
    if p == 5:
        return t2 * t2, a
    if p == 6:
        t3 = t2 * a
        return t3, t3
    if p == 7:
        return t2 * t2, t2 * a
    t4 = t2 * t2
    return t4, t4


def terms(Q, X, p, e, scale=True):
    """[nq][n][D] the chain's two f32 factors of every element (scale=False: the screen without its scale)."""
    s = F32(np.ldexp(1.0, -e)) if scale else F32(1.0)
    q = np.asarray(Q, np.float64).astype(F32) * s
    x = np.asarray(X, np.float64).astype(F32) * s
    with np.errstate(over="ignore", invalid="ignore"):
        t = x[None, :, :] - q[:, None, :]
        return chain(t, p)


def _pairwise(t):
    d = t.shape[-1]
    w = 1
    while w < d:
        w *= 2
    t = np.concatenate([t, np.zeros(t.shape[:-1] + (w - d,), F32)], axis=-1)
    while t.shape[-1] > 1:
        t = t[..., 0::2] + t[..., 1::2]
    return t[..., 0]


def _strided32(t):
    """32 lanes, lane l sums columns l, l + 32, ... sequentially, then a butterfly over the lanes."""
    d = t.shape[-1]
    t = np.concatenate([t, np.zeros(t.shape[:-1] + ((-d) % 32,), F32)], axis=-1)
    lanes = np.cumsum(t.reshape(t.shape[:-1] + (-1, 32)), axis=-2, dtype=F32)[..., -1, :]
    while lanes.shape[-1] > 1:
        h = lanes.shape[-1] // 2
        lanes = lanes[..., :h] + lanes[..., h:]
    return lanes[..., 0]


def power_sum(Q, X, p, e, order="sequential", scale=True):
    """[nq][n] f32 S~: sequential = the kernel's FFMA chain over the elements in order; pairwise / strided32 = other
    f32 summation orders of the rounded terms (the bound holds for any order)."""
    a, b = terms(Q, X, p, e, scale)
    with np.errstate(over="ignore", invalid="ignore"):
        if order == "sequential":
            acc = np.zeros(a.shape[:-1], F32)
            for i in range(a.shape[-1]):
                acc = _fma32(a[..., i], b[..., i], acc)
            return acc
        prod = a * b
    return _pairwise(prod) if order == "pairwise" else _strided32(prod)


def score_norm(S, p, e):
    """n~ = fl32(S~^(1/p) 2^e) (minkowski_score; f64 pow, one rounding to f32)."""
    S = np.asarray(S, np.float64)
    with np.errstate(over="ignore"):
        r = S if p == 1 else np.power(S, 1.0 / p)
        return np.ldexp(r, e).astype(F32)


def reference(Q, X, p):
    """[nq][n] the exact kernel's distance: acc += pow(|x_i - q_i|, p) sequentially in f64, then pow(acc, 1/p)."""
    x = np.asarray(X, np.float64)
    out = np.empty((np.asarray(Q).shape[0], x.shape[0]))
    with np.errstate(over="ignore", invalid="ignore"):
        for j, q in enumerate(np.asarray(Q, np.float64)):
            t = np.power(np.abs(x - q[None, :]), float(p))
            out[j] = np.power(np.cumsum(t, axis=-1)[..., -1], 1.0 / p)
    return out


def beps(p, dim, mnorm, q32, e, underflow=True, subnormal_rounding=True):
    """per query: cand_begin_minkowski_kernel's bound (before its rounding up to f32).  Mutants of the bound:
    underflow=False drops the underflow terms under the scale, subnormal_rounding=False the unscaled R 2^-149 of
    rounding f64 values in f32's subnormal range to f32."""
    q = np.abs(np.asarray(q32, F32).astype(np.float64))
    D, P, up = float(dim), float(p), 1.0 + 2.0 ** -40
    R = D ** (1.0 / P) * up
    se = 2.0 ** e
    amax = q.max(axis=-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        qn = np.where(amax > 0, amax * (((q / np.where(amax > 0, amax, 1.0)[..., None]) ** P).sum(axis=-1)) ** (1 / P)
                      * up, 0.0)
    w = (R * float(mnorm) + qn + R * 2.0 ** -148) * (1.0 + 2.0 * U)
    gn = (D + P - 1.0) * U
    g = gn / (1.0 - gn)
    rel = 3.0 * U + g / (P * (1.0 - g)) + 2.0 ** -44 + (D + 2.0 * P + 810.0) * 2.0 ** -53
    eps = rel * w * (1.0 + 2.0 ** -20) + (D * 2.0 ** -1073) ** (1.0 / P) * up + 2.0 ** -149
    if subnormal_rounding:
        eps = eps + R * 2.0 ** -149
    if underflow:
        eps = eps + R * 2.0 ** -149 * se + (D * (P * P + 1.0) * 2.0 ** -149) ** (1.0 / P) * up * se
    return eps
