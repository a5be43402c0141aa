"""Test reference for the brute-force screens (csrc/corpus.cu, candidates.cu, screen_tc.cu, screen_simt.cu): the
operand copies the kernels score with, the exact quantities they approximate, and the bounds the exactness proof of
cand_final_kernel relies on.

  magnitude(X)                      sqrt(sum x^2), sequential f64 (the reference's `magnitude()`, finalize_rows_kernel)
  bf16_rne(x) / bf16_to_f32(b)      __float2bfloat16_rn and back (bit patterns as uint16)
  quantize_rows(X, mag, scale)      quantize_rows_kernel: clamp(rint(f32(x * f32(1/|x|)) * f32(1/s)), +-127)
  quantize_queries(Q32)             prep_queries_i8_kernel: per-query scale max|q|/127, same rounding
  cosine_sim(Q, X), euclid_score(Q, X)
                                    the exact f64 similarity and the euclidean screen score 2 q.x - |x|^2
  screen_eps_rel, screen_beps       cand_begin_kernel's error bound of each screen
  proof_bound_cosine / _euclid      the distance bound cand_final_kernel derives from a threshold (tau, beps)

All f32 steps are IEEE operations as written in the kernels (the Makefile does not use fast math, so division is
correctly rounded and nothing but the explicit fmaf calls is fused where it would change a quantised value);
__float2int_rn is round-half-to-even, i.e. np.rint.
"""
import numpy as np

F32 = np.float32


def magnitude(X):
    X = np.asarray(X, np.float64)
    s = np.zeros(X.shape[0], np.float64)
    for c in range(X.shape[1]):  # strictly left to right, as the reference folds
        s = s + X[:, c] * X[:, c]
    return np.sqrt(s)


def bf16_rne(x):
    """__float2bfloat16_rn of f32 values, as uint16 bit patterns (NaN stays a quiet NaN)."""
    u = np.asarray(x, F32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, F32))
    return np.where(nan, ((u >> 16) | 0x40).astype(np.uint16), r)


def bf16_to_f32(b):
    return (np.asarray(b, np.uint16).astype(np.uint32) << 16).view(F32)


def quantize_rows(X, mag, scale):
    """int8 copy of the normalised rows with the corpus' global scale s (rows must be valid: finite, non-zero)."""
    X = np.asarray(X, F32)
    inv_norm = (F32(1.0) / np.asarray(mag, np.float64).astype(F32)).astype(F32)
    xn = (X * inv_norm[:, None]).astype(F32)
    inv = F32(1.0) / F32(scale)
    return np.clip(np.rint((xn * inv).astype(F32)), -127, 127).astype(np.int8)


def quantize_queries(Q32):
    """int8 copies and scales of f32 queries (a query whose max |q| is 0 or not finite gets scale 1 and zeros)."""
    Q32 = np.asarray(Q32, F32)
    mx = np.abs(Q32).max(axis=1).astype(F32)
    ok = (mx > 0) & np.isfinite(mx)
    s = np.where(ok, (mx / F32(127.0)).astype(F32), F32(1.0)).astype(F32)
    inv = (F32(1.0) / s).astype(F32)
    with np.errstate(invalid="ignore"):
        q8 = np.clip(np.rint((Q32 * inv[:, None]).astype(F32)), -127, 127)
    q8 = np.where(ok[:, None], q8, 0).astype(np.int8)
    return q8, s


def cosine_sim(Q, X):
    Q = np.asarray(Q, np.float64)
    X = np.asarray(X, np.float64)
    return (Q @ X.T) / np.linalg.norm(Q, axis=1)[:, None] / np.linalg.norm(X, axis=1)[None, :]


def euclid_score(Q, X):
    """2 q.x - |x|^2: larger = closer; |q - x|^2 = |q|^2 - score."""
    Q = np.asarray(Q, np.float64)
    X = np.asarray(X, np.float64)
    return 2.0 * (Q @ X.T) - (X * X).sum(axis=1)[None, :]


def screen_eps_rel(screen, dim, eq, ex):
    """cand_begin_kernel's relative error bound of a screen.  eq / ex: the query's and the corpus' measured residual
    (int8: q8err, max_rel_qerr; bf16: qbferr, bf16_rel_err; unused for SIMT_F32)."""
    eq, ex = np.asarray(eq, np.float64), np.float64(ex)
    if screen == "TC_INT8":
        return (1.0 + eq) * ex + eq + 2e-6
    if screen == "TC_BF16":
        return ex + eq + ex * eq + dim * 2.0**-21 + 1e-5  # D * 2^-21: the fp32 accumulation of the tensor cores
    return np.full(eq.shape, (dim / 16.0 + 16.0) * 2.0**-23)


def screen_beps(metric, eps_rel, qmag, max_norm):
    """beps: |screened similarity - similarity| (cosine) or |screened score - score| (euclidean) is at most this."""
    if metric == "COSINE":
        return eps_rel
    mn = np.float64(max_norm)
    return 2.0 * eps_rel * qmag * mn + 4.8e-7 * (mn * mn + 2.0 * qmag * mn) + 1e-30


def proof_bound_cosine(tau, bscale, qmag, beps):
    """A row whose screen score is <= tau has cosine distance >= this (cand_final_kernel)."""
    return 1.0 - np.float64(tau) * np.float64(bscale) / qmag - np.float64(beps) - 1e-9


def proof_bound_euclid(tau, qmag, beps):
    """A row whose screen score is <= tau has euclidean distance >= this; NaN where the proof has no bound (L <= 0)."""
    L = -np.float64(tau) + qmag * qmag - np.float64(beps)
    with np.errstate(invalid="ignore"):
        return np.where(L > 0.0, np.sqrt(np.maximum(L, 0.0)) * (1.0 - 1e-12), np.nan)
