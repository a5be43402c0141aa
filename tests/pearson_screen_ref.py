"""numpy restatement of the PEARSON screen (corpus.cu finalize_pearson_kernel / to_bf16_kernel / quantize_rows_kernel,
candidates.cu prep_queries_pearson_kernel / cand_final_pearson_kernel; DESIGN.md section 2, "PEARSON screen").

The reference's pearson is the cosine of the rows and the query centred in f64 with their own sequential means, up to
f64 rounding: the cosine screens run on dx = x - m1 against -dq, and the proof adds eps_ref for the gap."""
import numpy as np

U = 2.0 ** -53


def seq_sum(a):
    """sequential f64 sum along the last axis (the reference's left-to-right fold)"""
    a = np.asarray(a, np.float64)
    if a.shape[-1] == 0:
        return np.zeros(a.shape[:-1])
    return np.add.accumulate(a, axis=-1)[..., -1]


def moments(X):
    """m1 = (sum x) / D and S1 = sum (x_i - m1)^2 (sequential f64), and dx = x - m1 in f64"""
    X = np.asarray(X, np.float64)
    D = X.shape[-1]
    m1 = seq_sum(X) / D
    dx = X - m1[..., None]
    return m1, seq_sum(dx * dx), dx


def pearson(X, q):
    """the reference's pearson of every row of X against q, op for op (exact_keys_kernel's arithmetic)"""
    X = np.atleast_2d(np.asarray(X, np.float64))
    D = X.shape[1]
    _, s1, dx = moments(X)
    _, s2, dq = moments(np.asarray(q, np.float64)[None, :])
    with np.errstate(all="ignore"):
        covar = seq_sum(dx * dq) / D
        sd1 = np.sqrt(s1 / D) if D > 1 else np.zeros_like(s1)
        sd2 = np.sqrt(s2 / D) if D > 1 else np.zeros_like(s2)
        return covar / (sd1 * sd2)


def eps_ref(D):
    """bound of |pearson - cos(dx, dq)|: (2 D + 6) 2^-53 to first order, +2 units for the rest (cand_final)"""
    return (2.0 * D + 8.0) * U


def is_special(X):
    """rows the screen cannot stand for (finalize_pearson_kernel): ranked exactly on every query"""
    m1, s1, dx = moments(X)
    with np.errstate(all="ignore"):
        nrm = np.sqrt(s1)
        inv32 = (1.0 / nrm).astype(np.float32)
        n32 = nrm.astype(np.float32)
        amax = np.nanmax(np.abs(dx), axis=1) if dx.shape[1] else np.zeros(len(dx))
    tiny = np.float32(1.17549435e-38)
    bad = ~(s1 > 0) | ~np.isfinite(s1) | ~np.isfinite(m1) | ~(amax <= 3.4028234663852886e38) | np.isnan(dx).any(1)
    bad |= ~(nrm >= 2.0 ** -100) | ~((n32 >= tiny) & np.isfinite(n32)) | ~((np.abs(inv32) >= tiny) & np.isfinite(inv32))
    return bad


def bf16_rn(v):
    """f64 -> bf16 in one rounding (round to nearest even), returned as f64 values"""
    v = np.asarray(v, np.float64)
    out = np.zeros_like(v)
    nz = (v != 0) & np.isfinite(v)
    e = np.floor(np.log2(np.abs(v[nz])))
    scale = np.exp2(np.maximum(e - 7.0, -133.0))
    out[nz] = np.round(v[nz] / scale) * scale
    out[~nz] = v[~nz]
    return out


def bf16_residual(X):
    """max over the screened rows of |dx - bf16(dx)| / |dx| (the figure to_bf16_kernel measures)"""
    _, s1, dx = moments(X)
    ok = ~is_special(X)
    r = np.sqrt(((dx[ok] - bf16_rn(dx[ok])) ** 2).sum(1)) / np.sqrt(s1[ok])
    return r.max() if r.size else 0.0


def int8_copy(X, scale):
    """int8 copy of dx / |dx| with the corpus scale (quantize_rows_kernel), and each row's residual norm"""
    _, s1, dx = moments(X)
    xn = dx / np.sqrt(s1)[:, None]
    q = np.clip(np.rint(xn / np.float64(scale)), -127, 127)
    res = np.sqrt(((xn - q * np.float64(scale)) ** 2).sum(1))
    return q.astype(np.int8), res


def proof_bound(tau, bscale, qmag, beps, D):
    """the proof's lower bound of pearson for a row the screen left out (score <= tau), before directed rounding"""
    return -np.float64(tau) * np.float64(bscale) / np.float64(qmag) - np.float64(beps) - eps_ref(D)
