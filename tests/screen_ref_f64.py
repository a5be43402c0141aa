"""Test reference for the screen copies of F64 corpora (csrc/corpus.cu, the double instantiations of to_bf16_kernel,
quantize_scan_kernel and quantize_rows_kernel), next to tests/screen_ref.py for F32 ones.

  bf16_rne_f64(x)                      cvt.rn.bf16.f64: each f64 rounded to nearest-even bf16 in ONE step (as uint16)
  normalise_f64(X, mag)                x / |x| in f64, correctly rounded per element
  quantize_rows_f64(X, mag, scale)     clamp(rint((x / |x|) / f64(scale)), +-127) with f64 divisions
  rmax_f64(X, mag)                     max_i |x_i| / |x| in f64, rounded up to f32 (the outlier rule's figure)
  bf16_residual_f64 / i8_residual_f64  the residual norms the finalize measures, in f64

Rounding f64 -> f32 -> bf16 would round twice (1 + 2^-8 + 2^-40 would land on the tie 1 + 2^-8 and go to even); the
helper instead truncates to f32 and sets the sticky bit (round to odd), after which one round-to-nearest-even to bf16
is exact: f32 keeps 16 bits more than bf16, in the subnormal range too.
"""
import numpy as np

F32 = np.float32


def bf16_rne_f64(x):
    """uint16 bit patterns of the nearest-even bf16 of f64 values (overflow to +-inf, NaN stays a quiet NaN)."""
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = x.astype(F32)
        # round toward zero: step back where nearest rounding went away from zero (including overflow to inf)
        away = np.abs(f.astype(np.float64)) > np.abs(x)
        f = np.where(away, np.nextafter(f, F32(0)), f).astype(F32)
        u = f.view(np.uint32).copy()
        inexact = (f.astype(np.float64) != x) & ~np.isnan(x)
    u = np.where(inexact, u | np.uint32(1), u).astype(np.uint32)
    w = u.astype(np.uint64)
    r = ((w + 0x7FFF + ((w >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), ((w >> 16) | 0x40).astype(np.uint16), r)


def bf16_to_f64(b):
    return (np.asarray(b, np.uint16).astype(np.uint32) << 16).view(F32).astype(np.float64)


def normalise_f64(X, mag):
    return np.asarray(X, np.float64) / np.asarray(mag, np.float64)[:, None]


def quantize_rows_f64(X, mag, scale):
    """int8 copy of f64 rows with the corpus' global scale (an f32 value) -- valid rows only."""
    with np.errstate(invalid="ignore", divide="ignore"):
        t = normalise_f64(X, mag) / np.float64(F32(scale))
    return np.clip(np.rint(t), -127, 127).astype(np.int8)


def rmax_f64(X, mag):
    """max_i |x_i| / |x| per row in f64, rounded up to f32 (__double2float_ru)."""
    v = np.abs(np.asarray(X, np.float64)).max(axis=1) / np.asarray(mag, np.float64)
    f = v.astype(F32)
    return np.where(f.astype(np.float64) < v, np.nextafter(f, F32(np.inf)), f).astype(F32)


def bf16_residual_f64(X, xbf, mag):
    """|x - bf16(x)| / |x| per row, in f64."""
    return np.linalg.norm(np.asarray(X, np.float64) - bf16_to_f64(xbf), axis=1) / np.asarray(mag, np.float64)


def i8_residual_f64(X, x8, mag, scale):
    """|x/|x| - s x8| per row, in f64."""
    return np.linalg.norm(normalise_f64(X, mag) - np.float64(F32(scale)) * np.asarray(x8, np.float64), axis=1)
