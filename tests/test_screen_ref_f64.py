"""Pins the F64 screen-copy reference (tests/screen_ref_f64.py) to hand-computed cases, so that the GPU tests that hold
the kernels against it compare with the right thing: ties to even, values that are not f32, subnormals, overflow."""
import numpy as np
import pytest

import screen_ref_f64 as R


@pytest.mark.parametrize("x,want", [
    (1.0, 0x3F80),
    (-2.0, 0xC000),
    (0.0, 0x0000),
    (-0.0, 0x8000),
    (1.0 + 2.0**-8, 0x3F80),                 # tie between 0x3F80 and 0x3F81: even
    (1.0 + 3 * 2.0**-8, 0x3F82),             # tie between 0x3F81 and 0x3F82: even
    (1.0 + 2.0**-8 + 2.0**-40, 0x3F81),      # above the tie by less than an f32 ulp: via f32 it would go to 0x3F80
    (1.0 + 2.0**-8 - 2.0**-40, 0x3F80),      # below the tie by less than an f32 ulp
    (-(1.0 + 2.0**-8 + 2.0**-40), 0xBF81),
    (0.1, 0x3DCD),                           # 0x3DCCCCCD as f32; not an f32 itself
    (1e-200, 0x0000),                        # below half the smallest bf16 subnormal
    (5e-324, 0x0000),                        # smallest f64 subnormal
    (-5e-324, 0x8000),
    (2.0**-133, 0x0001),                     # smallest bf16 subnormal
    (2.0**-134, 0x0000),                     # tie between 0 and it: even
    (2.0**-134 + 2.0**-170, 0x0001),         # just above that tie (the excess is not an f32)
    (3 * 2.0**-134, 0x0002),                 # tie between 0x0001 and 0x0002: even
    (2.0**-126, 0x0080),                     # smallest normal
    (3.3895313892515355e38, 0x7F7F),         # largest finite bf16
    ((2 - 2.0**-8) * 2.0**127, 0x7F80),      # tie between the largest bf16 and 2^128: even = inf
    ((2 - 2.0**-8) * 2.0**127 - 2.0**80, 0x7F7F),
    (3.4028234663852886e38, 0x7F80),         # FLT_MAX rounds up to inf in bf16
    (1e39, 0x7F80),                          # beyond f32
    (-1e300, 0xFF80),
    (np.inf, 0x7F80),
    (-np.inf, 0xFF80),
])
def test_bf16_rne_f64_cases(x, want):
    assert int(R.bf16_rne_f64(np.array([x]))[0]) == want, hex(int(R.bf16_rne_f64(np.array([x]))[0]))


def test_bf16_rne_f64_nan():
    b = R.bf16_rne_f64(np.array([np.nan, -np.nan]))
    assert np.isnan(R.bf16_to_f64(b)).all()


def test_bf16_rne_f64_is_nearest_on_random_values():
    # against a brute-force nearest search over the neighbouring bf16 values (exact in f64)
    rng = np.random.default_rng(7)
    x = rng.uniform(-1, 1, 20000) * np.exp2(rng.integers(-140, 127, 20000).astype(np.float64))
    b = R.bf16_rne_f64(x)
    for d in (-1, 1):
        nb = (b.astype(np.int32) + d).astype(np.uint16)
        ok = np.isfinite(R.bf16_to_f64(nb)) & ((nb & 0x7FFF) != 0x7F80)
        err, err_n = np.abs(x - R.bf16_to_f64(b)), np.abs(x - R.bf16_to_f64(nb))
        assert (err[ok] <= err_n[ok]).all()
        tie = ok & (err == err_n)
        assert ((b[tie] & 1) == 0).all()


def test_normalise_f64_is_correctly_rounded():
    x = np.array([[3.0, 4.0], [0.1, 0.2]])
    mag = np.array([5.0, np.sqrt(0.1 * 0.1 + 0.2 * 0.2)])
    xn = R.normalise_f64(x, mag)
    assert xn[0, 0] == 0.6 and xn[0, 1] == 0.8
    assert xn[1, 0] == 0.1 / mag[1] and xn[1, 0] != np.float32(0.1) / np.float32(mag[1])


def test_quantize_rows_f64_cases():
    # |x| = 4: x / |x| = 0.75 and 0.25; at s = 0.5 the quotients are the ties 1.5 -> 2 and 0.5 -> 0
    x = np.array([[3.0, 1, 1, 1, 1, 1, 1, 1]])
    assert R.quantize_rows_f64(x, [4.0], 0.5).tolist() == [[2, 0, 0, 0, 0, 0, 0, 0]]
    assert R.quantize_rows_f64(-x, [4.0], 0.5).tolist() == [[-2, 0, 0, 0, 0, 0, 0, 0]]
    # clamped at +-127
    assert R.quantize_rows_f64(x, [4.0], 2.0**-10).tolist() == [[127] * 8]
    # values that are not f32: 0.1 / |(0.1, 0.2)| in f64, divided by the f32 scale taken exactly
    y = np.array([[0.1, 0.2]])
    m = np.sqrt(0.01 + 0.04)
    s = np.float32(1.0 / 127.0)
    want = np.clip(np.rint(np.array([0.1 / m, 0.2 / m]) / np.float64(s)), -127, 127)
    assert R.quantize_rows_f64(y, [m], s)[0].tolist() == want.tolist() == [57, 114]
    # an f64-subnormal row normalises to 1
    assert R.quantize_rows_f64(np.array([[5e-324]]), [5e-324], s).tolist() == [[127]]


def test_rmax_f64_rounds_up():
    x = np.array([[0.1, 0.2], [3.0, 4.0]])
    mag = np.array([np.sqrt(0.05), 5.0])
    r = R.rmax_f64(x, mag)
    v = np.array([0.2 / mag[0], 0.8])
    assert (r.astype(np.float64) >= v).all()
    assert (np.nextafter(r, np.float32(0)).astype(np.float64) < v).all()


def test_residuals():
    x = np.array([[1.0 + 2.0**-8 + 2.0**-40, 0.0]])
    b = R.bf16_rne_f64(x)
    assert R.bf16_residual_f64(x, b, [x[0, 0]])[0] == pytest.approx((2.0**-8 - 2.0**-40) / x[0, 0], rel=1e-15)
    x8 = R.quantize_rows_f64(np.array([[3.0, 1, 1, 1, 1, 1, 1, 1]]), [4.0], 0.5)
    # 0.75 - 1.0 and 7 x 0.25 left over
    assert R.i8_residual_f64(np.array([[3.0, 1, 1, 1, 1, 1, 1, 1]]), x8, [4.0], 0.5)[0] == np.sqrt(0.0625 * 8)
