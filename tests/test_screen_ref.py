"""Pins the numpy restatement of the screens' rounding (tests/screen_ref.py) on hand-picked values, so that the GPU
invariant tests compare the kernels with the intended arithmetic and not with a second copy of a mistake."""
import numpy as np

import screen_ref as R


def bits(x):
    return int(np.float32(x).view(np.uint32))


def test_bf16_round_to_nearest_even_at_midpoints():
    one = bits(1.0)  # 0x3F800000
    cases = [
        (one, 0x3F80),                # exact
        (one + 0x7FFF, 0x3F80),       # just below the midpoint: down
        (one + 0x8000, 0x3F80),       # midpoint, even low bit: stays
        (one + 0x8001, 0x3F81),       # just above: up
        (one + 0x18000, 0x3F82),      # midpoint, odd low bit: up to even
        (0xBF818000, 0xBF82),         # negative midpoint, odd: away from zero to even
        (0x7F7FFFFF, 0x7F80),         # largest f32 rounds to inf
        (0x00008000, 0x0000),         # subnormal midpoint to even zero
    ]
    for u, want in cases:
        x = np.array([u], np.uint32).view(np.float32)
        assert int(R.bf16_rne(x)[0]) == want, hex(u)
    assert np.isnan(R.bf16_to_f32(R.bf16_rne(np.array([np.nan], np.float32))))[0]
    x = np.array([1.5, -3.25, 0.0], np.float32)
    assert np.array_equal(R.bf16_to_f32(R.bf16_rne(x)), x)


def test_int8_query_quantisation_ties_to_even_and_clamp():
    # scale = 127 / 127 = 1: q / s is the value itself, so the rounding is visible directly
    q = np.array([[127.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.49]], np.float32)
    q8, s = R.quantize_queries(q)
    assert s[0] == np.float32(1.0)
    assert list(q8[0]) == [127, 0, 2, 2, 0, -2, -2, 126]
    q8, s = R.quantize_queries(np.zeros((1, 4), np.float32))  # zero query: scale 1, all zero
    assert s[0] == 1.0 and not q8.any()


def test_int8_row_quantisation_clamps_at_127():
    # a scale smaller than the largest normalised component (the gap rule sets outliers aside and then quantises the
    # rest with a smaller scale) saturates at +-127 instead of wrapping
    x = np.array([[3.0, -4.0, 0.0]], np.float32)
    mag = R.magnitude(x)
    assert mag[0] == 5.0
    q8 = R.quantize_rows(x, mag, np.float32(0.8 / 127))
    assert list(q8[0]) == [95, -127, 0]  # 0.6 / (0.8/127) = 95.25; -0.8 / s rounds to -127 exactly, beyond clamps
    q8 = R.quantize_rows(x, mag, np.float32(0.5 / 127))
    assert list(q8[0]) == [127, -127, 0]


def test_magnitude_is_a_sequential_f64_fold():
    # left to right every 2^-54 is lost against 1.0 (ties to even); summed small-first they would make 1 + 2^-52
    y = np.array([[1.0] + [2.0**-27] * 4])
    assert R.magnitude(y)[0] == 1.0
    assert R.magnitude(y[:, ::-1])[0] == np.sqrt(1.0 + 2.0**-52)


def test_proof_bounds():
    assert R.proof_bound_cosine(0.5, 2.0, 4.0, 0.01) == 1.0 - 0.25 - 0.01 - 1e-9
    assert np.isnan(R.proof_bound_euclid(10.0, 1.0, 0.0))  # L = -9: no bound
    assert R.proof_bound_euclid(-3.0, 1.0, 0.0) == 2.0 * (1.0 - 1e-12)
