"""The CPU model of the fp8 block-linear quantisation (tests/_fp8_ref.py) against hand-computed bytes and scales.

e4m3 (bias 7, 3 mantissa bits): 448 = 0x7E, 2^-3 = 0x20, 224 = 0x76, 128 = 0x70, 64 = 0x68, 16 = 0x58, 20 = 0x5A;
subnormals are m * 2^-9 with byte m; 0x80 is -0 and 0x7F is NaN.
"""

import math

import pytest
import torch

from _fp8_ref import exponent, quantize_cols_t, quantize_rows

BF16 = torch.bfloat16


def _q(*rows):
    return quantize_rows(torch.tensor(rows, dtype=torch.float32).to(BF16))


def _bytes(q, row=0):
    return q[row].tolist()


@pytest.mark.parametrize("k", [-20, 0, 3, 40])
def test_amax_exactly_448_times_a_power_of_two_gets_that_power(k):
    amax = 448.0 * 2.0 ** k
    q, s = _q([amax, -amax, 2.0 ** (k - 3)])
    assert s.tolist() == [2.0 ** k]
    assert _bytes(q) == [0x7E, 0xFE, 0x20]  # 448, -448 and 2^-3 after the scaling


def test_one_bf16_ulp_above_448_moves_to_the_next_exponent():
    # bf16 spacing at 3584 = 448 * 8 is 16: 3600 needs e = 4, and 3600 / 16 = 225 rounds to 224
    q, s = _q([3600.0, 1.0])
    assert s.tolist() == [16.0]
    assert _bytes(q) == [0x76, 0x18]  # 224; 1/16 = 2^-4 -> exponent field 3


def test_one_bf16_ulp_below_448_keeps_the_exponent_and_rounds_up_to_448():
    # 3568 / 8 = 446 lies between 416 and 448 (spacing 32): nearest is 448, reached by rounding, not by saturation
    q, s = _q([3568.0])
    assert s.tolist() == [8.0]
    assert _bytes(q) == [0x7E]


def test_exponent_from_the_bit_pattern():
    a = torch.tensor([448.0, 448.0 * 1.0000001, 447.99997, 1.0, 0.0, 3.0e38, 2.0 ** -126])
    # 1.0 / 448 = 2^-8.8: e = -8; 0 and the smallest normal clamp to -126; 3e38 = 1.76 * 2^127 -> 120
    assert exponent(a).tolist() == [0, 1, 0, -8, -126, 120, -126]
    for x in (1e-30, 1e-3, 0.7, 5.0, 1e4, 1e30):
        xb = float(torch.tensor(x).to(BF16).float())
        assert int(exponent(torch.tensor([xb]))[0]) == max(-126, math.ceil(math.log2(xb / 448))), x


def test_zero_row():
    q, s = _q([0.0] * 16)
    assert s.tolist() == [2.0 ** -126]
    assert _bytes(q) == [0] * 16


def test_bf16_subnormals_are_flushed_to_signed_zeros():
    tiny = 2.0 ** -130  # a bf16 subnormal
    q, s = _q([tiny, -tiny, 2.0 ** -133, 0.0])
    assert s.tolist() == [2.0 ** -126]
    assert _bytes(q) == [0x00, 0x80, 0x00, 0x00]


def test_the_exponent_clamps_at_minus_126():
    # amax 2^-120: ceil(log2(2^-120 / 448)) = -128 -> -126, so the row maps to 2^6 = 64, not 448
    q, s = _q([2.0 ** -120, 2.0 ** -122])
    assert s.tolist() == [2.0 ** -126]
    assert _bytes(q) == [0x68, 0x58]  # 64, 16


def test_ties_round_to_even():
    # with 448 in the row e = 0; between 16 and 32 the spacing is 2: 17 -> 16 (even mantissa), 19 -> 20
    q, s = _q([448.0, 17.0, 19.0, -17.0])
    assert s.tolist() == [1.0]
    assert _bytes(q) == [0x7E, 0x58, 0x5A, 0xD8]


def test_e4m3_subnormal_outputs():
    # e = 0; subnormals are m * 2^-9: 2^-8 -> m = 2; 1.5 * 2^-9 ties to 2; 2^-10 ties to 0; 2.5 * 2^-9 ties to 2
    q, s = _q([448.0, 2.0 ** -8, 1.5 * 2.0 ** -9, 2.0 ** -10, 2.5 * 2.0 ** -9, 7 * 2.0 ** -9, -(2.0 ** -9)])
    assert s.tolist() == [1.0]
    assert _bytes(q) == [0x7E, 0x02, 0x02, 0x00, 0x02, 0x07, 0x81]


@pytest.mark.parametrize("bad", [math.inf, -math.inf, math.nan])
def test_a_nonfinite_element_makes_the_whole_row_nan(bad):
    q, s = _q([1.0, bad, 3.0, 0.0], [1.0, 2.0, 3.0, 0.0])
    assert math.isnan(s[0]) and s[1] == 2.0 ** -7  # 3 / 448 = 2^-7.2 -> e = -7
    assert _bytes(q) == [0x7F] * 4
    assert _bytes(q, 1) == [0x70, 0x78, 0x7C, 0x00]  # 128, 256, 384, 0


def test_negative_zero():
    q, s = _q([-0.0, 0.0, -0.0])
    assert s.tolist() == [2.0 ** -126]
    assert _bytes(q) == [0x80, 0x00, 0x80]


def test_columns_of_w_are_rows_of_w_transposed():
    w = torch.tensor([[448.0, 1.0], [0.5, 2.0], [-224.0, 0.0]]).to(BF16)  # N = 3, K = 2
    q, s = quantize_cols_t(w)
    assert q.shape == (2, 3) and s.tolist() == [1.0, 2.0 ** -7]
    assert _bytes(q) == [0x7E, 0x30, 0xF6]  # 448, 0.5, -224
    assert _bytes(q, 1) == [0x70, 0x78, 0x00]  # 1 * 128, 2 * 128, 0
