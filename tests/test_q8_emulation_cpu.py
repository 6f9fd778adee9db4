"""The CPU emulation of the Q8G fp8 format (``_q8_emulation``) that the GPU tests compare the kernels against, checked on
its own: the e4m3 code table, round-to-nearest-even with saturation as ``cvt.rn.satfinite`` does it, the group rules
(amax floor, non-finite groups), the layout, and that every deliberate deviation from the kernels' arithmetic changes
bytes on the test data (so a kernel that made one of them could not pass the exact GPU tests)."""

from __future__ import annotations

import math

import pytest
import torch

import _q8_emulation as E


def _e4m3_value(code: int) -> float:
    """e4m3fn by its definition: 1 sign, 4 exponent (bias 7), 3 mantissa bits, no inf, S.1111.111 is NaN."""
    sign = -1.0 if code & 0x80 else 1.0
    exp, man = (code >> 3) & 0xF, code & 0x7
    if exp == 0xF and man == 0x7:
        return math.nan
    if exp == 0:
        return sign * man / 8 * 2.0 ** -6
    return sign * (1 + man / 8) * 2.0 ** (exp - 7)


def test_all_256_codes_decode_to_the_e4m3_table():
    got = E.e4m3_decode(torch.arange(256, dtype=torch.uint8))
    for c in range(256):
        want = _e4m3_value(c)
        if math.isnan(want):
            assert math.isnan(got[c].item()), c
        else:
            assert got[c].item() == want and math.copysign(1, got[c].item()) == math.copysign(1, want), c
    assert E.e4m3_decode(torch.tensor([0x7E], dtype=torch.uint8)).item() == 448.0


def test_rounding_is_nearest_even_and_saturates_like_cvt_satfinite():
    finite = sorted({_e4m3_value(c) for c in range(0x7F)})  # every non-negative finite value
    lo, hi = torch.tensor(finite[:-1]), torch.tensor(finite[1:])
    mid = (lo + hi) / 2  # exact in fp32: neighbours differ in the last of 4 significant bits
    even = torch.tensor([c for c in range(0x7E)], dtype=torch.uint8)  # code of lo; lo -> lo+1 is the next code
    lo_codes, hi_codes = even, even + 1
    tie = torch.where(lo_codes % 2 == 0, lo_codes, hi_codes)
    for sign in (1.0, -1.0):
        sb = 0x80 if sign < 0 else 0
        assert torch.equal(E.e4m3_codes(sign * mid), tie | sb)
        assert torch.equal(E.e4m3_codes(sign * torch.nextafter(mid, torch.tensor(0.0))), lo_codes | sb)
        assert torch.equal(E.e4m3_codes(sign * torch.nextafter(mid, torch.tensor(1e9))), hi_codes | sb)
        assert torch.equal(E.e4m3_codes(sign * lo), lo_codes | sb)
    big = torch.tensor([448.0, 449.0, 464.0, 480.0, 1e30, 3.4e38, math.inf])
    assert E.e4m3_codes(big).tolist() == [0x7E] * 7
    assert E.e4m3_codes(-big).tolist() == [0xFE] * 7
    assert (E.e4m3_codes(torch.tensor([math.nan])) & 0x7F).item() == 0x7F
    assert E.e4m3_codes(torch.tensor([2.0 ** -10, -(2.0 ** -10), 2.0 ** -11, 3 * 2.0 ** -10])).tolist() == [0, 0x80, 0, 2]


def test_ftz_keeps_the_sign_and_normal_values():
    x = torch.tensor([2.0 ** -127, -(2.0 ** -149), 2.0 ** -126, -(2.0 ** -126), 0.0, 1.0, math.inf, math.nan])
    y = E.ftz(x)
    assert y[:2].tolist() == [0.0, 0.0] and math.copysign(1, y[1].item()) == -1.0
    assert E.equal_bits(y[2:], x[2:])


def test_layout():
    assert [E.ngroups(n, w) for n, w in ((1, 1), (512, 1), (513, 1), (513, 3), (0, 2), (512 * 8 + 1, 8))] == \
        [1, 1, 2, 3, 0, 16]
    assert E.payload_off(1) == 16 and E.payload_off(4) == 16 and E.payload_off(5) == 32
    assert E.buffer_bytes(513, 3) == 16 + 3 * 512
    q = E.quantize(torch.randn(1000), E.ngroups(1000, 3))
    b = q.to_bytes()
    assert b.numel() == E.buffer_bytes(1000, 3) and b[12:16].tolist() == [0] * 4
    assert E.equal_q8(E.Q8.from_bytes(b, q.ng), q)
    assert E.staging_chunk(1 << 20, 4) % (512 * 4) == 0


def test_group_rules():
    """amax floor: a tiny group keeps normal scale and finite multiplier, zeros stay exactly zero; an inf anywhere makes
    the whole group NaN; NaN alone is ignored by the amax and stays in its element."""
    tiny = 1e-37  # below 448/FLT_MAX: without the floor m would be inf and 0 * m NaN
    rows = torch.zeros(6, E.GROUP)
    rows[1, 3] = tiny
    rows[2, :] = torch.linspace(-3e-36, 3e-36, E.GROUP)
    rows[3, 7] = math.inf
    rows[3, 8] = 5.0
    rows[4, 9] = math.nan
    rows[4, 10] = -2.0
    rows[5, 0] = 3.4e38
    q = E.group_quant(rows)
    assert torch.all(q.scales[:3] >= E.TINY) and torch.all(q.scales[:3] < math.inf)
    d = E.dequant(q)
    assert E.equal_bits(d[0], torch.zeros(E.GROUP))
    assert d[1, 3].item() != 0 and abs(d[1, 3].item() / tiny - 1) <= 1 / 16
    assert (d[2] != 0).sum() > E.GROUP // 2 and not torch.isnan(d[2]).any()
    assert math.isnan(q.scales[3].item()) and torch.isnan(d[3]).all()
    assert torch.isnan(d[4, 9]) and d[4, 10].item() == -2.0 and (~torch.isnan(d[4])).sum() == E.GROUP - 1
    assert d[5, 0].item() > 3.3e38 and torch.isfinite(d[5]).all()


def test_reduction_keeps_nan_through_the_requantisation():
    """The sum of a NaN group is NaN; requantising it (fmaxf ignores NaN, so the amax is the floor) keeps NaN codes."""
    a = torch.ones(2, E.GROUP)
    b = torch.ones(2, E.GROUP)
    b[1, 5] = math.inf
    qa, qb = E.group_quant(a), E.group_quant(b)
    acc = E.reduce([qa, qb], torch.tensor([0, 1]), 0.5)
    assert torch.equal(acc[0], torch.ones(E.GROUP)) and torch.isnan(acc[1]).all()
    red = E.group_quant(acc)
    assert torch.isnan(E.dequant(red)[1]).all() and not torch.isnan(E.dequant(red)[0]).any()


VARIANTS = {
    "order_from_zero": E.Variant(order_from_zero=True),
    "m_from_s": E.Variant(m_from_s=True),
    "fma": E.Variant(fma=True),
    "post_before_sum": E.Variant(post_before_sum=True),
    "no_ftz": E.Variant(no_ftz=True),
}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_every_variant_changes_bytes_on_the_test_data(name):
    """At W = 3 on ``E.message``, the data of the exact GPU tests: the result bits and the reduced message of the fused
    all-reduce both differ from the exact emulation for every variant."""
    v, W, n = VARIANTS[name], 3, 512 * 3 * 8 + 40
    a, b = E.message(n, W, 1), E.message(n, W, 2)
    xs = [E.pseudo_grad(x, y) for x, y in zip(a, b)]
    want, want_red = E.allreduce(xs, 1.0 / W)
    got, got_red = E.allreduce([E.pseudo_grad(x, y, v) for x, y in zip(a, b)], 1.0 / W, v=v)
    assert not E.equal_bits(got, want)
    assert not E.equal_q8(got_red, want_red)


def test_emulated_allreduce_is_close_to_the_exact_sum():
    """Sanity of the emulation itself: within the reference's 0.04 mean relative error of the fp64 sum."""
    W, n = 3, 100_003
    g = torch.Generator().manual_seed(0)
    xs = [torch.randn(n, generator=g) for _ in range(W)]
    got, _ = E.allreduce(xs, 1.0 / W, per=E.GROUP * W * 16)
    ref = sum(x.double() for x in xs) / W
    assert ((got.double() - ref).abs().mean() / ref.abs().mean()).item() <= 0.04
