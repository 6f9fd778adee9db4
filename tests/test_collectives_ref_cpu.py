"""The numpy model of the data-plane reductions (``_collectives_ref``) on hand-computed cases: the GPU tests compare
the kernels against it bit for bit, so it has to be right about flushing, rounding, overflow and NaN."""

from __future__ import annotations

import numpy as np

import _collectives_ref as R


def f32(*xs):
    return np.array(xs, dtype=np.float32).view(np.uint32)


def bf16(*xs):
    return R.round_to(np.array(xs, dtype=np.float32), "bf16")


def f16(*xs):
    return np.array(xs, dtype=np.float16).view(np.uint16)


def test_fp32_subnormal_operands_and_sums_flush_to_signed_zero():
    sub = 2.0 ** -130
    assert R.allreduce([f32(sub), f32(sub)], "f32", R.SUM, 1.0).tolist() == [0]
    # two normals whose difference is subnormal: the sum flushes, keeping its sign
    m = 2.0 ** -126
    assert R.allreduce([f32(-1.5 * m), f32(m)], "f32", R.SUM, 1.0).tolist() == [0x80000000]
    # a normal result scaled into the subnormal range flushes too
    assert R.allreduce([f32(m), f32(m)], "f32", R.SUM, 0.25).tolist() == [0]
    # a subnormal operand is zero to MAX as well
    assert R.allreduce([f32(-sub), f32(-1.0)], "f32", R.MAX, 1.0).tolist() == [0x80000000]


def test_bf16_subnormals_vanish_and_fp16_subnormals_stay():
    assert R.allreduce([np.array([0x0001], np.uint16), np.array([0x0001], np.uint16)], "bf16", R.SUM, 1.0).tolist() == [0]
    tiny = np.array([0x0001], np.uint16)  # 2^-24, the smallest fp16 subnormal: normal in fp32
    assert R.allreduce([tiny, tiny, tiny], "f16", R.SUM, 1.0).tolist() == [0x0003]


def test_bf16_ties_round_to_even():
    # 1 + 2^-8 lies halfway between 1 and 1 + 2^-7: even is 1; 1 + 3*2^-8 is halfway between 1 + 2^-7 and 1 + 2^-6
    assert R.allreduce([bf16(1.0), bf16(2.0 ** -8)], "bf16", R.SUM, 1.0).tolist() == [0x3F80]
    assert R.allreduce([bf16(1.0), bf16(3 * 2.0 ** -8)], "bf16", R.SUM, 1.0).tolist() == [0x3F82]
    # one rounding only: the sum is exact in fp32 and rounds once, after the scale
    assert R.allreduce([bf16(1.0), bf16(2.0 ** -8), bf16(2.0 ** -8)], "bf16", R.SUM, 1.0).tolist() == [0x3F81]


def test_fp16_overflow_is_inf_and_the_range_limit_rounds_to_nearest():
    assert R.allreduce([f16(60000.0)] * 3, "f16", R.SUM, 1.0).tolist() == [0x7C00]
    assert R.allreduce([f16(-60000.0)] * 3, "f16", R.SUM, 1.0).tolist() == [0xFC00]
    assert R.allreduce([f16(60000.0)] * 3, "f16", R.SUM, 1.0 / 3).view(np.float16).tolist() == [60000.0]
    assert R.allreduce([f16(65504.0), f16(8.0)], "f16", R.SUM, 1.0).tolist() == [0x7BFF]
    assert R.allreduce([f16(65504.0), f16(16.0)], "f16", R.SUM, 1.0).tolist() == [0x7C00]


def test_nan_propagates_under_sum_and_loses_under_max_and_min():
    nan = float("nan")
    got = R.allreduce([f32(nan), f32(1.0)], "f32", R.SUM, 1.0)
    assert np.isnan(got.view(np.float32)).all()
    assert np.isnan(R.allreduce([f32(np.inf), f32(-np.inf)], "f32", R.SUM, 1.0).view(np.float32)).all()
    assert R.allreduce([f32(nan), f32(1.0)], "f32", R.MAX, 1.0).view(np.float32).tolist() == [1.0]
    assert R.allreduce([f32(2.0), f32(nan)], "f32", R.MIN, 1.0).view(np.float32).tolist() == [2.0]
    assert np.isnan(R.allreduce([f32(nan), f32(nan)], "f32", R.MAX, 1.0).view(np.float32)).all()


def test_quiet_rank_adds_positive_zero_in_its_place():
    assert R.allreduce([f32(-0.0), None], "f32", R.SUM, 1.0).tolist() == [0]
    assert R.allreduce([f32(-0.0), f32(-0.0)], "f32", R.SUM, 1.0).tolist() == [0x80000000]
    # MAX over negative values with a quiet rank is 0, MIN over positive ones too
    assert R.allreduce([bf16(-3.0), None, bf16(-1.0)], "bf16", R.MAX, 1.0).tolist() == [0]
    assert R.allreduce([None, f16(2.0)], "f16", R.MIN, 1.0).tolist() == [0]


def test_world_one_scale_copy():
    x = f32(3.0, 2.0 ** -130, -1.0)
    assert R.scale_copy(x, "f32", 0.5, True).view(np.float32).tolist() == [1.5, 0.0, -0.5]
    assert R.scale_copy(x, "f32", 0.5, False).tolist() == [0, 0, 0]


def test_check_accepts_any_nan_and_signed_zeros_only_under_max_min():
    a, b = np.array([0x7FC00000], np.uint32), np.array([0xFFFFFFFF], np.uint32)
    assert R.mismatch(a, b, "f32", R.SUM) is None
    z, nz = f32(0.0), f32(-0.0)
    assert R.mismatch(z, nz, "f32", R.MAX) is None and R.mismatch(z, nz, "f32", R.MIN) is None
    assert R.mismatch(z, nz, "f32", R.SUM) is not None
    assert R.mismatch(bf16(1.0), bf16(1.0078125), "bf16", R.SUM) is not None


def test_values_cover_every_magnitude_class_and_the_specials():
    rng = np.random.default_rng(0)
    for dt in R.DTYPES:
        v = R.values(rng, 10_000, dt)
        assert v.dtype == R.BITS[dt] and len(v) == 10_000
        assert np.isin(R.SPECIALS[dt], v).all()
        f = np.abs(R.to_f32(v, dt))
        assert (f == 0).any() and ((f > 0) & (f < 0.1)).any() and (f[np.isfinite(f)] > 100).any()
