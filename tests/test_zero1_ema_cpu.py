"""FT-ZeRO-1 EMA of the weights, without a GPU: the numpy specification of the update kernel's EMA step and of its
rounding bits, why a bf16 EMA needs stochastic rounding, the agreement check, the checkpoint header and sections, and the
restore's read and seed plan over files with and without an EMA."""

from __future__ import annotations

import numpy as np
import pytest

from _zero1_replicas import widen
from torchft_b200.checkpointing.sharded import file_dtype, payload_bytes, sections
from torchft_b200.parallel.zero1 import (SR_SEED, SR_SEED_EMA, bf16_sr, bf16_sr_ema, check_ema_agreement, ckpt_read_plan,
                                         ema_coefficient, ema_decay_value, ema_record, ema_step, merge_ranges,
                                         split_ema_reads, sr_bits, sr_bits_ema)


# ----------------------------------------------------------------------------- the step
def test_the_coefficient_is_one_minus_decay_rounded_once_to_fp32():
    for d in (0.9, 0.99, 0.999, 0.9999):
        c = ema_coefficient(d)
        assert c == float(np.float32(1.0 - d)) and 0 < c < 1
    # 1 - fp32(d) would keep only the digits fp32(d) has near 1: 2^-24 steps, a relative error of 6e-5 at 0.999
    assert ema_coefficient(0.999) != float(np.float32(1.0) - np.float32(0.999))


def test_ema_step_rounds_each_of_its_three_operations_to_fp32():
    rng = np.random.default_rng(0)
    ema = rng.standard_normal(10000).astype(np.float32)
    w = (ema + rng.standard_normal(10000).astype(np.float32) * np.float32(1e-3)).astype(np.float32)
    c = ema_coefficient(0.999)
    got = ema_step(ema, w, c)
    assert got.dtype == np.float32
    d = (w.astype(np.float64) - ema).astype(np.float32)  # each operation exact in double, then rounded
    p = (np.float64(np.float32(c)) * d).astype(np.float32)
    want = (ema.astype(np.float64) + p).astype(np.float32)
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
    # a fused multiply-add would round once: it differs somewhere, which is why the kernel spells the three out
    fused = (ema.astype(np.float64) + np.float64(np.float32(c)) * d).astype(np.float32)
    assert (fused.view(np.uint32) != want.view(np.uint32)).any()
    # a fixed point: ema == w stays put
    assert (ema_step(w, w, c) == w).all()


def test_ema_decay_value_takes_the_argument_or_the_environment(monkeypatch):
    monkeypatch.delenv("TORCHFT_B200_Z1_EMA_DECAY", raising=False)
    assert ema_decay_value(None) is None
    assert ema_decay_value(0.999) == 0.999
    monkeypatch.setenv("TORCHFT_B200_Z1_EMA_DECAY", "0.9995")
    assert ema_decay_value(None) == 0.9995
    assert ema_decay_value(0.5) == 0.5  # the argument wins
    monkeypatch.setenv("TORCHFT_B200_Z1_EMA_DECAY", " ")
    assert ema_decay_value(None) is None
    for bad in (0.0, 1.0, -0.1, 1.5, float("nan"), float("inf"), 1e-9):  # fp32(1 - 1e-9) is 1: the EMA would copy w
        with pytest.raises(ValueError, match="ema_decay"):
            ema_decay_value(bad)


# ----------------------------------------------------------------------------- the rounding bits
def test_the_ema_bits_are_the_moment_hash_with_its_own_seed():
    e = np.arange(0, 1 << 16, dtype=np.uint64) * np.uint64(977) + np.uint64(1 << 33)
    for t in (1, 2, 1000):
        assert (sr_bits_ema(e, t) == sr_bits(e, t, SR_SEED_EMA)).all()
        assert (sr_bits(e, t) == sr_bits(e, t, SR_SEED)).all()
    assert SR_SEED_EMA != SR_SEED
    # the EMA is rounded with the low half of its own bits
    x = np.random.default_rng(1).standard_normal(e.size).astype(np.float32)
    r = sr_bits_ema(e, 7) & np.uint32(0xFFFF)
    assert (bf16_sr_ema(x, e, 7) == bf16_sr(x, e, 7, 0, r=r)).all()
    assert (bf16_sr_ema(x, e, 7) != bf16_sr(x, e, 7, 0)).any()


def test_the_ema_bits_are_independent_of_the_moment_bits():
    n = 1 << 18
    e = np.arange(n, dtype=np.uint64)
    for t in (1, 5, 999):
        ema = (sr_bits_ema(e, t) & np.uint32(0xFFFF)).astype(np.float64)
        mv = sr_bits(e, t)
        for other in ((mv & np.uint32(0xFFFF)).astype(np.float64), (mv >> np.uint32(16)).astype(np.float64)):
            # equal 16-bit draws as often as chance allows (n / 2^16 = 4 expected), no linear correlation
            assert int((ema == other).sum()) < 40
            assert abs(np.corrcoef(ema, other)[0, 1]) < 0.01
            # the rounding decisions of one value at the same element: agreement is chance (1/2 for a half-way fraction)
            assert abs(float(((ema < 32768) == (other < 32768)).mean()) - 0.5) < 0.01
        # uniform: each of 16 bins holds 1/16 of the draws
        hist = np.bincount((ema // 4096).astype(np.int64), minlength=16) / n
        assert np.abs(hist - 1 / 16).max() < 0.003


def test_a_bf16_ema_stalls_with_round_to_nearest_and_tracks_with_stochastic_rounding():
    """At d = 0.999 a step moves the EMA by 1e-3 of the gap: far below half a bf16 ulp, so round-to-nearest never moves
    it. Stochastic rounding moves it by a whole ulp with the probability of the fraction, and follows the fp32 EMA."""
    n, steps, d = 4096, 2000, 0.999
    c = ema_coefficient(d)
    e = np.arange(n, dtype=np.uint64)
    rng = np.random.default_rng(3)
    start = (1.0 + rng.random(n) * 0.5).astype(np.float32)
    start = widen((start.view(np.uint32) >> np.uint32(16)).astype(np.uint16))  # bf16 values
    target = (start + np.float32(0.5)).astype(np.float32)  # the weights sit half a unit above, ~32 bf16 ulps
    rn_bits = (start.view(np.uint32) >> np.uint32(16)).astype(np.uint16)
    sr = rn_bits.copy()
    f32 = start.copy()
    import torch

    for t in range(1, steps + 1):
        f32 = ema_step(f32, target, c)
        rn = torch.from_numpy(ema_step(widen(rn_bits), target, c)).bfloat16().view(torch.int16).numpy().view(np.uint16)
        assert (rn == rn_bits).all(), "round-to-nearest moved"
        sr = bf16_sr_ema(ema_step(widen(sr), target, c), e, t)
    expect = 0.5 * (1 - d ** steps)  # of the gap, ~0.432
    moved_sr = float((widen(sr) - start).mean())
    assert abs(moved_sr - expect) < 0.01 * expect, (moved_sr, expect)
    assert abs(float((f32 - start).mean()) - expect) < 1e-3
    # element by element the rounding noise adds up like a random walk that the decay pulls back: a stationary spread of
    # about sqrt(p (1 - p) / 2c) bf16 ulps (2^-7 at [1, 2)) around the fp32 EMA, p the fraction a step moves (~0.06 here)
    dev = (widen(sr) - f32) / 2.0 ** -7
    assert float(np.sqrt((dev ** 2).mean())) < 8, float(np.sqrt((dev ** 2).mean()))
    assert abs(float(dev.mean())) < 0.5


# ----------------------------------------------------------------------------- agreement
def test_agreement_accepts_one_coefficient_or_none_and_raises_otherwise():
    c = ema_record(ema_coefficient(0.999))
    assert c == float(np.float32(1 - 0.999)).hex() and ema_record(None) is None
    check_ema_agreement({0: {"t": 1}, 1: {"t": 1}})
    check_ema_agreement({0: {"ema": c}, 1: {"ema": c, "moments": "bf16"}})
    for bad in ({0: {"ema": c}, 1: {}}, {0: {"ema": c}, 1: {"ema": ema_record(ema_coefficient(0.99))}}):
        with pytest.raises(RuntimeError, match="disagree on the EMA"):
            check_ema_agreement(bad)
    # decays whose 1 - d rounds to the same fp32 agree: the holders run the same bits
    assert ema_record(ema_coefficient(0.999)) == ema_record(ema_coefficient(0.999 + 1e-13))


# ----------------------------------------------------------------------------- checkpoint format
def test_header_sections_and_payload_with_and_without_an_ema():
    n = 1000
    plain = {"elements": n}
    assert sections(n) == {"param": 0, "master": 2 * n, "m": 6 * n, "v": 10 * n}  # unchanged
    assert sections(n, 2) == {"param": 0, "master": 2 * n, "m": 6 * n, "v": 8 * n}
    assert sections(n, 4, ema=True) == {"param": 0, "master": 2 * n, "m": 6 * n, "v": 10 * n, "ema": 14 * n}
    assert sections(n, 2, ema=True) == {"param": 0, "master": 2 * n, "m": 6 * n, "v": 8 * n, "ema": 10 * n}
    assert payload_bytes(plain) == 14 * n
    assert payload_bytes({"elements": n, "moments": "bf16"}) == 10 * n
    with_ema = {"elements": n, "ema": {"decay": 0.999}}
    assert payload_bytes(with_ema) == 18 * n
    assert payload_bytes({**with_ema, "moments": "bf16"}) == 12 * n
    import torch

    assert file_dtype(with_ema, "ema") == torch.float32
    assert file_dtype({**with_ema, "moments": "bf16"}, "ema") == torch.bfloat16
    # the sections end where the payload does
    for h, ms in ((with_ema, 4), ({**with_ema, "moments": "bf16"}, 2)):
        assert sections(n, ms, ema=True)["ema"] + ms * n == payload_bytes(h)


def test_restore_reads_the_ema_where_files_have_it_and_seeds_it_elsewhere():
    a = {"name": "a", "ema": {"decay": 0.999}, "sections": sections(64, 4, ema=True)}
    b = {"name": "b", "sections": sections(64, 4)}
    c = {"name": "c", "ema": {"decay": 0.999}, "moments": "bf16", "sections": sections(32, 2, ema=True)}
    files = [(a, [(0, 64, 0)]), (b, [(64, 96, 0), (128, 160, 32)]), (c, [(96, 128, 0)])]
    reads = ckpt_read_plan([(16, 150)], files)
    have, seed = split_ema_reads(reads)
    assert [(h["name"], off, lo, hi) for h, off, lo, hi in have] == [("a", 16, 16, 64), ("c", 0, 96, 128)]
    assert seed == [(64, 96), (128, 150)]
    # every element is read or seeded, once
    assert merge_ranges([(lo, hi) for _, _, lo, hi in have] + seed) == [(16, 150)]
    assert split_ema_reads(ckpt_read_plan([(0, 64)], files)) == (ckpt_read_plan([(0, 64)], files), [])
    assert split_ema_reads([]) == ([], [])
