"""FT-ZeRO-1 bf16 moments, host logic (no GPU): the stochastic rounding's specification (``bf16_sr`` / ``sr_bits``), the
case that motivates it, the byte accounting of checkpoints and pools for both moment types, and the agreement check."""

from __future__ import annotations

import json

import numpy as np
import pytest
import torch

from _zero1_replicas import widen
from _zero1_sim import UNITS
from torchft_b200.checkpointing.sharded import encode_header, file_dtype, moment_size, payload_bytes, sections
from torchft_b200.parallel.zero1 import (PAGE_SHIFT, ShardLayout, bf16_sr, check_moment_agreement, moment_type,
                                         newest_complete_step, pool_pages, sr_bits)


def _down(x):
    """The bf16 neighbour of fp32 ``x`` towards zero, as bits."""
    return (np.asarray(x, dtype=np.float32).view(np.uint32) >> np.uint32(16)).astype(np.uint16)


# ----------------------------------------------------------------------------- the rounding
def test_exact_bf16_values_come_back_unchanged_for_every_r():
    exact = widen(np.array([0x0000, 0x8000, 0x3F80, 0xBF80, 0x0001, 0x8001, 0x7F7F, 0xFF7F, 0x4049, 0x0080], np.uint16))
    r = np.arange(1 << 16, dtype=np.uint32)
    for x in exact:
        out = bf16_sr(np.full(r.shape, x, np.float32), None, None, 0, r=r)
        assert (out == _down(x)).all(), x


def test_result_is_one_of_the_two_neighbours_and_rounds_away_from_zero_with_the_discarded_fraction():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(4096) * np.exp(rng.uniform(-30, 30, 4096))).astype(np.float32)
    x[:4] = [np.float32(1e-40), np.float32(-1e-40), np.float32(3.3e38), np.float32(-3.3e38)]  # subnormal, near the top
    e, t = np.arange(4096, dtype=np.uint64) * np.uint64(977), 12
    for which in (0, 1):
        out = bf16_sr(x, e, t, which)
        lo = _down(x)
        assert ((out == lo) | (out == lo + 1)).all()
        assert (np.abs(widen(out)) >= np.abs(widen(lo))).all()
    # every r: the value goes up exactly when r reaches 2**16 - (discarded bits)
    r = np.arange(1 << 16, dtype=np.uint32)
    for v in (np.float32(1.2345678), np.float32(-7.000123e-12)):
        frac = int(v.view(np.uint32)) & 0xFFFF
        up = bf16_sr(np.full(r.shape, v, np.float32), None, None, 0, r=r) != _down(v)
        assert int(up.sum()) == frac and (up == (r >= (1 << 16) - frac)).all()
    # the largest finite value may round to infinity, as round-to-nearest does
    assert bf16_sr(np.float32(3.4e38), None, None, 0, r=np.uint32(0xFFFF)) == 0x7F80


def test_inf_and_nan_pass_through():
    r = np.array([0, 1, 0x8000, 0xFFFF], np.uint32)
    for x, want in ((np.inf, 0x7F80), (-np.inf, 0xFF80)):
        assert (bf16_sr(np.full(4, x, np.float32), None, None, 0, r=r) == want).all()
    nans = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF80FFFF, 0x7FFFFFFF], np.uint32).view(np.float32)
    for which in (0, 1):
        out = bf16_sr(nans, np.arange(5), 3, which)
        assert np.isnan(widen(out)).all()
        assert ((out & 0x8000) == (nans.view(np.uint32) >> 16 & 0x8000)).all()  # the sign is kept


def test_mean_is_unbiased_over_elements_and_over_updates():
    """N draws of a fixed x: the error of the mean has standard deviation <= ulp / (2 sqrt(N)); 5 of those is the bound."""
    n = 1 << 16
    for x in (np.float32(1.2345678), np.float32(-0.00317), np.float32(1.0 + 2.0 ** -15)):
        ulp = float(np.abs(widen(_down(x) + 1) - widen(_down(x))))
        bound = 5 * ulp / (2 * np.sqrt(n))
        streams = {"elements": (np.arange(n, dtype=np.uint64) + np.uint64(1 << 33), 7),
                   "updates": (np.uint64(123456789), np.arange(1, n + 1)),
                   "both": (np.arange(n, dtype=np.uint64) * np.uint64(8), np.arange(n) % 251)}
        for name, (e, t) in streams.items():
            for which in (0, 1):
                got = widen(bf16_sr(np.full(n, x, np.float32), e, t, which)).astype(np.float64).mean()
                assert abs(got - float(x)) < bound, (x, name, which, got - float(x), bound)


def test_the_two_halves_are_uniform_and_uncorrelated():
    """Over N draws the sample correlation of two independent streams has standard deviation 1 / sqrt(N)."""
    n = 1 << 18
    bound = 5 / np.sqrt(n)
    for e, t in ((np.arange(n, dtype=np.uint64), 1), (np.uint64(40), np.arange(n)),
                 (np.arange(n, dtype=np.uint64) + np.uint64(0xFFFFFF00), 9)):  # the last crosses 2**32
        bits = sr_bits(e, t)
        lo, hi = (bits & 0xFFFF).astype(np.float64), (bits >> 16).astype(np.float64)
        assert abs(np.corrcoef(lo, hi)[0, 1]) < bound
        assert abs(np.corrcoef(lo[:-1], lo[1:])[0, 1]) < bound and abs(np.corrcoef(hi[:-1], hi[1:])[0, 1]) < bound
        for h in (lo, hi):  # uniform on [0, 2**16): mean within 5 sigma
            assert abs(h.mean() - 32767.5) < 5 * 65536 / np.sqrt(12 * n)
    # one element at consecutive updates and consecutive elements at one update do not share bits
    assert len(set(sr_bits(5, np.arange(1000)).tolist())) == 1000
    assert len(set(sr_bits(np.arange(1000), 5).tolist())) == 1000
    assert sr_bits(1 << 32, 0) != sr_bits(0, 0), "the upper index half counts"


def test_bits_are_a_pure_function_of_element_update_and_moment():
    e = np.arange(0, 80000, 8, dtype=np.uint64)
    a = sr_bits(e, 17)
    assert a.dtype == np.uint32 and (a == sr_bits(e.copy(), 17)).all()
    assert (a[::-1] == sr_bits(e[::-1], 17)).all(), "no dependence on the order elements are visited in"
    assert (sr_bits(e, 17)[100] == sr_bits(e[100], 17)).all()
    assert (a != sr_bits(e, 18)).mean() > 0.999
    x = np.full(e.shape, np.float32(0.3), np.float32)
    assert (bf16_sr(x, e, 17, 0) == bf16_sr(x, e, 17, 0)).all()
    assert (bf16_sr(x, e, 17, 0) != bf16_sr(x, e, 17, 1)).any()
    with pytest.raises(ValueError):
        bf16_sr(x, e, 17, 2)
    # a fixed vector: the definition does not drift
    assert sr_bits(np.array([0, 1, 8, 1 << 40], np.uint64), 1).tolist() == _reference_bits([0, 1, 8, 1 << 40], 1)


def _reference_bits(es, t):
    """The mix written out with Python integers."""
    out = []
    for e in es:
        x = ((e & 0xFFFFFFFF) * 0x9E3779B1 + (e >> 32) * 0x85EBCA77 + t * 0xC2B2AE3D + 0x27D4EB2F) & 0xFFFFFFFF
        x ^= x >> 16
        x = x * 0x85EBCA6B & 0xFFFFFFFF
        x ^= x >> 13
        x = x * 0xC2B2AE35 & 0xFFFFFFFF
        x ^= x >> 16
        out.append(x)
    return out


# ----------------------------------------------------------------------------- why not round to nearest
def test_second_moment_with_beta2_999_stalls_under_round_to_nearest_and_converges_under_bf16_sr():
    b2, g2, n, steps = np.float32(0.999), np.float32(1.0), 256, 6000
    e = np.arange(n, dtype=np.uint64)
    rn = torch.zeros(n, dtype=torch.bfloat16)
    sr = np.zeros(n, np.float32)
    for t in range(1, steps + 1):
        rn = (rn.float() * float(b2) + float(np.float32(1) - b2) * float(g2)).bfloat16()
        sr = widen(bf16_sr(b2 * sr + (np.float32(1) - b2) * g2, e, t, 1))
    rn = rn.float().numpy()
    assert (rn == rn[0]).all() and rn[0] < 0.3, f"round-to-nearest stalls far below g^2: {rn[0]}"
    # 1 - 0.999**6000 = 0.9975; one element's stationary noise is ulp / sqrt(6 * 2 * 0.001) = 3.6 % (1 sigma)
    assert abs(sr.mean() - 1.0) < 0.02, sr.mean()
    assert np.abs(sr - 1.0).max() < 0.2


# ----------------------------------------------------------------------------- bytes
def test_sections_and_payload_of_both_moment_types():
    e = 8 * 1234
    assert sections(e) == {"param": 0, "master": 2 * e, "m": 6 * e, "v": 10 * e}, "fp32 files keep their layout"
    assert sections(e, 4) == sections(e)
    assert sections(e, 2) == {"param": 0, "master": 2 * e, "m": 6 * e, "v": 8 * e}
    fp32, bf16 = {"elements": e}, {"elements": e, "moments": "bf16"}
    assert payload_bytes(fp32) == 14 * e and payload_bytes(bf16) == 10 * e
    assert moment_size(fp32) == 4 and moment_size(bf16) == 2
    assert file_dtype(fp32, "m") == torch.float32 and file_dtype(bf16, "v") == torch.bfloat16
    assert file_dtype(bf16, "master") == torch.float32 and file_dtype(bf16, "param") == torch.bfloat16
    for sec in (sections(e), sections(e, 2)):
        assert all(off % 16 == 0 for off in sec.values())
    with pytest.raises(ValueError):
        moment_size({"elements": e, "moments": "fp8"})
    # an fp32 header carries no new key, so its bytes are what they were
    h = {"version": 1, "numel": e, "T": 3, "elements": e, "sections": sections(e)}
    assert b"moments" not in encode_header(h)
    assert json.loads(encode_header(h)[16:].rstrip(b"\0")) == h


def test_pool_bytes_shrink_by_a_third():
    L = ShardLayout(UNITS, 2)
    page = 1 << 8
    for min_world in (1, 4, 7):
        pages = pool_pages(L, min_world, page)  # pages hold elements: the count does not depend on the moment type
        assert 3 * (pages * page * (4 + 2 * 2)) == 2 * (pages * page * (4 + 2 * 4))
    assert PAGE_SHIFT == 16


def test_newest_complete_step_passes_over_an_update_count_with_files_of_both_types():
    n = 64
    f = lambda t, lo, hi, **kw: dict({"T": t, "ranges": [[lo, hi, 0]]}, **kw)  # noqa: E731
    bf = {"moments": "bf16"}
    assert newest_complete_step([f(4, 0, 32), f(4, 32, 64)], n) == 4
    assert newest_complete_step([f(4, 0, 32, **bf), f(4, 32, 64, **bf)], n) == 4
    mixed = [f(5, 0, 32, **bf), f(5, 32, 64)]
    assert newest_complete_step(mixed, n) is None
    assert newest_complete_step(mixed + [f(4, 0, 64, **bf)], n) == 4
    assert newest_complete_step(mixed + [f(4, 0, 64, **bf), f(6, 0, 64)], n) == 6


# ----------------------------------------------------------------------------- agreement, configuration
def test_mixed_moment_types_in_one_quorum_raise_and_uniform_quorums_do_not():
    fp32 = {"t": 3, "hold": [[0, 64]]}
    bf16 = {"t": 3, "hold": [[0, 64]], "moments": "bf16"}
    assert "moments" not in fp32
    check_moment_agreement({0: fp32, 1: dict(fp32), 2: dict(fp32)})
    check_moment_agreement({0: bf16, 1: dict(bf16)})
    check_moment_agreement({0: bf16})
    for records in ({0: fp32, 1: bf16}, {0: bf16, 1: bf16, 2: fp32}):
        with pytest.raises(RuntimeError, match="disagree on the type of the optimizer moments"):
            check_moment_agreement(records)


def test_moment_type_from_the_argument_or_the_environment(monkeypatch):
    monkeypatch.delenv("TORCHFT_B200_Z1_MOMENTS", raising=False)
    assert moment_type(None) == torch.float32
    assert moment_type(torch.bfloat16) == torch.bfloat16
    monkeypatch.setenv("TORCHFT_B200_Z1_MOMENTS", "bf16")
    assert moment_type(None) == torch.bfloat16
    assert moment_type(torch.float32) == torch.float32, "the argument wins"
    monkeypatch.setenv("TORCHFT_B200_Z1_MOMENTS", "fp32")
    assert moment_type(None) == torch.float32
    monkeypatch.setenv("TORCHFT_B200_Z1_MOMENTS", "fp8")
    with pytest.raises(ValueError):
        moment_type(None)
    with pytest.raises(ValueError):
        moment_type(torch.float16)
