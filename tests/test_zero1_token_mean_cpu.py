"""FT-ZeRO-1 global token mean without a GPU: the trainer refuses the option off FT-ZeRO-1, and the pure-Python statement
of what the commit kernel computes (``token_mean_factor``, ``token_mean_commit``), which the GPU tests use as their
specification."""

from __future__ import annotations

import math

import numpy as np
import pytest

from torchft_b200.parallel.zero1 import token_mean_commit, token_mean_factor


@pytest.mark.parametrize("kw", [dict(zero1=False), dict(backend="nccl")])
def test_trainer_refuses_the_option_off_ft_zero1(kw):
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    with pytest.raises(ValueError, match=r"global_token_mean needs the FT-ZeRO-1 pipeline \(backend='b200', zero1=True\)"):
        FaultTolerantTrainer("llama3_debug", "unused:0", global_token_mean=True, **kw)


def test_llama_forward_takes_count_valid():
    import inspect

    from torchft_b200.models.llama import Llama

    p = inspect.signature(Llama.forward).parameters["count_valid"]
    assert p.default is True


@pytest.mark.parametrize("P,M,c", [(1, 1, 256), (2, 1, 8192), (3, 2, 4 * 8192), (8, 4, 2 * 8192)])
def test_factor_is_exactly_one_when_no_target_is_ignored(P, M, c):
    assert token_mean_factor(P * M * c, P * M * c) == 1.0


def test_factor_is_the_fp32_rounding_of_the_fp64_quotient():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        d = int(rng.integers(1, 1 << 40))
        n = int(rng.integers(1, d + 1))
        f = token_mean_factor(d, n)
        assert f == float(np.float32(np.float64(d) / np.float64(n)))
        assert abs(f - d / n) <= 2 ** -24 * (d / n)


def test_no_valid_target_gives_the_divisor_and_no_nan():
    assert token_mean_factor(3 * 2 * 512, 0) == 3 * 2 * 512
    out = token_mean_commit([(0, 0.0, 1024), (0, 0.0, 1024)], 1024, 2048)
    assert out["N"] == 0 and out["f"] == 2048.0 and out["loss"] == 0.0 and not out["veto"]
    # the reduced gradient is exactly 0 then: 0 * f is 0, and so is the norm
    out = token_mean_commit([(0, 0.0, 1024)], 1024, 1024, max_norm=1.0, norm=0.0)
    assert out["norm"] == 0.0 and out["coef"] == 1024.0 and not out["veto"]


def test_counts_and_losses_are_summed_in_rank_order():
    pub = [(100, 0.1, 512), (0, 0.0, 512), (37, 1e17, 512), (400, -1e17, 512)]
    out = token_mean_commit(pub, 512, 4 * 512)
    assert out["N"] == 537
    L = ((0.0 + 0.1) + 0.0 + 1e17) + -1e17  # fp64 in rank order (0.1 is lost against 1e17)
    assert out["loss"] == float(np.float32(L / 537)) == 0.0
    assert out["f"] == float(np.float32(2048 / 537))
    assert out["coef"] == out["f"]


def test_different_rows_veto_and_report_the_own_mean():
    pub = [(10, 25.0, 512), (20, 30.0, 1024)]
    for own, rows in ((0, 512), (1, 1024)):
        out = token_mean_commit(pub, rows, 2 * rows, own=own)
        assert out["veto"], "each rank sees a peer whose rows differ from its own"
        n, loss, _ = pub[own]
        assert out["loss"] == float(np.float32(loss / n))
    assert not token_mean_commit([(10, 25.0, 512), (20, 30.0, 512)], 512, 1024)["veto"]


def test_clipping_takes_the_norm_of_the_rescaled_gradient():
    f32 = np.float32
    pub = [(300, 1.0, 512), (212, 2.0, 512)]
    out = token_mean_commit(pub, 512, 1024, max_norm=1.0, norm=3.0)
    f = out["f"]
    assert f == float(f32(1024 / 512)) == 2.0
    assert out["norm"] == 6.0
    assert out["coef"] == float(f32(2.0) * min(f32(1.0), f32(f32(1.0) / f32(f32(6.0) + f32(1e-6))) * f32(1.0)))
    # with f = 1 norm and coefficient are what clipping alone gives
    full = token_mean_commit([(512, 1.0, 512)], 512, 512, max_norm=1.0, norm=3.0)
    assert full["f"] == 1.0 and full["norm"] == 3.0
    assert full["coef"] == float(min(f32(1.0), f32(f32(1.0) / f32(f32(3.0) + f32(1e-6))) * f32(1.0)))
    # an infinite max_norm never scales; a non-finite norm vetoes
    assert token_mean_commit(pub, 512, 1024, max_norm=math.inf, norm=3.0)["coef"] == f
    assert token_mean_commit(pub, 512, 1024, max_norm=1.0, norm=math.inf)["veto"]
