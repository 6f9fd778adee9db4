"""FT-ZeRO-1 gradient clipping: the threshold the optimizer accepts, from its argument or the environment (no GPU)."""

from __future__ import annotations

import math

import pytest

from torchft_b200.parallel.zero1 import Zero1Optimizer, clip_threshold


def test_unset_means_off(monkeypatch):
    monkeypatch.delenv("TORCHFT_B200_Z1_MAX_GRAD_NORM", raising=False)
    assert clip_threshold(None) is None
    monkeypatch.setenv("TORCHFT_B200_Z1_MAX_GRAD_NORM", "")
    assert clip_threshold(None) is None


def test_env_supplies_the_threshold_and_an_argument_overrides_it(monkeypatch):
    monkeypatch.setenv("TORCHFT_B200_Z1_MAX_GRAD_NORM", "1.0")
    assert clip_threshold(None) == 1.0
    assert clip_threshold(0.5) == 0.5
    monkeypatch.setenv("TORCHFT_B200_Z1_MAX_GRAD_NORM", "inf")
    assert math.isinf(clip_threshold(None))


@pytest.mark.parametrize("bad", [0.0, -1.0, float("nan"), float("-inf")])
def test_non_positive_or_nan_threshold_raises(bad, monkeypatch):
    monkeypatch.delenv("TORCHFT_B200_Z1_MAX_GRAD_NORM", raising=False)
    with pytest.raises(ValueError, match="max_grad_norm"):
        clip_threshold(bad)
    # the optimizer checks before it touches the process group or the device
    with pytest.raises(ValueError, match="max_grad_norm"):
        Zero1Optimizer(None, 8, max_grad_norm=bad)
    monkeypatch.setenv("TORCHFT_B200_Z1_MAX_GRAD_NORM", str(bad))
    with pytest.raises(ValueError, match="max_grad_norm"):
        Zero1Optimizer(None, 8)
