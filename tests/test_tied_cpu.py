"""Tied embeddings and Llama-3.1 RoPE scaling without a GPU: the Llama-3.2 parameter counts, the tied model's parameters
and flat layout, the RoPE table against an fp64 implementation of the scaling rule, and the refusals."""

import dataclasses
import math
from types import SimpleNamespace

import pytest
import torch

from torchft_b200.models.llama import CONFIGS, LLAMA3_1_ROPE_SCALING, FlatParams, Llama
from torchft_b200.ops import fused

COUNTS = {"llama3_2_1b": 1_235_814_400, "llama3_2_3b": 3_212_749_824}


def _tied_debug():
    return dataclasses.replace(CONFIGS["llama3_debug"], tie_embeddings=True, rope_scaling=LLAMA3_1_ROPE_SCALING)


@pytest.mark.parametrize("name", list(COUNTS))
def test_llama3_2_parameter_counts(name):
    cfg = CONFIGS[name]
    assert cfg.tie_embeddings and cfg.rope_scaling == (32.0, 1.0, 4.0, 8192) and cfg.max_seq_len == 8192
    assert cfg.num_params() == COUNTS[name]
    m = Llama(cfg, device="meta")
    assert sum(p.numel() for p in m.parameters()) == COUNTS[name]
    if name == "llama3_2_3b":
        assert cfg.head_dim == 128
    # the head GEMM still runs: tying leaves the FLOP count of the untied twin
    assert cfg.flops_per_token(8192) == dataclasses.replace(cfg, tie_embeddings=False).flops_per_token(8192)


def test_rope_scaling_is_immutable():
    with pytest.raises(AttributeError):
        LLAMA3_1_ROPE_SCALING.factor = 8.0  # type: ignore[misc]


def test_tied_model_has_no_output_parameter_and_no_duplicate_key():
    m = Llama(CONFIGS["llama3_2_1b"], device="meta")
    names = [n for n, _ in m.named_parameters(remove_duplicate=False)]
    assert "output" not in names and not hasattr(m, "output")
    assert len(names) == len(set(names))
    keys = list(m.state_dict().keys())
    assert len(keys) == len(set(keys)) and "output" not in keys
    assert m.head_weight() is m.tok_embeddings
    untied = Llama(CONFIGS["llama3_1b"], device="meta")
    assert untied.head_weight() is untied.output


def test_tied_flat_layout_and_stages():
    from torchft_b200.parallel.trainer import FaultTolerantTrainer, no_decay_ranges

    m = Llama(_tied_debug(), device="meta")
    flat = FlatParams(m, device="cpu")
    assert flat.params[0] is m.norm and flat.params[-1] is m.tok_embeddings
    assert all(o % FlatParams.ALIGN == 0 for o in flat.offsets)
    stages = m.param_stages()
    assert stages[0] == [m.tok_embeddings] and stages[-1] == [m.norm] and len(stages) == m.cfg.n_layers + 2
    ranges = FaultTolerantTrainer._compute_stage_ranges(SimpleNamespace(flat=flat, model=m))
    # forward order runs backwards through the buffer: the embedding's unit is the last range of it
    assert ranges[0][1] == flat.numel and ranges[-1][0] == 0
    assert all(a[0] == b[1] for a, b in zip(ranges, ranges[1:]))
    assert ranges[-1] == (0, FlatParams.ALIGN * math.ceil(m.cfg.dim / FlatParams.ALIGN))
    # the no-decay selectors see the tied weight under its one name
    (r,) = no_decay_ranges(flat, m, lambda n, p: n == "tok_embeddings")
    assert r == ranges[0]


def _inv(head_dim, theta=500000.0):
    return 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32) / head_dim))


def _rule64(f, factor, low, high, orig):
    """The Llama-3.1 rule on one fp64 frequency."""
    w = 2 * math.pi / f
    if w < orig / high:
        return f
    if w > orig / low:
        return f / factor
    s = (orig / w - low) / (high - low)
    return (1 - s) * f / factor + s * f


def test_unscaled_table_is_bit_equal_to_the_plain_formula():
    for D in (64, 128):
        inv = _inv(D)
        ang = torch.outer(torch.arange(300, dtype=torch.float32), inv)
        ref = torch.stack((ang.cos(), ang.sin()), dim=-1)
        assert torch.equal(fused.rope_table(300, D, 500000.0, torch.device("cpu")), ref)
        assert torch.equal(fused.rope_table(300, D, 500000.0, torch.device("cpu"), scaling=None), ref)


@pytest.mark.parametrize("D", [64, 128])
def test_scaled_table_follows_the_rule_in_fp64(D):
    factor, low, high, orig = LLAMA3_1_ROPE_SCALING
    inv = _inv(D)
    got = fused.rope_scaled_frequencies(inv, LLAMA3_1_ROPE_SCALING)
    bands = {"high": 0, "low": 0, "mid": 0}
    for i, f in enumerate(inv.double().tolist()):
        w = 2 * math.pi / f
        g = got[i].item()
        if w < orig / high:
            bands["high"] += 1
            assert got[i].view(torch.int32) == inv[i].view(torch.int32), (i, "high-frequency band changed")
        elif w > orig / low:
            bands["low"] += 1
            assert g == float(torch.tensor(f / factor, dtype=torch.float32)), (i, "low band is not f / factor")
        else:
            bands["mid"] += 1
            assert g == float(torch.tensor(_rule64(f, factor, low, high, orig), dtype=torch.float32)), (i, "band")
    assert all(bands.values()), bands  # every band is exercised at both head widths
    cs = fused.rope_table(8192, D, 500000.0, torch.device("cpu"), scaling=LLAMA3_1_ROPE_SCALING)
    ang = torch.outer(torch.arange(8192, dtype=torch.float32), got)
    assert torch.equal(cs, torch.stack((ang.cos(), ang.sin()), dim=-1))


def test_mutant_band_interpolated_on_the_wavelength():
    """The smooth band interpolated on w instead of orig / w: the fp64 rule check must fail."""
    factor, low, high, orig = LLAMA3_1_ROPE_SCALING
    inv = _inv(64).double()
    w = 2 * math.pi / inv
    s = (w - low) / (high - low)
    mutant = torch.where(w < orig / high, inv, torch.where(w > orig / low, inv / factor, (1 - s) * inv / factor + s * inv))
    ref = torch.tensor([_rule64(f, factor, low, high, orig) for f in inv.tolist()], dtype=torch.float64)
    assert not torch.equal(mutant.float(), ref.float())
    assert torch.equal(fused.rope_scaled_frequencies(_inv(64), LLAMA3_1_ROPE_SCALING), ref.float())


def test_reference_scaling_is_its_own_and_agrees():
    from torchft_b200.models.reference import _scaled

    for D in (64, 128):
        assert torch.equal(_scaled(_inv(D), LLAMA3_1_ROPE_SCALING, torch.float64).float(),
                           fused.rope_scaled_frequencies(_inv(D), LLAMA3_1_ROPE_SCALING))


def test_embedding_bwd_refuses_a_row_width_off_the_vector():
    dx = torch.zeros(5, 12, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="multiple of 8"):
        fused.embedding_bwd(torch.zeros(5, dtype=torch.int64), dx, torch.zeros(7, 12, dtype=torch.bfloat16))
    from torchft_b200.ops import _native

    # the launcher itself refuses it before any launch, as ValueError too
    with pytest.raises(ValueError, match="multiple of 8"):
        _native.load().embedding_bwd(0, 0, 0, 12, 0, 0, 5, 12, 0)


def test_hsdp_refuses_a_tied_model_before_building_anything():
    from torchft_b200.parallel.hsdp import HSDPTrainer

    with pytest.raises(ValueError, match="tied"):
        HSDPTrainer("llama3_2_1b", "localhost:0", shards=1)
