"""The node bounds of ``_node_ref`` on the CPU: a torch-CPU emulation of each fused node (bf16 operands, fp32 arithmetic,
one rounding to bf16 per stored tensor, e4m3 operands from the CPU model of ``_fp8_ref``) passes its bound, and each
mutant the GPU tests inject fails it while passing the whole-tensor check the nodes had before (2 % in norm)."""

import pytest
import torch

from _fp64 import _WORST, _report_margins  # noqa: F401
from _fp8_ref import dequantize, quantize_cols_t, quantize_rows
from _node_ref import check_linear, check_norm_linear, check_rope, check_swiglu_linear, fp8_linear, rel_norm, row_ratios

BF = torch.bfloat16
EPS = 1e-5
T, H, N, F = 67, 256, 384, 192  # a ragged token count


def _bf(t):
    return t.float().to(BF)


def _mm(a, b):
    """bf16 GEMM emulation: fp32 products and sums, one rounding."""
    return _bf(a.float() @ b.float())


def _deq(qs):
    return dequantize(*qs).float()


def _fp8_fwd(a, W):
    """Dequantised operands of the forward fp8 GEMM ``a @ W^T``: a per row, W per output channel."""
    return dequantize(*quantize_rows(a)), dequantize(*quantize_rows(W)).t()


def _fp8_bwd(dy, W):
    """... of the input-gradient fp8 GEMM ``dy @ W``: dy per row, W per input channel."""
    return dequantize(*quantize_rows(dy)), dequantize(*quantize_cols_t(W)).t()


def _data(seed, *shapes, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(*s, generator=g) * scale).to(BF) for s in shapes]


# ------------------------------------------------------------------------------------------------------- emulations
def emu_linear(x, W, res, dy, fp8):
    if fp8:
        A, B = _fp8_fwd(x, W)
        y = _bf(A.float() @ B.float())
        y = y if res is None else _bf(y.float() + res.float())
        A, B = _fp8_bwd(dy, W)
        dx = _bf(A.float() @ B.float())
    else:
        y = _bf(x.float() @ W.float().t() + (0 if res is None else res.float()))
        dx = _mm(dy, W)
    return {"y": y, "dx": dx, "dW": _mm(dy.t(), x), "dres": dy if res is not None else None}


def emu_rmsnorm(x, g):
    r = torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + EPS)
    return _bf(x.float() * r * g.float()), r


def emu_norm_linear(x, g, W, dy, dres, fp8):
    n, r = emu_rmsnorm(x, g)
    dn = _bf(_deq(quantize_rows(dy)) @ _deq(quantize_cols_t(W)).t()) if fp8 else _mm(dy, W)
    y = _bf(_deq(quantize_rows(n)) @ _deq(quantize_rows(W)).t()) if fp8 else _mm(n, W.t())
    xh = x.float() * r
    gw = dn.float() * g.float()
    dx = r * (gw - xh * (gw * xh).mean(-1, keepdim=True)) + (0 if dres is None else dres.float())
    return n, {"x_out": x, "y": y, "dx": _bf(dx), "dg": _bf((dn.float() * xh).sum(0)), "dW": _mm(dy.t(), n)}


def emu_swiglu(gu):
    g, u = gu.float().chunk(2, 1)
    return _bf(torch.nn.functional.silu(g) * u)


def emu_swiglu_linear(gu, W2, res, dy, fp8):
    a = emu_swiglu(gu)
    if fp8:
        y = _bf(_deq(quantize_rows(a)) @ _deq(quantize_rows(W2)).t())
        y = y if res is None else _bf(y.float() + res.float())
        da = _bf(_deq(quantize_rows(dy)) @ _deq(quantize_cols_t(W2)).t())
    else:
        y = _bf(a.float() @ W2.float().t() + (0 if res is None else res.float()))
        da = _mm(dy, W2)
    g, u = gu.float().chunk(2, 1)
    s = torch.sigmoid(g)
    d = da.float()
    dgu = torch.cat([d * u * (s + g * s * (1 - s)), d * g * s], 1)
    return a, {"y": y, "dgu": _bf(dgu), "dW": _mm(dy.t(), a), "dres": dy if res is not None else None}


def emu_rope(qkv, cs, B, S, Hq, Hkv, D, dq, dk, dv):
    def rot(x, sign):
        x2 = x.float().unflatten(-1, (-1, 2))
        c, s = cs[:S][None, :, None, :, 0], sign * cs[:S][None, :, None, :, 1]
        return _bf(torch.stack((x2[..., 0] * c - x2[..., 1] * s, x2[..., 0] * s + x2[..., 1] * c), -1).flatten(-2))

    p = qkv.view(B, S, Hq + 2 * Hkv, D)
    q, k, v = rot(p[:, :, :Hq], 1.0), rot(p[:, :, Hq:Hq + Hkv], 1.0), p[:, :, Hq + Hkv:]
    dqkv = torch.cat([rot(dq, -1.0), rot(dk, -1.0), dv], 2).reshape(B * S, -1)
    return q, k, v, dqkv


def _fp8_ops(fp8, fwd, bwd):
    return (fwd, bwd) if fp8 else (None, None)


# ------------------------------------------------------------------------------------------------------- the bounds
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("res", [False, True])
def test_linear_emulation_passes_its_bound(res, fp8):
    x, W, r, dy = _data(1, (T, H), (N, H), (T, N), (T, N))
    W = _bf(W.float() * 0.05)
    r = r if res else None
    got = emu_linear(x, W, r, dy, fp8)
    fwd, bwd = _fp8_ops(fp8, _fp8_fwd(x, W), _fp8_bwd(dy, W))
    check_linear(f"cpu linear res={res} fp8={fp8}", x, W, r, dy, got, fwd, bwd)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("dres", [False, True])
def test_norm_linear_emulation_passes_its_bound(dres, fp8):
    x, g, W, dy, d = _data(2, (T, H), (H,), (N, H), (T, N), (T, H))
    g = _bf(1 + 0.1 * g.float())
    W = _bf(W.float() * 0.05)
    d = d if dres else None
    n, got = emu_norm_linear(x, g, W, dy, d, fp8)
    fwd, bwd = _fp8_ops(fp8, _fp8_fwd(n, W), _fp8_bwd(dy, W))
    check_norm_linear(f"cpu norm_linear dres={dres} fp8={fp8}", x, g, W, dy, d, EPS, n, 1, got, fwd, bwd)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("res", [False, True])
def test_swiglu_linear_emulation_passes_its_bound(res, fp8):
    gu, W2, r, dy = _data(3, (T, 2 * F), (H, F), (T, H), (T, H))
    W2 = _bf(W2.float() * 0.05)
    r = r if res else None
    a, got = emu_swiglu_linear(gu, W2, r, dy, fp8)
    fwd, bwd = _fp8_ops(fp8, _fp8_fwd(a, W2), _fp8_bwd(dy, W2))
    check_swiglu_linear(f"cpu swiglu_linear res={res} fp8={fp8}", gu, W2, r, dy, a, got, fwd, bwd)


def _rope_case():
    from torchft_b200.ops import fused

    B, S, Hq, Hkv, D = 2, 33, 4, 2, 64
    cs = fused.rope_table(S + 5, D, 5e5, torch.device("cpu"))
    qkv, dq, dk, dv = _data(4, (B * S, (Hq + 2 * Hkv) * D), (B, S, Hq, D), (B, S, Hkv, D), (B, S, Hkv, D))
    return qkv, cs, (B, S, Hq, Hkv, D), dq, dk, dv


def test_rope_emulation_passes_its_bound():
    qkv, cs, dims, dq, dk, dv = _rope_case()
    q, k, v, dqkv = emu_rope(qkv, cs, *dims, dq, dk, dv)
    check_rope("cpu rope", qkv, cs, *dims, q, k, v, dq, dk, dv, dqkv)


# ----------------------------------------------------------------------------------------------------------- mutants
def _forget(prefix):
    """Drop the mutants' failures from the margin summary."""
    for what in [w for w in _WORST if w.startswith(prefix)]:
        del _WORST[what]


def _ulps(t, n, where):
    """``t`` with the elements at ``where`` moved ``n`` bf16 ulps away from zero."""
    t = t.clone()
    t.view(torch.int16)[where] += n
    return t


def test_residual_gradient_row_scaled_by_2_to_minus_5_fails_the_bound():
    x, g, W, dy, d = _data(2, (T, H), (H,), (N, H), (T, N), (T, H))
    g, W = _bf(1 + 0.1 * g.float()), _bf(W.float() * 0.05)
    n, good = emu_norm_linear(x, g, W, dy, d, False)
    bad_d = d.clone()
    bad_d[T // 2] = _bf(d[T // 2].float() * (1 + 2.0 ** -5))
    _, bad = emu_norm_linear(x, g, W, dy, bad_d, False)
    assert rel_norm(bad["dx"], good["dx"]) < 0.02
    with pytest.raises(AssertionError, match="dx"):
        check_norm_linear("cpu mutant dres row", x, g, W, dy, d, EPS, n, 1, bad)
    _forget("cpu mutant")


def test_one_kv_head_of_dv_moved_by_4_ulps_fails_the_bound():
    qkv, cs, dims, dq, dk, dv = _rope_case()
    bad_dv = _ulps(dv, 4, (slice(None), slice(None), 1))
    q, k, v, good = emu_rope(qkv, cs, *dims, dq, dk, dv)
    _, _, _, bad = emu_rope(qkv, cs, *dims, dq, dk, bad_dv)
    assert rel_norm(bad, good) < 0.02
    with pytest.raises(AssertionError, match="dv"):
        check_rope("cpu mutant dv head", qkv, cs, *dims, q, k, v, dq, dk, dv, bad)
    _forget("cpu mutant")


def test_one_weight_gradient_vector_moved_by_4_ulps_fails_the_bound():
    x, W, dy = _data(1, (T, H), (N, H), (T, N))
    W = _bf(W.float() * 0.05)
    got = emu_linear(x, W, None, dy, False)
    good = got["dW"]
    got["dW"] = _ulps(good, 4, (N // 3, slice(8 * 5, 8 * 6)))
    assert rel_norm(got["dW"], good) < 0.02
    with pytest.raises(AssertionError, match="dW"):
        check_linear("cpu mutant dW vector", x, W, None, dy, got)
    _forget("cpu mutant")


# ---------------------------------------------------------------------------------------------- the eager reference
def test_reference_loss_runs_in_fp64_and_bf16_on_the_cpu():
    """The eager reference in fp64 and in bf16 agree with the fp32 default to their precision (llama3_tiny)."""
    from torchft_b200.models.llama import CONFIGS, Llama
    from torchft_b200.models.reference import reference_loss

    cfg = CONFIGS["llama3_tiny"]
    torch.manual_seed(0)
    m = Llama(cfg)
    m.init_weights(0)
    tok = torch.randint(0, cfg.vocab_size, (2, 32))
    tgt = torch.randint(0, cfg.vocab_size, (2, 32))
    tgt[0, :5] = -100
    l32, g32 = reference_loss(m, tok, tgt)
    l64, g64 = reference_loss(m, tok, tgt, dtype=torch.float64)
    l16, g16 = reference_loss(m, tok, tgt, dtype=torch.bfloat16)
    l8, g8 = reference_loss(m, tok, tgt, dtype=torch.float64, linear=fp8_linear)
    assert abs(l8 - l64) <= 2.0 ** -5 * abs(l64) and all(rel_norm(g8[n], g64[n]) < 0.3 for n in g64)
    assert abs(l64 - l32) <= 1e-5 * abs(l64) and abs(l16 - l64) <= 2.0 ** -6 * abs(l64)
    for name in g64:
        assert g64[name].dtype == torch.float64 and g16[name].dtype == torch.bfloat16, name
        assert rel_norm(g32[name], g64[name]) < 1e-5, name
        assert rel_norm(g16[name], g64[name]) < 0.1, name


def test_fp8_linear_reference_quantises_like_the_cpu_model():
    """The eager reference's fp8 block linear: forward on x per row and W per output channel, input gradient on dy per
    row and W per input channel (the bytes of _fp8_ref), weight gradient on the unquantised operands."""
    x, W, dy = _data(6, (2, 33, H), (N, H), (2, 33, N))
    W = _bf(W.float() * 0.05)
    xl, Wl = x.double().requires_grad_(), W.double().requires_grad_()
    y = fp8_linear(xl, Wl)
    y.backward(dy.double())
    A, B = _fp8_fwd(x.view(-1, H), W)
    assert torch.equal(y.detach().view(-1, N), A @ B)
    A, B = _fp8_bwd(dy.view(-1, N), W)
    assert torch.equal(xl.grad.view(-1, H), A @ B)
    assert torch.equal(Wl.grad, dy.view(-1, N).double().t() @ x.view(-1, H).double())


def test_row_ratios_catch_one_row_a_norm_accepts():
    gen = torch.Generator().manual_seed(5)
    r64 = torch.randn(512, 256, generator=gen, dtype=torch.float64)
    b16 = r64.to(BF)
    bad = r64.to(BF)
    bad[300] = (r64[300] * (1 + 2.0 ** -5)).to(BF)
    assert rel_norm(bad, r64) < 0.02
    ratio, eg, eb = row_ratios(bad, r64, b16, 4)
    assert int(ratio.argmax()) == 300 and float(ratio.max()) > 1 and float(ratio[:300].max()) <= 0.5
    assert row_ratios(torch.ones(64), torch.ones(64), torch.ones(64), 4)[0].shape == (8,)  # 8-element norm vectors
