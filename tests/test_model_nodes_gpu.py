"""The fused Llama nodes (``ops/fused.py``), the model step and its activation checkpointing against fp64 and against
themselves, at Llama-3 1B and 8B layer shapes.

1. Each node, bf16 and fp8, element by element against the fp64 references and bounds of ``_node_ref``, and bit for bit
   against the same verified kernels and torch GEMMs composed by hand with the same operand layouts (the zero-tolerance
   check that catches plumbing: a reused buffer, a stride, a residual routed to the wrong place). The node's weight
   gradient is taken both into a new tensor and into a NaN-filled flat-gradient slot.
2. Exact equalities of the model step: activation checkpointing and direct weight gradients change no bit.
3. The model's loss and every parameter gradient, row by row, against an fp64 eager reference, with the bf16 eager
   reference as the yardstick.
4. Mutants, injected from the test, that the new checks catch and the old whole-tensor norms do not.
"""

import contextlib
import dataclasses

import pytest
import torch

from _fp64 import _WORST, _report_margins  # noqa: F401
from _node_ref import (bits_equal, check_linear, check_norm_linear, check_rope, check_swiglu_linear, fp8_linear, rel_norm,
                       row_ratios)

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn
EPS = 1e-5
RAN = set()  # (node, fp8, res/dres, direct, shape) of every node case below, for test_every_case_ran
SHAPES = {"1b": ("llama3_1b", 8192), "8b": ("llama3_8b", 8192), "1b-T8191": ("llama3_1b", 8191)}


def _K():
    from torchft_b200.ops import _native

    return _native.load()


def _sp():
    from torchft_b200.ops import _native

    return _native.stream_ptr()


def _cfg(shape):
    from torchft_b200.models.llama import CONFIGS

    name, T = SHAPES[shape]
    return CONFIGS[name], T


def _randn(gen, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=gen) * scale).to(BF16)


def _leaf(t):
    return t.detach().clone().requires_grad_()


def _deq(q, s):
    """fp64 values of e4m3 ``q [R, C]`` with one scale per row."""
    return q.view(E4M3).double() * s.double().reshape(-1, 1)


def _twice(f):
    """``f()``'s tensors, after checking that a second call returns the same bits."""
    a, b = f(), f()
    for x, y in zip(a, b):
        bits_equal(x.view(torch.uint8) if x.dtype == E4M3 else x, y.view(torch.uint8) if y.dtype == E4M3 else y,
                   "repeat of a kernel call")
    return a


def _mm8(a, b):
    """The rowwise fp8 GEMM of the nodes, called directly."""
    return torch._scaled_mm(a[0], b[0], scale_a=a[1], scale_b=b[1], out_dtype=BF16, use_fast_accum=False)


def _fwd8(a, W):
    """Forward fp8 GEMM ``a @ W^T`` by hand; returns the output and the dequantised operands."""
    from torchft_b200.ops import fused

    qw, sw = _twice(lambda: fused.fp8_rows(W))
    return _mm8(a, (qw.t(), sw.view(1, -1))), (_deq(*a), _deq(qw, sw).t())


def _dgrad8(dy2, W):
    """Input-gradient fp8 GEMM ``dy @ W`` by hand; returns the output and the dequantised operands."""
    from torchft_b200.ops import fused

    qd, sd = _twice(lambda: fused.fp8_rows(dy2))
    qt, st = _twice(lambda: fused.fp8_cols_t(W))
    return _mm8((qd, sd), (qt.t(), st)), (_deq(qd, sd), _deq(qt, st).t())


def _same(got, hand, tag):
    for name, v in hand.items():
        if v is None:
            assert got[name] is None, (tag, name)
        else:
            bits_equal(got[name], v, f"{tag} {name} vs the hand composition")


def _slot(W, direct):
    """With ``direct``, a NaN-filled flat-gradient slot for W's weight gradient (what FlatParams gives it)."""
    if not direct:
        return None
    W._flat_grad = torch.full_like(W, float("nan"))
    return W._flat_grad


def _landed(W, slot, tag):
    if slot is not None:
        bits_equal(slot, W.grad, f"{tag}: the weight gradient in its flat slot")


# ---------------------------------------------------------------------------------------------------- norm_linear_res
def _norm_linear_node(x0, g0, W0, dy, dres, fp8, direct, tag, hooks=()):
    from torchft_b200.ops import fused

    x, g, W = _leaf(x0), _leaf(g0), _leaf(W0)
    slot = _slot(W, direct)
    xs, y = fused.norm_linear_res(x, g, W, EPS, fp8=fp8)
    for h in hooks:
        xs.register_hook(h)
    out = {"x_out": xs.detach(), "y": y.detach()}
    torch.autograd.backward([y, xs] if dres is not None else [y], [dy, dres] if dres is not None else [dy])
    _landed(W, slot, tag)
    return {**out, "dx": x.grad, "dg": g.grad, "dW": W.grad}


def _norm_linear_by_hand(x, g, W, dy, dres, fp8):
    """The node's kernels and GEMMs composed here; returns (recomputed n, outputs, fp8 operands)."""
    K, sp = _K(), _sp()
    T, H = x.shape
    rstd = torch.empty(T, device="cuda")
    fwd = bwd = None

    def norm():
        n = torch.empty_like(x)
        K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), T, H, EPS, sp)
        return (n, rstd.clone())

    if fp8:
        def norm8():
            q = torch.empty(T, H, dtype=E4M3, device="cuda")
            qs = torch.empty(T, 1, device="cuda")
            K.rmsnorm_fwd_fp8(x.data_ptr(), g.data_ptr(), q.data_ptr(), qs.data_ptr(), rstd.data_ptr(), T, H, EPS, sp)
            return q, qs

        y, fwd = _fwd8(_twice(norm8), W)
    n, r = _twice(norm)
    if not fp8:
        y = n @ W.t()
    dW = dy.t() @ n
    if fp8:
        dn, bwd = _dgrad8(dy, W)
    else:
        dn = dy @ W
    dx, dg = torch.empty_like(x), torch.empty_like(g)
    partial = torch.empty(K.rmsnorm_bwd_grid(T), H, device="cuda")
    K.rmsnorm_bwd(dn.data_ptr(), x.data_ptr(), g.data_ptr(), r.data_ptr(), dx.data_ptr(), partial.data_ptr(),
                  dg.data_ptr(), False, T, H, sp, dres.data_ptr() if dres is not None else 0)
    return n, {"x_out": x, "y": y, "dx": dx, "dg": dg, "dW": dW}, fwd, bwd


def _norm_linear_data(shape, which, seed):
    cfg, T = _cfg(shape)
    N = (cfg.n_heads + 2 * cfg.n_kv_heads) * cfg.head_dim if which == "wqkv" else 2 * cfg.ffn_dim
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = _randn(gen, T, cfg.dim)
    g = (1 + 0.1 * torch.randn(cfg.dim, device="cuda", generator=gen)).to(BF16)
    W = _randn(gen, N, cfg.dim, scale=0.02)
    dy = _randn(gen, T, N, scale=1e-2)
    dres = _randn(gen, T, cfg.dim, scale=1e-2)
    return x, g, W, dy, dres


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("dres", [False, True])
@pytest.mark.parametrize("which", ["wqkv", "w13"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_norm_linear_res(shape, which, dres, fp8):
    x, g, W, dy, d = _norm_linear_data(shape, which, seed=len(shape) + len(which) + 2 * dres + fp8)
    d = d if dres else None
    tag = f"norm_linear {shape} {which} dres={dres} fp8={fp8}"
    n, hand, fwd, bwd = _norm_linear_by_hand(x, g, W, dy, d, fp8)
    for direct in (False, True):
        got = _norm_linear_node(x, g, W, dy, d, fp8, direct, tag)
        _same(got, hand, f"{tag} direct={direct}")
        RAN.add(("norm_linear", fp8, dres, direct, shape))
    check_norm_linear(tag, x, g, W, dy, d, EPS, n, _K().rmsnorm_bwd_grid(x.shape[0]), got, fwd, bwd)


# ------------------------------------------------------------------------------------------------------ swiglu_linear
def _swiglu_linear_node(gu0, W0, res0, dy, fp8, direct, tag):
    from torchft_b200.ops import fused

    gu, W = _leaf(gu0), _leaf(W0)
    res = _leaf(res0) if res0 is not None else None
    slot = _slot(W, direct)
    y = fused.swiglu_linear(gu, W, res=res, fp8=fp8)
    y.backward(dy)
    _landed(W, slot, tag)
    return {"y": y.detach(), "dgu": gu.grad, "dW": W.grad, "dres": res.grad if res is not None else None}


def _swiglu_linear_by_hand(gu, W2, res, dy, fp8):
    K, sp = _K(), _sp()
    T, F = gu.shape[0], gu.shape[1] // 2
    fwd = bwd = None

    def prod():
        a = torch.empty(T, F, dtype=BF16, device="cuda")
        K.swiglu_fwd(gu.data_ptr(), a.data_ptr(), T, F, sp)
        return (a,)

    if fp8:
        def prod8():
            q = torch.empty(T, F, dtype=E4M3, device="cuda")
            qs = torch.empty(T, 1, device="cuda")
            K.fp8_swiglu(gu.data_ptr(), q.data_ptr(), qs.data_ptr(), T, F, sp)
            return q, qs

        y, fwd = _fwd8(_twice(prod8), W2)
        if res is not None:
            y.add_(res)
    (a,) = _twice(prod)
    if not fp8:
        y = a @ W2.t() if res is None else torch.addmm(res, a, W2.t())
    dW = dy.t() @ a
    if fp8:
        da, bwd = _dgrad8(dy, W2)
    else:
        da = torch.mm(dy, W2, out=torch.empty_like(a))
    dgu = torch.empty_like(gu)
    K.swiglu_bwd(da.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, F, sp)
    return a, {"y": y, "dgu": dgu, "dW": dW, "dres": dy if res is not None else None}, fwd, bwd


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_swiglu_linear(shape, res, fp8):
    cfg, T = _cfg(shape)
    gen = torch.Generator(device="cuda").manual_seed(100 + len(shape) + 2 * res + fp8)
    gu = _randn(gen, T, 2 * cfg.ffn_dim, scale=2.0)
    W2 = _randn(gen, cfg.dim, cfg.ffn_dim, scale=0.02)
    r = _randn(gen, T, cfg.dim) if res else None
    dy = _randn(gen, T, cfg.dim, scale=1e-2)
    tag = f"swiglu_linear {shape} res={res} fp8={fp8}"
    a, hand, fwd, bwd = _swiglu_linear_by_hand(gu, W2, r, dy, fp8)
    for direct in (False, True):
        got = _swiglu_linear_node(gu, W2, r, dy, fp8, direct, tag)
        _same(got, hand, f"{tag} direct={direct}")
        RAN.add(("swiglu_linear", fp8, res, direct, shape))
    check_swiglu_linear(tag, gu, W2, r, dy, a, got, fwd, bwd)


# ------------------------------------------------------------------------------------------------------------- linear
def _linear_node(x0, W0, res0, dy, fp8, direct, tag):
    from torchft_b200.ops import fused

    x, W = _leaf(x0), _leaf(W0)
    res = _leaf(res0) if res0 is not None else None
    slot = _slot(W, direct)
    y = fused.linear(x, W, res=res, fp8=fp8)
    assert y.shape == x.shape[:-1] + (W.shape[0],)
    y.backward(dy)
    _landed(W, slot, tag)
    return {"y": y.detach(), "dx": x.grad, "dW": W.grad, "dres": res.grad if res is not None else None}


def _linear_by_hand(x, W, res, dy, fp8):
    """x, res, dy 3-D as the node gets them; the outputs come back 2-D."""
    from torchft_b200.ops import fused

    x2, dy2 = x.reshape(-1, x.shape[-1]), dy.reshape(-1, dy.shape[-1])
    r2 = res.reshape(-1, res.shape[-1]) if res is not None else None
    fwd = bwd = None
    if fp8:
        y, fwd = _fwd8(_twice(lambda: fused.fp8_rows(x2)), W)
        if r2 is not None:
            y.add_(r2)
        dx, bwd = _dgrad8(dy2, W)
    else:
        y = (x @ W.t()).reshape(x2.shape[0], -1) if r2 is None else torch.addmm(r2, x2, W.t())
        dx = dy2 @ W
    return {"y": y, "dx": dx, "dW": dy2.t() @ x2, "dres": dy2 if res is not None else None}, fwd, bwd


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_linear(shape, res, fp8):
    """wo of the model on a 3-D [B, S, dim] input, B = 2 where T is even."""
    cfg, T = _cfg(shape)
    B = 2 if T % 2 == 0 else 1
    gen = torch.Generator(device="cuda").manual_seed(200 + len(shape) + 2 * res + fp8)
    x = _randn(gen, B, T // B, cfg.dim)
    W = _randn(gen, cfg.dim, cfg.dim, scale=0.02)
    r = _randn(gen, B, T // B, cfg.dim) if res else None
    dy = _randn(gen, B, T // B, cfg.dim, scale=1e-2)
    tag = f"linear {shape} res={res} fp8={fp8}"
    hand, fwd, bwd = _linear_by_hand(x, W, r, dy, fp8)
    if res and not fp8:
        # what the residual bound of _node_ref.with_res rests on: the addmm epilogue rounds the product first
        x2, r2 = x.reshape(-1, cfg.dim), r.reshape(-1, cfg.dim)
        bits_equal(torch.addmm(r2, x2, W.t()), x2 @ W.t() + r2, f"{tag}: addmm vs the product rounded, then the add")
    flat = lambda t: None if t is None else t.reshape(-1, t.shape[-1])  # noqa: E731
    for direct in (False, True):
        got = _linear_node(x, W, r, dy, fp8, direct, tag)
        assert got["dx"].shape == x.shape and (r is None or got["dres"].shape == r.shape)
        got = {k: flat(v) if k != "dW" else v for k, v in got.items()}
        _same(got, hand, f"{tag} direct={direct}")
        RAN.add(("linear", fp8, res, direct, shape))
    check_linear(tag, flat(x), W, flat(r), flat(dy), got, fwd, bwd)


# ------------------------------------------------------------------------------------------------------- RoPE + SDPA
def _rope_sdpa(qkv0, cs, B, S, Hq, Hkv, D, do, hooks=()):
    """rope_qkv then causal GQA SDPA, backward from ``do``; SDPA's dq, dk, dv captured by hooks on q, k, v (``hooks``
    run after the capture, on v's gradient)."""
    from torchft_b200.ops import fused

    qkv = _leaf(qkv0)
    q, k, v = fused.rope_qkv(qkv, cs, B, S, Hq, Hkv, D)
    cap = {}
    for name, t in (("dq", q), ("dk", k), ("dv", v)):
        t.register_hook(lambda gr, name=name: cap.__setitem__(name, gr))
    for h in hooks:
        v.register_hook(h)
    o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                         is_causal=True, enable_gqa=True)
    o.backward(do)
    return q.detach(), k.detach(), v.detach(), cap, qkv.grad


def _rope_case(B, S, D, seed):
    from torchft_b200.ops import fused

    Hq, Hkv = 32, 8
    cs = fused.rope_table(8192, D, 5e5, torch.device("cuda"))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    qkv = _randn(gen, B * S, (Hq + 2 * Hkv) * D)
    do = _randn(gen, B, Hq, S, D)
    return qkv, cs, (B, S, Hq, Hkv, D), do


@pytest.mark.parametrize("B,S", [(1, 8192), (2, 4096)])
@pytest.mark.parametrize("D", [64, 128])
def test_rope_qkv_through_sdpa(D, B, S):
    """D = 64 (1B) and 128 (8B), GQA 32/8. The backward reads SDPA's gradients in the strides SDPA returned; the hand
    composition feeds the same launcher contiguous copies."""
    K = _K()
    qkv, cs, dims, do = _rope_case(B, S, D, seed=D + S)
    _, _, Hq, Hkv, _ = dims
    q, k, v, cap, dqkv = _rope_sdpa(qkv, cs, *dims, do)
    tag = f"rope+sdpa D={D} B={B} S={S}"
    row = (Hq + 2 * Hkv) * D
    q2, k2, v2 = (torch.empty(B, S, h, D, device="cuda", dtype=BF16) for h in (Hq, Hkv, Hkv))
    K.rope_qkv(qkv.data_ptr(), row, q2.data_ptr(), k2.data_ptr(), v2.data_ptr(),
               [*q2.stride()[:3], *k2.stride()[:3], *v2.stride()[:3]], cs.data_ptr(), B * S, S, D, Hq, Hkv, 0, _sp())
    for a, b, name in ((q, q2, "q"), (k, k2, "k"), (v, v2, "v")):
        bits_equal(a, b, f"{tag} {name} vs the launcher")
    dq, dk, dv = (cap[n].contiguous() for n in ("dq", "dk", "dv"))
    hand = torch.empty(B * S, row, dtype=BF16, device="cuda")
    K.rope_qkv(hand.data_ptr(), row, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
               [*dq.stride()[:3], *dk.stride()[:3], *dv.stride()[:3]], cs.data_ptr(), B * S, S, D, Hq, Hkv, 1, _sp())
    bits_equal(dqkv, hand, f"{tag} dqkv vs the launcher on contiguous copies")
    RAN.add(("rope", False, None, False, f"D={D} B={B} S={S}"))
    check_rope(tag, qkv, cs, *dims, q, k, v, cap["dq"], cap["dk"], cap["dv"], dqkv)


# ----------------------------------------------------------------------------------------------- the model vs fp64
# The yardstick of a row is the error of the bf16 eager reference in that row. Measured on an H100 80GB HBM3 (700 W), the
# fused bf16 model's median row error is 0.65 to 1.03 of the eager one (above 0.92 only in a 32-vector norm weight of
# llama3_debug). Yet with factor 2 a few rows of some parameters exceed it: at most 29 of 2048 rows of the second
# layer's wo at 1B shapes, worst |g - r64| = 3.7 |b16 - r64|. They are rows where the eager rounding errors happen to
# cancel and the fused ones happen not to: two independent roundings of the same sums, not a fault (a fault moves every
# row it touches, as the mutants below do). So the per-row factor is 4, and the median row error of the model must not
# exceed 1.25 times the eager one: a model twice as noisy as the eager bf16 one fails that in every parameter.
# fp8: the e4m3 quantisation of the block linears errs by up to 2^-4 per operand, so the model's gradients are 7-25 %
# (median row) away from the unquantised fp64 model. The reference therefore quantises the same operands the same way
# (_node_ref.fp8_linear) in fp64 and in bf16. Both errors are then dominated by e4m3 roundings that land on the other
# side of a boundary, in different elements for the model and for the eager run: the medians are equal (0.97 to 1.0 of
# the eager one, 1.26 in a 32-vector norm weight of llama3_debug), and the worst row is 4.7 times the eager error. The
# fp8 factor is 6 and the median limit 1.5; a wrong scale or a wrong operand moves every row far beyond both.
FACTOR = {False: 4, True: 6}
MEDIAN = {False: 1.25, True: 1.5}
MODEL_CASES = [("llama3_debug", 2, 512, False), ("llama3_debug", 2, 512, True), ("1b-2layer", 1, 2048, False),
               ("8b-1layer", 1, 1024, False)]


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name,B,S,ignored", MODEL_CASES)
def test_model_rows_against_fp64(name, B, S, ignored, fp8):
    """Every row of every parameter gradient (each 8-element vector of a norm weight), and the loss:
    |g - r64| <= FACTOR |b16 - r64| + 2^-9 |r64|, r64 the eager reference in fp64 and b16 the same in bf16 (with the
    model's e4m3 operands for fp8); and the median row error within MEDIAN of the eager one. The one-layer 8B-shaped model has a 32768-token vocabulary."""
    from torchft_b200.models.llama import CONFIGS, Llama
    from torchft_b200.models.reference import reference_loss

    if name == "8b-1layer":
        cfg = dataclasses.replace(CONFIGS["llama3_8b"], n_layers=1, vocab_size=32768, fp8_linears=fp8)
    else:
        cfg = _model_cfg(name, fp8_linears=fp8)
    tok, tgt = _batch(cfg, B, S, seed=17, ignored=ignored)
    m = Llama(cfg, device="cuda")
    m.init_weights(0)
    loss = m(tok, tgt)
    loss.backward()
    lin = fp8_linear if fp8 else None
    l16, g16 = reference_loss(m, tok, tgt, dtype=torch.bfloat16, linear=lin)
    l64, g64 = reference_loss(m, tok, tgt, dtype=torch.float64, linear=lin)
    tag = f"{name} B={B} S={S} ignored={ignored} fp8={fp8}"
    lr = abs(loss.item() - l64) / (FACTOR[fp8] * abs(l16 - l64) + 2.0 ** -9 * abs(l64))
    print(f"[model rows] {tag} loss {loss.item():.9g} r64 {l64:.9g} b16 {l16:.9g} ratio {lr:.3g}")
    bad = []
    for pname, p in m.named_parameters():
        ratio, eg, eb = row_ratios(p.grad, g64[pname], g16[pname], FACTOR[fp8])
        i = int(ratio.argmax())
        med = float(eg.median() / eb.median())
        print(f"[model rows] {tag} {pname}: worst row {i} ratio {float(ratio[i]):.3g}, median row error "
              f"{float(eg.median()):.3g} vs eager {float(eb.median()):.3g}")
        if float(ratio[i]) > 1 or med > MEDIAN[fp8]:
            bad.append((pname, i, float(ratio[i]), med))
        del g64[pname], g16[pname]
    assert lr <= 1, (tag, "loss", lr)
    assert not bad, (tag, bad)


# ------------------------------------------------------------------------------------------------------------ mutants
def _forget(prefix):
    for what in [w for w in _WORST if w.startswith(prefix)]:
        del _WORST[what]


def _ulps(t, n, where):
    t = t.clone()
    t.view(torch.int16)[where] += n
    return t


def test_mutant_residual_gradient_row_scaled():
    """One token row of the residual gradient that norm_linear_res adds into dx, scaled by 1 + 2^-5 on its way in."""
    x, g, W, dy, d = _norm_linear_data("1b", "wqkv", seed=7)

    def scale_row(gr):
        gr = gr.clone()
        gr[4321] *= 1 + 2.0 ** -5
        return gr

    good = _norm_linear_node(x, g, W, dy, d, False, False, "mutant")
    bad = _norm_linear_node(x, g, W, dy, d, False, False, "mutant", hooks=(scale_row,))
    n, _, _, _ = _norm_linear_by_hand(x, g, W, dy, d, False)
    assert rel_norm(bad["dx"], good["dx"]) < 0.02  # the old norm check passes it
    with pytest.raises(AssertionError, match="dx"):
        check_norm_linear("mutant dres row", x, g, W, dy, d, EPS, n, _K().rmsnorm_bwd_grid(x.shape[0]), bad)
    _forget("mutant")


def test_mutant_one_kv_head_of_dv_moved_by_4_ulps():
    qkv, cs, dims, do = _rope_case(1, 8192, 64, seed=5)
    _, _, _, _, good = _rope_sdpa(qkv, cs, *dims, do)
    q, k, v, cap, bad = _rope_sdpa(qkv, cs, *dims, do, hooks=(lambda gr: _ulps(gr, 4, (slice(None), slice(None), 3)),))
    assert rel_norm(bad, good) < 0.02
    with pytest.raises(AssertionError, match="dv"):
        check_rope("mutant dv head", qkv, cs, *dims, q, k, v, cap["dq"], cap["dk"], cap["dv"], bad)
    _forget("mutant")


@pytest.mark.parametrize("direct", [False, True])
def test_mutant_weight_gradient_vector_moved_by_4_ulps(monkeypatch, direct):
    """An 8-element vector of wo's weight gradient moved 4 ulps inside the node (a wrapper around ``_wgrad``), whether
    the GEMM wrote a new tensor or the flat slot. The bit equality with the hand composition catches it; the fp64 bound
    alone does not at this shape: with K = T = 8192 its slack K U (|dy|^T @ |x|) is a few percent of |dW|, more than 4
    ulps (test_node_ref_cpu shows the bound catching it at T = 67)."""
    from torchft_b200.ops import fused

    cfg, T = _cfg("1b")
    gen = torch.Generator(device="cuda").manual_seed(8)
    x = _randn(gen, 2, T // 2, cfg.dim)
    W = _randn(gen, cfg.dim, cfg.dim, scale=0.02)
    dy = _randn(gen, 2, T // 2, cfg.dim, scale=1e-2)
    good = _linear_node(x, W, None, dy, False, direct, "mutant")
    real = fused._wgrad

    def wrong(dy2, x2, W_):
        dW = real(dy2, x2, W_)
        dW.view(torch.int16)[1234, 8 * 50:8 * 51] += 4
        return dW

    monkeypatch.setattr(fused, "_wgrad", wrong)
    bad = _linear_node(x, W, None, dy, False, direct, "mutant")
    monkeypatch.setattr(fused, "_wgrad", real)
    assert rel_norm(bad["dW"], good["dW"]) < 0.02
    hand, _, _ = _linear_by_hand(x, W, None, dy, False)
    bits_equal(good["dW"], hand["dW"], "unmutated weight gradient")
    with pytest.raises(AssertionError, match="mutated weight gradient"):
        bits_equal(bad["dW"], hand["dW"], "mutated weight gradient")


# ---------------------------------------------------------------------------------------------- the model, exactly
def _model_cfg(name, **kw):
    """llama3_debug, or two layers of llama3_1b with its vocabulary."""
    from torchft_b200.models.llama import CONFIGS

    if name == "1b-2layer":
        return dataclasses.replace(CONFIGS["llama3_1b"], n_layers=2, **kw)
    return dataclasses.replace(CONFIGS[name], **kw)


def _batch(cfg, B, S, seed, ignored=False):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    tok = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=gen)
    tgt = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=gen)
    if ignored:
        tgt[torch.rand(B, S, device="cuda", generator=gen) < 0.25] = -100
    return tok, tgt


MODEL_BATCH = {"llama3_debug": (2, 512), "1b-2layer": (1, 2048)}


def _step(cfg, tok, tgt):
    from torchft_b200.models.llama import Llama

    m = Llama(cfg, device="cuda")
    m.init_weights(0)
    loss = m(tok, tgt)
    loss.backward()
    return loss.detach(), {n: p.grad for n, p in m.named_parameters()}


@contextlib.contextmanager
def _deterministic_attention(monkeypatch):
    """SDPA's flash backward, with deterministic algorithms on: by default it accumulates dq with atomics, and at 1B
    layer shapes two identical steps then differ in the last bits of most gradients. The flag holds for every op inside
    the block, not only attention (uninitialised torch.empty memory is then filled with NaN, too). Setting
    CUBLAS_WORKSPACE_CONFIG after cuBLAS is initialised only satisfies torch's check that comes with the flag; it does
    not change cuBLAS's workspace, and does not need to: on one stream the same GEMM gives the same bits."""
    from torch.nn.attention import SDPBackend, sdpa_kernel

    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
            yield
    finally:
        torch.use_deterministic_algorithms(False)


def _equal_steps(a, b, what):
    bits_equal(a[0], b[0], f"{what}: loss")
    for name in a[1]:
        bits_equal(a[1][name], b[1][name], f"{what}: grad {name}")


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name", list(MODEL_BATCH))
def test_activation_checkpointing_changes_no_bit(name, fp8, monkeypatch):
    """activation_checkpoint="full" recomputes every block's forward in backward: the loss and every gradient must be
    those of "none", bit for bit. The "none" step is first run twice, so that a nondeterministic kernel cannot pass
    for (or hide) a difference the checkpoint makes; attention runs SDPA's flash kernels with deterministic algorithms
    on (see _deterministic_attention)."""
    cfg = _model_cfg(name, fp8_linears=fp8)
    tok, tgt = _batch(cfg, *MODEL_BATCH[name], seed=3)
    with _deterministic_attention(monkeypatch):
        ref = _step(cfg, tok, tgt)
        _equal_steps(_step(cfg, tok, tgt), ref, f"{name} fp8={fp8}: two runs")
        _equal_steps(_step(dataclasses.replace(cfg, activation_checkpoint="full"), tok, tgt), ref,
                     f"{name} fp8={fp8}: checkpointed")


@pytest.mark.parametrize("fp8", [False, True])
def test_activation_checkpointing_changes_no_bit_of_zero1_steps(fp8, monkeypatch):
    """Three FT-ZeRO-1 steps of llama3_debug with and without activation checkpointing: the same losses and the same
    parameter buffer, bit for bit. The "none" arm runs twice first; attention as in
    test_activation_checkpointing_changes_no_bit."""
    from _zero1_replicas import trainer

    cfg = _model_cfg("llama3_debug")
    g = torch.Generator().manual_seed(11)
    batches = [tuple(torch.randint(0, cfg.vocab_size, (2, 256), generator=g).pin_memory() for _ in range(2))
               for _ in range(3)]
    out = []
    with _deterministic_attention(monkeypatch):
        for i, ckpt in enumerate(("none", "none", "full")):
            with trainer("llama3_debug", f"ckpt_{i}_{int(fp8)}", seed=0, activation_checkpoint=ckpt, fp8_linears=fp8) as tr:
                assert tr.cfg.activation_checkpoint == ckpt
                losses = [tr.step(tok, tgt) for tok, tgt in batches]
                tr.join()
                torch.cuda.synchronize()
                out.append((losses, tr.state_dict()["param"].clone()))
    for i, what in ((1, "two runs"), (2, "checkpointed")):
        assert out[i][0] == out[0][0], (what, out[i][0], out[0][0])
        bits_equal(out[i][1], out[0][1], f"fp8={fp8}: {what}: parameter buffer after 3 steps")


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name", list(MODEL_BATCH))
def test_direct_weight_gradients_change_no_bit(name, fp8, monkeypatch):
    """FlatParams.reset_grads(zero=False), every slot pre-filled with NaN so producers must overwrite it all, against
    reset_grads(zero=True): after adopt_grad the whole flat gradient is identical, and the padding between parameters
    stays zero. The zeroed arm runs twice first; attention as in test_activation_checkpointing_changes_no_bit."""
    cfg = _model_cfg(name, fp8_linears=fp8)
    tok, tgt = _batch(cfg, *MODEL_BATCH[name], seed=4)
    grads = []
    with _deterministic_attention(monkeypatch):
        for zero in (True, True, False):
            grads.append(_flat_step(cfg, tok, tgt, zero))
    bits_equal(grads[1], grads[0], f"{name} fp8={fp8}: two zeroed runs")
    assert not bool(grads[2].isnan().any())
    bits_equal(grads[2], grads[0], f"{name} fp8={fp8}: direct vs zeroed flat gradient")


def _flat_step(cfg, tok, tgt, zero):
    """One step of a FlatParams model from reset_grads(zero); returns the flat gradient after adopt_grad."""
    from torchft_b200.models.llama import FlatParams, Llama

    m = Llama(cfg, device="meta")
    flat = FlatParams(m, device=torch.device("cuda"))
    m.init_weights(0)
    flat.grad.zero_()
    if not zero:
        for p in flat.params:
            p._flat_grad.fill_(float("nan"))
    flat.reset_grads(zero=zero)
    m(tok, tgt).backward()
    for p in flat.params:
        flat.adopt_grad(p)
    pad = torch.ones(flat.numel, dtype=torch.bool, device="cuda")
    for p, o in zip(flat.params, flat.offsets):
        pad[o:o + p.numel()] = False
    assert bool((flat.grad[pad] == 0).all()), f"zero={zero}: padding written"
    return flat.grad.clone()


# ------------------------------------------------------------------------------------------------------------ coverage
def test_every_case_ran():
    """Every node case above ran (run the whole module)."""
    want = set()
    for shape in SHAPES:
        for fp8 in (False, True):
            for flag in (False, True):
                for direct in (False, True):
                    want |= {(node, fp8, flag, direct, shape) for node in ("norm_linear", "swiglu_linear", "linear")}
    want |= {("rope", False, None, False, f"D={D} B={B} S={S}") for D in (64, 128) for B, S in ((1, 8192), (2, 4096))}
    missing = sorted(want - RAN, key=str)
    assert not missing, f"never ran: {missing}"
    print(f"[peak] max memory allocated {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
