"""The fp8 block linears on the GPU: the quantisation kernels byte for byte against the CPU model (tests/_fp8_ref.py), the
fused RMSNorm / SwiGLU instances against the bf16 kernels followed by fp8_rows, the rowwise fp8 GEMMs element by element
against fp64 with a derived bound, the three autograd nodes, the model and the trainer."""

import math

import pytest
import torch

from _fp64 import _report_margins, assert_close_elementwise  # noqa: F401
from _fp8_ref import dequantize, quantize_cols_t, quantize_rows

gpu = pytest.mark.gpu
pytestmark = gpu
BF16 = torch.bfloat16
T = 8192
RAN = set()  # (kernel, NV, TPB) of every launch below, for test_every_kernel_instance_ran


def _K():
    from torchft_b200.ops import _native

    return _native.load()


def _sp():
    from torchft_b200.ops import _native

    return _native.stream_ptr()


def _shape(C):
    return tuple(_K().fp8_rows_shape(C))


def _rms_shape(H):
    # the RMSNorm forward table (model_ops.cu rms_shape): 128 threads doubling until 4 vectors of 8 per thread cover H
    v = 1
    while v * 128 < H // 8:
        v *= 2
    nv = min(v, 4)
    return nv, 128 * v // nv


def fp8_rows(x):
    from torchft_b200.ops import fused

    RAN.add(("rows",) + _shape(x.shape[1]))
    return fused.fp8_rows(x)


def _same(q, s, ref, what):
    rq, rs = ref
    got = q.view(torch.uint8).cpu()
    bad = (got != rq).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.shape[0]} bytes differ, first at {tuple(bad[0].tolist())}: " \
                             f"{int(got[tuple(bad[0])])} != {int(rq[tuple(bad[0])])}"
    s = s.reshape(-1).cpu()
    assert torch.equal(s.isnan(), rs.isnan()), what
    ok = ~rs.isnan()
    assert torch.equal(s[ok], rs[ok]), what


def _llama_shapes(name):
    from torchft_b200.models.llama import CONFIGS

    c = CONFIGS[name]
    qkv = (c.n_heads + 2 * c.n_kv_heads) * c.head_dim
    return c, {"wqkv": (qkv, c.dim), "wo": (c.dim, c.dim), "w13": (2 * c.ffn_dim, c.dim), "w2": (c.dim, c.ffn_dim)}


# ------------------------------------------------------------------------------------------------------- fp8_rows
def _act_grad_widths(name):
    """Row lengths of every linear input (activation) and grad-output of a model: K and N of its four weights."""
    _, w = _llama_shapes(name)
    return sorted({d for shape in w.values() for d in shape})


@pytest.mark.parametrize("name", ["llama3_1b", "llama3_8b"])
def test_fp8_rows_matches_the_model_at_every_llama_activation_and_gradient_width(name):
    gen = torch.Generator(device="cuda").manual_seed(1)
    for C in _act_grad_widths(name):
        x = (torch.randn(T, C, device="cuda", generator=gen) * 0.3).to(BF16)
        q, s = fp8_rows(x)
        _same(q, s, quantize_rows(x), f"{name} C={C}")
        del x, q, s


@pytest.mark.parametrize("R", [1, 3, 8191])
@pytest.mark.parametrize("C", [16, 2048, 4096 + 16, 28672])
def test_fp8_rows_row_counts_and_scales_from_1e_30_to_1e30(R, C):
    gen = torch.Generator(device="cuda").manual_seed(R + C)
    scales = torch.logspace(-30, 30, R, device="cuda", dtype=torch.float64) if R > 1 else torch.ones(1, device="cuda")
    x = (torch.randn(R, C, device="cuda", generator=gen) * scales[:, None].float()).to(BF16)
    q, s = fp8_rows(x)
    _same(q, s, quantize_rows(x), f"R={R} C={C}")


def test_fp8_rows_reads_a_strided_view():
    gen = torch.Generator(device="cuda").manual_seed(3)
    big = torch.randn(513, 3072 + 64, device="cuda", generator=gen).to(BF16)
    x = big[:, 32:32 + 3072]  # row stride 3136 elements, 16-byte aligned
    q, s = fp8_rows(x)
    _same(q, s, quantize_rows(x), "strided")


def test_fp8_rows_special_rows():
    C = 1024
    gen = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(8, C, device="cuda", generator=gen).to(BF16)
    x[0] = 0.0
    x[1] = -0.0
    x[2] = (torch.randn(C, device="cuda", generator=gen) * 2.0 ** -130).to(BF16)  # bf16 subnormals
    x[3, 100] = float("inf")
    x[4, 5] = float("-inf")
    x[5, 1000] = float("nan")
    x[6, :512] = (torch.randn(512, device="cuda", generator=gen) * 2.0 ** -130).to(BF16)  # subnormals beside normals
    q, s = fp8_rows(x)
    _same(q, s, quantize_rows(x), "special rows")
    assert math.isnan(s[3]) and math.isnan(s[4]) and math.isnan(s[5]) and not math.isnan(s[6])
    assert bool((q[3:6].view(torch.uint8) == 0x7F).all())


def test_fp8_rows_refuses_bad_widths_and_misaligned_rows():
    K = _K()
    buf = torch.zeros(4, 64 + 16, device="cuda", dtype=BF16)
    q = torch.empty(4 * 80, device="cuda", dtype=torch.uint8)
    s = torch.empty(4, device="cuda")
    for C in (24, 8, 0, 40000):
        with pytest.raises(RuntimeError, match="multiple of 16"):
            K.fp8_rows(buf.data_ptr(), 80, q.data_ptr(), s.data_ptr(), 4, C, _sp())
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.fp8_rows(buf.data_ptr() + 2, 80, q.data_ptr(), s.data_ptr(), 4, 64, _sp())
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.fp8_rows(buf.data_ptr(), 68, q.data_ptr(), s.data_ptr(), 4, 64, _sp())
    from torchft_b200.ops import fused

    with pytest.raises(ValueError, match="aligned"):
        fused.fp8_rows(buf.view(-1)[1:65].view(1, 64))
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------- fp8_cols_t
@pytest.mark.parametrize("name", ["llama3_tiny", "llama3_debug", "llama3_1b", "llama3_8b"])
def test_fp8_cols_t_matches_the_model_for_every_weight(name):
    from torchft_b200.ops import fused

    _, shapes = _llama_shapes(name)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for wname, (N, Kd) in shapes.items():
        W = (torch.randn(N, Kd, device="cuda", generator=gen) * 0.02).to(BF16)
        W[:, 1] = 0.0  # a column of zeros
        W[N // 3, Kd - 2] = float("inf")  # a column holding one inf
        q, s = fused.fp8_cols_t(W)
        assert q.shape == (Kd, N) and s.shape == (1, Kd)
        _same(q, s, quantize_cols_t(W), f"{name}.{wname}")
        assert float(s[0, 1]) == 2.0 ** -126 and math.isnan(float(s[0, Kd - 2]))
        del W, q, s


# ------------------------------------------------------------------------------------------------ fused instances
@pytest.mark.parametrize("H", [16, 1040, 2048, 4096, 6144, 16384])
def test_fused_rmsnorm_bytes_equal_fp8_rows_of_rmsnorm_and_rstd_is_bit_identical(H):
    K = _K()
    rows = 1031
    gen = torch.Generator(device="cuda").manual_seed(H)
    x = (torch.randn(rows, H, device="cuda", generator=gen) * 3).to(BF16)
    x[7] = 0.0
    x[9, 3] = float("inf")
    w = (torch.randn(H, device="cuda", generator=gen) * 0.5 + 1).to(BF16)
    y = torch.empty_like(x)
    r0 = torch.empty(rows, device="cuda")
    K.rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), r0.data_ptr(), rows, H, 1e-5, _sp())
    q = torch.empty(rows, H, device="cuda", dtype=torch.uint8)
    s = torch.empty(rows, device="cuda")
    r1 = torch.empty(rows, device="cuda")
    K.rmsnorm_fwd_fp8(x.data_ptr(), w.data_ptr(), q.data_ptr(), s.data_ptr(), r1.data_ptr(), rows, H, 1e-5, _sp())
    RAN.add(("rmsnorm",) + _rms_shape(H))
    qr, sr = fp8_rows(y)
    assert torch.equal(q, qr.view(torch.uint8)), H
    assert torch.equal(s.isnan(), sr.view(-1).isnan()) and torch.equal(s[~s.isnan()], sr.view(-1)[~s.isnan()])
    assert torch.equal(r0.view(torch.int32), r1.view(torch.int32))


@pytest.mark.parametrize("F", [192, 768, 4096, 8192, 14336, 20480])
def test_fused_swiglu_bytes_equal_fp8_rows_of_swiglu(F):
    K = _K()
    Tn = 777
    gen = torch.Generator(device="cuda").manual_seed(F)
    gu = (torch.randn(Tn, 2 * F, device="cuda", generator=gen) * 2).to(BF16)
    gu[5, 10] = float("nan")
    a = torch.empty(Tn, F, device="cuda", dtype=BF16)
    K.swiglu_fwd(gu.data_ptr(), a.data_ptr(), Tn, F, _sp())
    q = torch.empty(Tn, F, device="cuda", dtype=torch.uint8)
    s = torch.empty(Tn, device="cuda")
    K.fp8_swiglu(gu.data_ptr(), q.data_ptr(), s.data_ptr(), Tn, F, _sp())
    RAN.add(("swiglu",) + _shape(F))
    qr, sr = fp8_rows(a)
    assert torch.equal(q, qr.view(torch.uint8)), F
    assert torch.equal(s.isnan(), sr.view(-1).isnan()) and torch.equal(s[~s.isnan()], sr.view(-1)[~s.isnan()])
    assert math.isnan(float(s[5]))


# ------------------------------------------------------------------------------------------------- GEMM numerics
# Bound of one output element of a rowwise fp8 GEMM against the fp64 product of the dequantised operands. The products of
# e4m3 values are exact and the scales are powers of two, so only the accumulation and the output rounding err:
#   * Hopper's fp8 MMA adds products in a fixed-point accumulator that keeps about 14 bits (DeepSeek-V3 technical report,
#     section 3.3.2); with use_fast_accum=False the library promotes that partial sum into an fp32 accumulator at least
#     every 128 products of K. We take 13 bits of the interval's magnitude, so an interval's partial sum errs by at most
#     2^-13 * sum |a_k b_k| over the interval, and twice that for the promotion into fp32 and its 2^-24 roundings: in all
#     2^-12 * sum_k |a_k b_k| over the whole row-column pair;
#   * rounding the fp32 result to bf16: half a bf16 ulp of the computed value, at most one ulp of the exact one.
# A scale off by one exponent changes an element by |ref| itself, about sqrt(K) / (2^-12 K) times this slack.
def _gemm_slack(A, B):
    """2^-12 * (|A| @ |B|) for fp64 operands A [M, K] and B [K, N]."""
    return 2.0 ** -12 * (A.abs() @ B.abs())


def _check_gemm(got, A, B, what):
    assert_close_elementwise(got.cpu(), A @ B, ulps=1, abs_slack=_gemm_slack(A, B), what=what)


@pytest.mark.parametrize("M,N,Kd", [(256, 384, 2048), (128, 512, 4096), (64, 256, 14336)])
def test_forward_and_input_gradient_gemms_against_fp64(M, N, Kd):
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(M + N + Kd)
    x = torch.randn(M, Kd, device="cuda", generator=gen).to(BF16)
    W = (torch.randn(N, Kd, device="cuda", generator=gen) * 0.02).to(BF16)
    dy = (torch.randn(M, N, device="cuda", generator=gen) * 1e-3).to(BF16)
    # forward: x @ W^T
    qa, sa = fp8_rows(x)
    qw, sw = fp8_rows(W)
    y = fused._fwd_fp8((qa, sa), W)
    A, B = dequantize(qa, sa), dequantize(qw, sw).t()
    _check_gemm(y, A, B, f"fp8 forward {M}x{N}x{Kd}")
    # input gradient: dy @ W
    qd, sd = fp8_rows(dy)
    qt, st = fused.fp8_cols_t(W)
    dx = fused._dgrad_fp8(dy, W)
    A, B = dequantize(qd, sd), dequantize(qt, st).t()
    _check_gemm(dx, A, B, f"fp8 input gradient {M}x{N}x{Kd}")


def test_a_scale_off_by_one_exponent_fails_the_bound():
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(64, 4096, device="cuda", generator=gen).to(BF16)
    W = (torch.randn(256, 4096, device="cuda", generator=gen) * 0.02).to(BF16)
    qa, sa = fp8_rows(x)
    qw, sw = fp8_rows(W)
    bad = sa.clone()
    bad[17] *= 2  # one row's exponent off by one
    y = fused._mm_fp8((qa, bad), (qw.t(), sw.view(1, -1)))
    with pytest.raises(AssertionError):
        _check_gemm(y, dequantize(qa, sa), dequantize(qw, sw).t(), "mutant")


# ------------------------------------------------------------------------------------------------------ the nodes
# dx of an fp8 node against the bf16 node: the e4m3 operands differ from the bf16 ones by at most 2^-4 relative (half an
# ulp of a 3-bit mantissa) plus, below 2^-6 * scale, half the subnormal spacing 2^-10 * scale; so each product differs by
# at most (2^-4 + 2^-4 + 2^-8) |a||b| plus the subnormal terms, and the GEMM slack of each side adds 2^-12 |a||b|.
# We bound the whole by 2^-3 * (|dy| @ |W|) + the subnormal terms + one bf16 ulp of each GEMM's output.
def _dgrad_bound(dy, W):
    sd = quantize_rows(dy)[1].double().reshape(-1, 1)
    sw = quantize_cols_t(W)[1].double().reshape(1, -1)
    a, b = dy.double().cpu().abs(), W.double().cpu().abs()
    sub = 2.0 ** -10 * (sd * b.sum(0, keepdim=True) + a.sum(1, keepdim=True) * sw)
    exact = dy.double().cpu() @ W.double().cpu()
    return 2.0 ** -3 * (a @ b) + sub + 2 * 2.0 ** -8 * exact.abs()


def _node_grads(fn, inputs, dout, fp8):
    xs = [t.detach().clone().requires_grad_(t.requires_grad) for t in inputs]
    for t in xs:
        t.grad = None
    out = fn(*xs, fp8=fp8)
    outs = out if isinstance(out, tuple) else (out,)
    torch.autograd.backward(outs, dout)
    return [t.grad for t in xs]


def test_linear_node_fp8_keeps_dw_bit_identical_and_dx_within_the_fp8_bound():
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(11)
    M, d = 1024, 2048
    x = torch.randn(4, M // 4, d, device="cuda", generator=gen).to(BF16).requires_grad_()
    W = (torch.randn(d, d, device="cuda", generator=gen) * 0.02).to(BF16).requires_grad_()
    res = torch.randn(4, M // 4, d, device="cuda", generator=gen).to(BF16).requires_grad_()
    dy = (torch.randn(4, M // 4, d, device="cuda", generator=gen) * 1e-2).to(BF16)
    g0 = _node_grads(lambda a, b, c, fp8: fused.linear(a, b, res=c, fp8=fp8), (x, W, res), (dy,), False)
    g1 = _node_grads(lambda a, b, c, fp8: fused.linear(a, b, res=c, fp8=fp8), (x, W, res), (dy,), True)
    assert torch.equal(g0[1].view(torch.int16), g1[1].view(torch.int16)), "dW must be the same bf16 GEMM"
    assert torch.equal(g0[2], g1[2])
    bound = _dgrad_bound(dy.view(M, d), W.detach())
    err = (g1[0].view(M, d).double().cpu() - g0[0].view(M, d).double().cpu()).abs()
    assert bool((err <= bound).all()), float((err / bound).max())


def test_norm_linear_node_fp8_keeps_dw_bit_identical_and_dx_within_the_fp8_bound():
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(12)
    M, d, N = 1024, 2048, 3072
    x = torch.randn(M, d, device="cuda", generator=gen).to(BF16).requires_grad_()
    g = (torch.randn(d, device="cuda", generator=gen) * 0.1 + 1).to(BF16).requires_grad_()
    W = (torch.randn(N, d, device="cuda", generator=gen) * 0.02).to(BF16).requires_grad_()
    dres = (torch.randn(M, d, device="cuda", generator=gen) * 1e-2).to(BF16)
    dy = (torch.randn(M, N, device="cuda", generator=gen) * 1e-2).to(BF16)
    fn = lambda a, b, c, fp8: fused.norm_linear_res(a, b, c, 1e-5, fp8=fp8)  # noqa: E731
    g0 = _node_grads(fn, (x, g, W), (dres, dy), False)
    g1 = _node_grads(fn, (x, g, W), (dres, dy), True)
    assert torch.equal(g0[2].view(torch.int16), g1[2].view(torch.int16)), "dW must be the same bf16 GEMM"
    # dx = r * (dn * g - xhat * mean(dn * g * xhat)) + dres is linear in dn: an error e in dn moves dx by at most
    # r * (|e| |g| + |xhat| mean(|e| |g| |xhat|)), plus a bf16 rounding of dx on each side
    xd = x.detach().double().cpu()
    r = (xd.pow(2).mean(1, keepdim=True) + 1e-5).rsqrt()
    xh, gd = xd * r, g.detach().double().cpu().abs()
    e = _dgrad_bound(dy, W.detach())
    bound = r * (e * gd + xh.abs() * (e * gd * xh.abs()).mean(1, keepdim=True))
    d0, d1 = g0[0].double().cpu(), g1[0].double().cpu()
    bound = bound + 2.0 ** -8 * (d0.abs() + d1.abs()) + 1e-30
    assert bool(((d1 - d0).abs() <= bound).all()), float(((d1 - d0).abs() / bound).max())


def test_swiglu_linear_node_fp8_keeps_dw_bit_identical_and_dx_within_the_fp8_bound():
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(13)
    M, F, d = 1024, 2048, 1024
    gu = torch.randn(M, 2 * F, device="cuda", generator=gen).to(BF16).requires_grad_()
    W2 = (torch.randn(d, F, device="cuda", generator=gen) * 0.02).to(BF16).requires_grad_()
    res = torch.randn(M, d, device="cuda", generator=gen).to(BF16).requires_grad_()
    dy = (torch.randn(M, d, device="cuda", generator=gen) * 1e-2).to(BF16)
    fn = lambda a, b, c, fp8: fused.swiglu_linear(a, b, res=c, fp8=fp8)  # noqa: E731
    g0 = _node_grads(fn, (gu, W2, res), (dy,), False)
    g1 = _node_grads(fn, (gu, W2, res), (dy,), True)
    assert torch.equal(g0[1].view(torch.int16), g1[1].view(torch.int16)), "dW must be the same bf16 GEMM"
    assert torch.equal(g0[2], g1[2])
    # dgu is linear in da: dg = da * u * (s + silu (1 - s)), du = da * silu
    gd, ud = gu.detach().double().cpu()[:, :F], gu.detach().double().cpu()[:, F:]
    s = torch.sigmoid(gd)
    e = _dgrad_bound(dy, W2.detach())
    coef = torch.cat([(ud * (s + gd * s * (1 - s))).abs(), (gd * s).abs()], 1)
    d0, d1 = g0[0].double().cpu(), g1[0].double().cpu()
    bound = torch.cat([e, e], 1) * coef * (1 + 2.0 ** -6) + 2.0 ** -8 * (d0.abs() + d1.abs()) + 1e-30
    assert bool(((d1 - d0).abs() <= bound).all()), float(((d1 - d0).abs() / bound).max())


# ------------------------------------------------------------------------------------------------------ the model
def test_llama_debug_with_fp8_linears_follows_the_fp32_reference():
    """llama3_debug at B=2, S=512 with fp8 block linears against the fp32 eager reference. The bf16 model is within
    2^-8 of its loss and 2 % of every gradient norm (test_model_ops_gpu). e4m3 carries 3 mantissa bits: one quantisation
    errs by up to 2^-4 relative, independently per element, so a GEMM output over K terms errs by about 2^-4 / sqrt(3)
    of its size (uniform rounding error), ~4 %, and the loss by far less since it averages thousands of tokens: we ask
    for 2^-6 on the loss, and a cosine similarity above 0.99 for every gradient (an error of 4 % in norm gives 0.9992;
    a gradient with the wrong sign or a missing term gives far less)."""
    from torchft_b200.models.llama import CONFIGS, Llama
    from torchft_b200.models.reference import reference_loss
    import dataclasses

    cfg = dataclasses.replace(CONFIGS["llama3_debug"], fp8_linears=True)
    gen = torch.Generator(device="cuda").manual_seed(17)
    m = Llama(cfg, device="cuda")
    m.init_weights(0)
    tok = torch.randint(0, cfg.vocab_size, (2, 512), device="cuda", generator=gen)
    tgt = torch.randint(0, cfg.vocab_size, (2, 512), device="cuda", generator=gen)
    loss = m(tok, tgt)
    loss.backward()
    ref_loss, ref_grads = reference_loss(m, tok, tgt)
    assert abs(loss.item() - ref_loss) <= 2.0 ** -6 * abs(ref_loss), (loss.item(), ref_loss)
    for name, p in m.named_parameters():
        cos = float(torch.nn.functional.cosine_similarity(p.grad.double().flatten(), ref_grads[name].double().flatten(), 0))
        print(f"[model fp8] {name}: cos {cos:.6f}")
        assert cos > 0.99, (name, cos)


# ---------------------------------------------------------------------------------------------------- the trainer
def _stream(vocab, steps, B, S, seed):
    """A learnable token stream: each sequence walks a fixed random permutation of a 64-token subset from a random start,
    so the next token is a function of the current one; targets are the inputs shifted by one."""
    g = torch.Generator().manual_seed(seed)
    sub = torch.randperm(vocab, generator=g)[:64]
    nxt = torch.randperm(64, generator=g)
    out = []
    for _ in range(steps):
        idx = torch.randint(0, 64, (B,), generator=g)
        seq = torch.empty(B, S + 1, dtype=torch.long)
        for t in range(S + 1):
            seq[:, t] = sub[idx]
            idx = nxt[idx]
        out.append((seq[:, :-1].contiguous().pin_memory(), seq[:, 1:].contiguous().pin_memory()))
    return out


def _train(tag, fp8, seed, steps=50):
    from _zero1_replicas import trainer

    with trainer("llama3_debug", tag, lr=3e-3, seed=seed, fp8_linears=fp8) as tr:
        assert tr.cfg.fp8_linears == fp8
        losses = [tr.step(tok, tgt) for tok, tgt in _stream(tr.cfg.vocab_size, steps, 4, 128, 99)]
        tr.join()
        torch.cuda.synchronize()
        sd = {k: (tuple(v.shape), v.dtype) if torch.is_tensor(v) else type(v) for k, v in tr.state_dict().items()}
        return losses, sd


def test_trainer_learns_with_fp8_linears_like_with_bf16():
    """50 FT-ZeRO-1 steps on a learnable stream. The final losses of fp8 and bf16 must agree within 4x the gap between
    two bf16 runs whose initial weights differ (seeds 0 and 1), plus 0.05 nats: that gap is what the run-to-run
    variation of the initialisation alone produces, and fp8 should look like another draw of it."""
    l8, sd8 = _train("fp8_on", True, 0)
    l0, sd0 = _train("fp8_off", False, 0)
    l1, _ = _train("fp8_off2", False, 1)
    print(f"[trainer] fp8 {l8[0]:.4f} -> {l8[-1]:.4f}; bf16 {l0[0]:.4f} -> {l0[-1]:.4f}; bf16 seed 1 -> {l1[-1]:.4f}")
    for ls in (l8, l0, l1):
        assert all(math.isfinite(x) for x in ls)
        assert ls[-1] <= 0.5 * ls[0], (ls[0], ls[-1])
    assert abs(l8[-1] - l0[-1]) <= 4 * abs(l1[-1] - l0[-1]) + 0.05, (l8[-1], l0[-1], l1[-1])
    assert sd8 == sd0, "fp8 linears add no state"


def test_trainer_reads_the_fp8_switch_from_the_environment(monkeypatch):
    from torchft_b200.parallel.trainer import fp8_linears_from_env

    monkeypatch.delenv("TORCHFT_B200_FP8", raising=False)
    assert fp8_linears_from_env() is False and fp8_linears_from_env(True) is True
    monkeypatch.setenv("TORCHFT_B200_FP8", "0")
    assert fp8_linears_from_env(True) is False
    monkeypatch.setenv("TORCHFT_B200_FP8", "1")
    assert fp8_linears_from_env() is True
    from _zero1_replicas import trainer

    with trainer("llama3_tiny", "fp8_env") as tr:
        assert tr.cfg.fp8_linears and all(b.cfg.fp8_linears for b in tr.model.layers)
    for v in ("yes", "true", "2", ""):
        monkeypatch.setenv("TORCHFT_B200_FP8", v)
        with pytest.raises(ValueError, match="TORCHFT_B200_FP8"):
            fp8_linears_from_env()


def test_a_nonfinite_activation_row_vetoes_the_step(monkeypatch):
    """With max_grad_norm=inf one inf in one token row of wo's input becomes a NaN row of the e4m3 operand, the GEMM output
    row is NaN, so is the gradient norm, and the device commit skips the step: the weights do not move."""
    from _zero1_replicas import trainer
    from torchft_b200.ops import fused

    with trainer("llama3_debug", "fp8_veto", max_grad_norm=float("inf"), fp8_linears=True) as tr:
        steps = _stream(tr.cfg.vocab_size, 3, 2, 128, 7)
        tr.step(*steps[0])
        tr.join()
        torch.cuda.synchronize()
        before = tr.state_dict()["param"].clone()
        real = fused.linear

        def poisoned(x, W, res=None, fp8=False):
            x = x.clone()
            x.view(-1, x.shape[-1])[5, 7] = float("inf")
            return real(x, W, res=res, fp8=fp8)

        monkeypatch.setattr(fused, "linear", poisoned)
        tr.step(*steps[1])
        monkeypatch.setattr(fused, "linear", real)
        tr.join()
        torch.cuda.synchronize()
        assert torch.equal(before, tr.state_dict()["param"]), "the poisoned step must not update the weights"
        tr.step(*steps[2])
        tr.join()
        tr.manager.state_dict()  # settles the last verdict
        assert tr.zopt.nonfinite_steps == 1 and tr.zopt.t == 2, (tr.zopt.nonfinite_steps, tr.zopt.t)


# ------------------------------------------------------------------------------------------------------ coverage
def test_every_kernel_instance_ran():
    """Every (chunks, threads) instance the fp8 row launchers can pick and every RMSNorm forward instance of the fp8
    output ran above (run the whole module)."""
    shapes = {(1, 128), (2, 128), (4, 128), (4, 256), (4, 512)}
    want = {(k,) + s for k in ("rows", "swiglu", "rmsnorm") for s in shapes}
    missing = sorted(want - RAN)
    assert not missing, f"never launched: {missing}"
