"""fp64 references and error bounds of the fused Llama nodes (``ops/fused.py``), shared by the GPU tests and their CPU
emulations.

Every reference is built in fp64 from the bf16 values the node really used. A node hides one intermediate: the normalised
activation ``n`` of ``norm_linear_res`` and the SwiGLU product ``a`` of ``swiglu_linear``. The caller passes the one the
node multiplied (the kernel's own output on the GPU), and for fp8 the dequantised e4m3 operands of each fp8 GEMM. Each
``check_*`` holds every output and every input gradient of a node, element by element, to the bound derived next to it:

* bf16 GEMM with fp32 accumulation over K terms: ``ulps=1`` and ``K U (|A| @ |B|)``;
* rowwise fp8 GEMM: ``ulps=1`` and ``2^-12 (|A| @ |B|)`` on the dequantised operands (see ``test_fp8_gpu._gemm_slack``);
* a residual, in a bf16 GEMM's epilogue (``addmm``, beta = 1) or added to an fp8 GEMM's bf16 output: the product's
  rounding to bf16, ``2^-8 |mm|``, before the final ulp. On an H100 (torch 2.11, CUDA 12.8) a bf16 ``addmm(res, a, b)`` is
  bit for bit ``bf16(a @ b) + res`` at every Llama-3 1B and 8B shape: the epilogue saves a pass, not a rounding;
* an unobserved bf16 input gradient ``dn = bf16(dy @ W)`` (or ``da``) carries ``e <= slack + 2^-8 |dy @ W|``, pushed
  through the linear map of the RMSNorm or SwiGLU backward, plus that kernel's own slack (``test_model_ops_gpu``).

The row loops keep the fp64 temporaries at about ``2^24`` elements each, so the peak stays bounded at Llama-3 8B shapes.
"""

from __future__ import annotations

import math

import torch

from _fp64 import FTZ, U, _f32, assert_close_elementwise

CHUNK = 1 << 24  # fp64 elements per row chunk of a reference
FDIV_FLOOR = 126 * math.log(2) - 1e-3  # __fdividef's sigmoid is 0 below -FDIV_FLOOR (test_model_ops_gpu)


def chunks(rows, width):
    step = max(1, CHUNK // max(1, width))
    for lo in range(0, rows, step):
        yield slice(lo, min(rows, lo + step))


def bits_equal(a, b, what):
    """Bit for bit, with +0 and -0 counted equal (torch.equal)."""
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if not torch.equal(a, b):
        diff = (a != b) & ~(a.isnan() & b.isnan())
        idx = diff.nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, first at {idx}")


def rel_norm(a, b):
    """The whole-tensor check the fused nodes had before: ``|a - b| / |b|``."""
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------------------ GEMMs
def gemm(A, B, fp8, K=None):
    """``(A @ B, slack)`` of fp64 operands ``A [M, K]``, ``B [K, N]``: bf16 operands with fp32 accumulation over ``K`` terms
    (``K`` may name the whole reduction when ``A`` and ``B`` are one chunk of it), or dequantised e4m3 operands."""
    mm = A @ B
    absab = A.abs() @ B.abs()
    return mm, (2.0 ** -12 if fp8 else (K or A.shape[1]) * U) * absab


def with_res(mm, sl, res):
    """Reference and slack of ``bf16(bf16(mm) + res)``: the product rounded once before the residual is added."""
    if res is None:
        return mm, sl
    return mm + res, sl + 2.0 ** -8 * mm.abs()


def _d(t):
    return t.double()


def _bwd_dn(dy, Wd, fp8_bwd, sl):
    """``(dn, slack)``: the exact input-gradient GEMM ``dy @ W`` over rows ``sl`` and its GEMM slack."""
    if fp8_bwd is None:
        return gemm(_d(dy[sl]), Wd, False)
    return gemm(fp8_bwd[0][sl], fp8_bwd[1], True)


def check_wgrad(dW, dy, x, tag):
    """dW = dy^T @ x over all T rows (chunked): bf16 GEMM, K = T."""
    T = dy.shape[0]
    ref = torch.zeros(dy.shape[1], x.shape[1], dtype=torch.float64, device=dy.device)
    sl = torch.zeros_like(ref)
    for s in chunks(T, max(dy.shape[1], x.shape[1])):
        r, e = gemm(_d(dy[s]).t(), _d(x[s]), False, K=T)
        ref += r
        sl += e
    for s in chunks(dW.shape[0], dW.shape[1]):
        assert_close_elementwise(dW[s], ref[s], ulps=1, abs_slack=sl[s] + FTZ, what=f"{tag} dW")


def check_forward(y, A_rows, B, res, fp8, tag):
    """y [T, N] = A @ B (+ res), rows chunked; ``A_rows(sl)`` gives the fp64 rows of A."""
    T, N = y.shape
    for s in chunks(T, N):
        mm, sl = gemm(A_rows(s), B, fp8)
        ref, sl = with_res(mm, sl, None if res is None else _d(res[s]))
        assert_close_elementwise(y[s], ref, ulps=1, abs_slack=sl + FTZ, what=f"{tag} y")


# ----------------------------------------------------------------------------------------------------------- linear
def check_linear(tag, x, W, res, dy, got, fp8_fwd=None, fp8_bwd=None):
    """``linear(x, W, res)``: got = {y, dx, dW, dres}; x, res, dy and got are 2-D views ``[T, .]``."""
    Wd = _d(W)
    fp8 = fp8_fwd is not None
    check_forward(got["y"], lambda s: _d(x[s]) if not fp8 else fp8_fwd[0][s], Wd.t() if not fp8 else fp8_fwd[1], res, fp8,
                  tag)
    T, H = x.shape
    for s in chunks(T, max(H, W.shape[0])):
        dn, sl = _bwd_dn(dy, Wd, fp8_bwd, s)
        # dx IS the input-gradient GEMM's output: its own slack, then one rounding (1 ulp)
        assert_close_elementwise(got["dx"][s], dn, ulps=1, abs_slack=sl + FTZ, what=f"{tag} dx")
    check_wgrad(got["dW"], dy, x, tag)
    if res is not None:
        bits_equal(got["dres"], dy, f"{tag} dres")
    else:
        assert got["dres"] is None, tag


# -------------------------------------------------------------------------------------------------- norm_linear_res
def check_norm_linear(tag, x, g, W, dy, dres, eps, n, grid, got, fp8_fwd=None, fp8_bwd=None):
    """``norm_linear_res(x, g, W)``: got = {x_out, y, dx, dg, dW}. ``n`` is the bf16 normalised activation the node
    multiplied (forward for bf16, and the recompute its weight gradient reads); ``grid`` is ``rmsnorm_bwd_grid(T)``.

    dx = r (dn g - xh mean(dn g xh)) + dres is linear in dn: an error e of dn moves it by at most
    r (|e| |g| + |xh| mean(|e| |g| |xh|)). The kernel's own slack (test_model_ops_gpu._check_rmsnorm) is taken on
    |dn| + e, what it may have read. dg = sum over rows of dn xh: e moves it by sum |e| |xh|."""
    T, H = x.shape
    N = W.shape[0]
    bits_equal(got["x_out"], x, f"{tag} residual output")
    fp8 = fp8_fwd is not None
    Wd, gd = _d(W), _d(g)
    check_forward(got["y"], lambda s: _d(n[s]) if not fp8 else fp8_fwd[0][s], Wd.t() if not fp8 else fp8_fwd[1], None, fp8,
                  tag)
    dg_ref = torch.zeros(H, dtype=torch.float64, device=x.device)
    dg_err, dg_abs = torch.zeros_like(dg_ref), torch.zeros_like(dg_ref)
    for s in chunks(T, max(H, N)):
        xd = _d(x[s])
        r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + _f32(eps))
        xh = xd * r
        dn, e = _bwd_dn(dy, Wd, fp8_bwd, s)
        e = e + 2.0 ** -8 * dn.abs()  # the unobserved bf16 dn
        gw = dn * gd
        ref = r * (gw - xh * (gw * xh).mean(-1, keepdim=True))
        if dres is not None:
            ref = ref + _d(dres[s])
        eg = e * gd.abs()
        prop = r * (eg + xh.abs() * (eg * xh.abs()).mean(-1, keepdim=True))
        ga = (dn.abs() + e) * gd.abs()
        kern = 2.0 ** -16 * (r * ga + r * xh.abs() * (ga * xh.abs()).mean(-1, keepdim=True))
        assert_close_elementwise(got["dx"][s], ref, ulps=1, abs_slack=prop + kern + FTZ, what=f"{tag} dx")
        dg_ref += (dn * xh).sum(0)
        dg_err += (e * xh.abs()).sum(0)
        dg_abs += ((dn.abs() + e) * xh.abs()).sum(0)
        del xd, dn, e, gw, ref, eg, prop, ga, kern
    chain = math.ceil(T / max(1, min(T, 132))) + math.ceil(grid / 32) + 32
    assert_close_elementwise(got["dg"], dg_ref, ulps=1, abs_slack=dg_err + (chain + 36) * U * dg_abs + FTZ, what=f"{tag} dg")
    check_wgrad(got["dW"], dy, n, tag)


# ---------------------------------------------------------------------------------------------------- swiglu_linear
def swiglu_bwd_ref(gu, da, e):
    """dgu of the SwiGLU backward in fp64 from the exact ``da`` and its error bound ``e``: dg = da u (s + silu (1 - s)),
    du = da silu; e through that linear map, plus the kernel's own slack (test_model_ops_gpu._swiglu_ref) on |da| + e."""
    F = gu.shape[1] // 2
    gd, ud = _d(gu[:, :F]), _d(gu[:, F:])
    s = torch.sigmoid(gd)
    silu = gd * s
    over = (-gd >= FDIV_FLOOR).double()
    rel = (11 + 2.32 * gd.abs()) * U
    coef_g = ud.abs() * (s + silu.abs() * (1 - s))
    dg = da * ud * (s + silu * (1 - s))
    du = da * silu
    dmax = da.abs() + e
    sl_g = e * coef_g + (rel + 3 * U) * dmax * coef_g + over * (dg.abs() + e * coef_g) + FTZ
    sl_u = e * silu.abs() + rel * dmax * silu.abs() + over * dmax * silu.abs() + FTZ
    return torch.cat([dg, du], 1), torch.cat([sl_g, sl_u], 1)


def check_swiglu_linear(tag, gu, W2, res, dy, a, got, fp8_fwd=None, fp8_bwd=None):
    """``swiglu_linear(gu, W2, res)``: got = {y, dgu, dW, dres}. ``a`` is the bf16 SwiGLU product the node multiplied
    (forward for bf16, and the recompute its weight gradient reads)."""
    T = gu.shape[0]
    fp8 = fp8_fwd is not None
    Wd = _d(W2)
    check_forward(got["y"], lambda s: _d(a[s]) if not fp8 else fp8_fwd[0][s], Wd.t() if not fp8 else fp8_fwd[1], res, fp8,
                  tag)
    for s in chunks(T, max(gu.shape[1], W2.shape[0])):
        da, e = _bwd_dn(dy, Wd, fp8_bwd, s)
        e = e + 2.0 ** -8 * da.abs()  # the unobserved bf16 da
        ref, sl = swiglu_bwd_ref(gu[s], da, e)
        assert_close_elementwise(got["dgu"][s], ref, ulps=1, abs_slack=sl, what=f"{tag} dgu")
        del da, e, ref, sl
    check_wgrad(got["dW"], dy, a, tag)
    if res is not None:
        bits_equal(got["dres"], dy, f"{tag} dres")
    else:
        assert got["dres"] is None, tag


# -------------------------------------------------------------------------------------------------------- RoPE + qkv
def rotate(x, cs, sign):
    """x [n, H, D] rotated in fp64 by the fp32 table rows cs [n, D/2, 2] the kernel reads (sign -1: the inverse). The
    kernel rotates in fp32: two roundings of terms <= |x0| + |x1| (2 U), then one to bf16 (1 ulp)."""
    xd = _d(x).unflatten(-1, (-1, 2))
    c, s = _d(cs)[:, None, :, 0], sign * _d(cs)[:, None, :, 1]
    x0, x1 = xd[..., 0], xd[..., 1]
    out = torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), -1).flatten(-2)
    sl = 2 * U * (x0.abs() + x1.abs())
    return out, torch.stack((sl, sl), -1).flatten(-2) + FTZ


def check_rope(tag, qkv, cs, B, S, Hq, Hkv, D, q, k, v, dq, dk, dv, dqkv):
    """rope_qkv forward (q, k rotated; v the projection's slice) and backward (dqkv: dq, dk rotated back; dv copied)."""
    row = (Hq + 2 * Hkv) * D
    assert dqkv.shape == (B * S, row)
    pk = qkv.view(B, S, Hq + 2 * Hkv, D)
    gp = dqkv.view(B, S, Hq + 2 * Hkv, D)
    bits_equal(v, pk[:, :, Hq + Hkv:], f"{tag} v")
    bits_equal(gp[:, :, Hq + Hkv:], dv, f"{tag} dv")
    for b in range(B):
        for s in chunks(S, 4 * row):
            c = cs[s]
            for name, got, x, sign in (("q", q[b, s], pk[b, s, :Hq], 1.0), ("k", k[b, s], pk[b, s, Hq:Hq + Hkv], 1.0),
                                       ("dq", gp[b, s, :Hq], dq[b, s], -1.0), ("dk", gp[b, s, Hq:Hq + Hkv], dk[b, s], -1.0)):
                ref, sl = rotate(x, c, sign)
                assert_close_elementwise(got, ref, ulps=1, abs_slack=sl, what=f"{tag} {name}")


# --------------------------------------------------------------------------------------------------------- the model
def _fake_e4m3_rows(x):
    """x rounded to the row-scaled e4m3 operand the fp8 kernels make of it (``_fp8_ref``), back in x's dtype: scale
    ``2^e`` from the row's amax, each element RN to e4m3 at that scale. Finite rows only, inputs above 2^-126."""
    from _fp8_ref import exponent

    x = x.detach()
    e = exponent(x.abs().amax(-1, keepdim=True).float()).float()
    return (x.float() * torch.exp2(-e)).to(torch.float8_e4m3fn).to(x.dtype) * torch.exp2(e).to(x.dtype)


class _FP8Linear(torch.autograd.Function):
    """``x @ W^T`` on the operands the fp8 block linears use: forward x per row and W per output channel, input gradient
    dy per row and W per input channel, the weight gradient on the unquantised x and dy."""

    @staticmethod
    def forward(ctx, x, W):  # type: ignore[override]
        ctx.save_for_backward(x, W)
        return _fake_e4m3_rows(x) @ _fake_e4m3_rows(W).t()

    @staticmethod
    def backward(ctx, dy):  # type: ignore[override]
        x, W = ctx.saved_tensors
        dx = _fake_e4m3_rows(dy) @ _fake_e4m3_rows(W.t()).t()
        dW = dy.reshape(-1, dy.shape[-1]).t() @ x.reshape(-1, x.shape[-1])
        return dx, dW


def fp8_linear(x, W):
    """The block linear of ``models.reference.reference_loss`` with the model's e4m3 operand quantisation."""
    return _FP8Linear.apply(x, W)


def row_ratios(g, r64, b16, factor):
    """Per row ``|g - r64| / (factor |b16 - r64| + 2^-9 |r64|)`` of a parameter gradient, and the row relative errors
    ``|g - r64| / |r64|`` and ``|b16 - r64| / |r64|``. Rows: the rows of a matrix, the 8-element vectors of a norm weight.
    A row where every side is 0 has ratio 0."""
    def rows(t):
        t = t.double()
        return t.reshape(-1, t.shape[-1]) if t.dim() >= 2 else t.reshape(-1, 8)

    G, R, Bb = rows(g), rows(r64.to(g.device)), rows(b16.to(g.device))
    eg, eb, rn = (G - R).norm(dim=1), (Bb - R).norm(dim=1), R.norm(dim=1)
    ratio = torch.where(eg == 0, 0.0, eg / (factor * eb + 2.0 ** -9 * rn))
    live = rn > 0
    return ratio, eg[live] / rn[live], eb[live] / rn[live]
