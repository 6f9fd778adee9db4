"""The model kernels (``csrc/kernels/model_ops.cu``) element by element against float64, at Llama-3 shapes.

Every reference is computed in float64 from the same rounded inputs the kernel saw, and every check is per element:
``|got - ref| <= ulps * ulp_out(ref) + abs_slack``. ``ulp_out`` is the spacing of the output dtype at ``|ref|``;
``abs_slack`` is an elementwise bound, derived next to each reference, on an error the kernel is allowed to make: fp32
accumulation, cancellation, or an approximation of ``--use_fast_math`` (FTZ, ``__expf``, ``__fdividef``, approximate
``sqrtf``/``rsqrtf``). A whole-tensor norm passes while one vector, one tail or one CTA's rows are wrong, so it is never
the check. Shapes: llama3_1b (H=2048, F=8192, Hq=32, Hkv=8, D=64), llama3_8b (H=4096, F=14336, D=128), V=128256,
T=B*S=8192, theta=5e5.
"""

import math

import pytest
import torch

from _fp64 import _WORST, FTZ, U, _adamw_ref, _f32, _report_margins, assert_close_elementwise  # noqa: F401

gpu = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-12)).item()


# ------------------------------------------------------------------ the checker itself (CPU)
def test_elementwise_checker_flags_what_a_tensor_norm_misses():
    gen = torch.Generator().manual_seed(0)
    ref = torch.randn(8192, 2048, generator=gen).double()  # fp32 values: the cast to bf16 rounds once
    good = ref.to(torch.bfloat16)
    assert_close_elementwise(good, ref, ulps=0.5, what="checker round-to-nearest")  # RN is within half an ulp
    one = good.clone()
    one.view(torch.int16)[4097, 1001] += 2  # one element 2 ulp larger in magnitude
    vec = good.clone()
    vec.view(torch.int16)[123, 8 * 77 : 8 * 78] += 2  # one 16-byte vector of 8 elements, 2 ulp each
    row = good.clone()
    row[8000] = (ref[8000] * (1 + 2.0 ** -6)).to(torch.bfloat16)  # one row off by 2^-6 relative (>= 1.5 ulp)
    for name, bad in (("element", one), ("vector", vec), ("row", row)):
        assert _rel(bad, ref) < 1e-2, name  # the whole-tensor check used so far accepts it
        with pytest.raises(AssertionError, match="worst element"):
            assert_close_elementwise(bad, ref, ulps=1, what=f"checker {name}")
    _WORST.clear()


# ------------------------------------------------------------------ fixtures / helpers
@pytest.fixture(scope="module")
def K():
    from torchft_b200.ops import _native

    return _native.load()


def _sp():
    from torchft_b200.ops import _native

    return _native.stream_ptr()


def _rows_with_scales(rows, H, gen, scales=(1.0, 1e3, 1e-3, 0.0)):
    x = torch.randn(rows, H, device="cuda", generator=gen)
    s = torch.tensor(scales, device="cuda")[torch.arange(rows, device="cuda") % len(scales)]
    return (x * s[:, None]).bfloat16()


# ------------------------------------------------------------------ RMSNorm
# rstd: the fp32 sum of H squares runs along a chain of <= 53 adds (32 per thread, 5 shuffle levels, 16 warp partials)
# -> 53 U; the fast-math division by H adds 2 ulp (4 U) and + eps U; the square root halves all that, and rsqrtf adds
# 2 ulp (4 U): (53 + 4 + 1) / 2 + 4 = 33 U, rounded up to 34 U for the reference's own rounding.
R_RSTD = 34 * U


def _check_rmsnorm(K, x, w, dy, dres, eps, tag, y, rstd, dx, dw):
    rows, H = x.shape
    wd = w.double()
    dw_ref = torch.zeros(H, dtype=torch.float64, device="cuda")
    dw_abs = torch.zeros_like(dw_ref)
    for lo in range(0, rows, max(1, (1 << 24) // H)):
        hi = min(rows, lo + max(1, (1 << 24) // H))
        xd, dyd = x[lo:hi].double(), dy[lo:hi].double()
        r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + _f32(eps))
        xh = xd * r
        assert_close_elementwise(rstd[lo:hi], r[:, 0], ulps=0, abs_slack=R_RSTD * r[:, 0], what=f"rmsnorm rstd {tag}")
        # y = bf16((x * r) * w): within R_RSTD + 2U of exact before the one rounding to bf16 -> 1 ulp
        assert_close_elementwise(y[lo:hi], xh * wd, ulps=1, abs_slack=(R_RSTD + 2 * U) * (xh * wd).abs() + FTZ,
                                 what=f"rmsnorm y {tag}")
        gw = dyd * wd
        dot = (gw * xh).mean(-1, keepdim=True)
        ref = r * (gw - xh * dot)
        if dres is not None:
            ref = ref + dres[lo:hi].double()
        # dx = r * (dy w - x r dot): the two terms carry <= ~140 U each (rstd twice, the dot's fp32 sum over <= 53
        # adds measured against the sum of |terms|); 2^-16 = 256 U of their magnitudes, which only shows where they cancel
        slack = 2.0 ** -16 * (r * gw.abs() + r * xh.abs() * (gw * xh).abs().mean(-1, keepdim=True)) + FTZ
        assert_close_elementwise(dx[lo:hi], ref, ulps=1, abs_slack=slack, what=f"rmsnorm dx {tag}")
        dw_ref += (dyd * xh).sum(0)
        dw_abs += (dyd * xh).abs().sum(0)
    # dw: fp32 partials per CTA (rows / grid rows each; every CTA cap is >= one CTA per SM, 132), then a column sum over
    # <= rmsnorm_bwd_grid(rows) partials (32-way, then 32 warp sums); each term carries R_RSTD + 2U
    chain = math.ceil(rows / max(1, min(rows, 132))) + math.ceil(K.rmsnorm_bwd_grid(rows) / 32) + 32
    assert_close_elementwise(dw, dw_ref, ulps=1, abs_slack=(chain + 36) * U * dw_abs + FTZ, what=f"rmsnorm dw {tag}")


def _run_rmsnorm(K, rows, H, seed, with_dres=False, tag=""):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = _rows_with_scales(rows, H, gen)
    w = (1 + 0.1 * torch.randn(H, device="cuda", generator=gen)).bfloat16()
    dy = torch.randn(rows, H, device="cuda", generator=gen).bfloat16()
    dres = torch.randn(rows, H, device="cuda", generator=gen).bfloat16() if with_dres else None
    y, dx = torch.empty_like(x), torch.empty_like(x)
    rstd = torch.empty(rows, device="cuda")
    partial = torch.empty(K.rmsnorm_bwd_grid(rows), H, device="cuda")
    dw = torch.full_like(w, float("nan"))
    K.rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), rows, H, 1e-5, _sp())
    K.rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), rstd.data_ptr(), dx.data_ptr(), partial.data_ptr(),
                  dw.data_ptr(), False, rows, H, _sp(), dres.data_ptr() if dres is not None else 0)
    _check_rmsnorm(K, x, w, dy, dres, 1e-5, f"{tag}H={H} rows={rows}", y, rstd, dx, dw)


@gpu
@pytest.mark.parametrize("H", [8, 2048, 2056, 4096, 8192, 16384])
@pytest.mark.parametrize("rows", [1, 263, 264, 265, 791, 792, 793, 8192])
def test_rmsnorm_raw_launchers(K, rows, H):
    """Rows below, at and above the CTA caps (792 forward, 264 backward): one row or many per CTA. The H set reaches
    every launch shape: forward (NV, TPB) (1,128) (2,128) (4,128) (4,256) (4,512), backward (1,256) (2,256) (4,256)
    (4,512)."""
    _run_rmsnorm(K, rows, H, seed=rows * 7 + H, with_dres=(rows % 2 == 1))


@gpu
@pytest.mark.parametrize("with_dres", [False, True])
@pytest.mark.parametrize("rows,H", [(265, 2048), (8192, 4096)])
def test_rmsnorm_autograd_wrappers(rows, H, with_dres):
    """fused.rmsnorm and fused.norm_linear_res (W = identity, so the GEMMs are exact and y / dn are the norm's own)."""
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(rows + H)
    x0 = _rows_with_scales(rows, H, gen)
    w0 = (1 + 0.1 * torch.randn(H, device="cuda", generator=gen)).bfloat16()
    dy = torch.randn(rows, H, device="cuda", generator=gen).bfloat16()
    dres = torch.randn(rows, H, device="cuda", generator=gen).bfloat16() if with_dres else None
    K = fused._native.load()
    x, w = x0.clone().requires_grad_(), w0.clone().requires_grad_()
    y = fused.rmsnorm(x, w, 1e-5)
    y.backward(dy)
    _check_rmsnorm(K, x0, w0, dy, None, 1e-5, f"fused.rmsnorm H={H} rows={rows}", y.detach(),
                   _kernel_rstd(K, x0, w0), x.grad, w.grad)
    x, w = x0.clone().requires_grad_(), w0.clone().requires_grad_()
    eye = torch.eye(H, device="cuda", dtype=torch.bfloat16)
    xs, y = fused.norm_linear_res(x, w, eye, 1e-5)
    torch.autograd.backward([y, xs] if with_dres else [y], [dy, dres] if with_dres else [dy])
    _check_rmsnorm(K, x0, w0, dy, dres, 1e-5, f"norm_linear_res H={H} rows={rows} dres={with_dres}", y.detach(),
                   _kernel_rstd(K, x0, w0), x.grad, w.grad)


def _kernel_rstd(K, x, w):
    rows, H = x.shape
    y, rstd = torch.empty_like(x), torch.empty(rows, device="cuda")
    K.rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), rows, H, 1e-5, _sp())
    return rstd


@gpu
def test_empty_input_is_a_no_op_for_every_op(K):
    """rows = 0 (and T = 0): nothing is launched that could fail, and gradients of an empty batch are zero."""
    from torchft_b200.ops import fused

    for H in (8, 2048, 16384):
        x = torch.empty(0, H, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        w = torch.ones(H, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        y = fused.rmsnorm(x, w, 1e-5)
        y.sum().backward()
        assert y.shape == (0, H) and torch.equal(w.grad, torch.zeros_like(w))
        dw = torch.full((H,), 3.0, device="cuda", dtype=torch.bfloat16)
        partial = torch.empty(0, H, device="cuda")
        K.rmsnorm_bwd(0, 0, w.data_ptr(), 0, 0, partial.data_ptr(), dw.data_ptr(), True, 0, H, _sp())
        assert torch.equal(dw, torch.full_like(dw, 3.0))  # accumulating nothing leaves dw as it was
        x2 = torch.empty(2, 0, H, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        eye = torch.eye(H, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        xs, y2 = fused.norm_linear_res(x2, w, eye, 1e-5)
        (y2.sum() + xs.sum()).backward()
        assert x2.grad.shape == x2.shape
    gu = torch.empty(0, 2 * 64, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    fused.swiglu(gu).sum().backward()
    assert gu.grad.shape == gu.shape
    qkv = torch.empty(0, 12 * 64, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    cs = fused.rope_table(8, 64, 5e5, qkv.device)
    q, k, v = fused.rope_qkv(qkv, cs, 0, 8, 8, 2, 64)
    (q.sum() + k.sum() + v.sum()).backward()
    logits = torch.empty(0, 1000, device="cuda", dtype=torch.bfloat16)
    assert fused.cross_entropy_inplace(logits, torch.empty(0, dtype=torch.long, device="cuda")).shape == (0,)
    torch.cuda.synchronize()


# ------------------------------------------------------------------ SwiGLU
SWIGLU_SPECIAL = (0.0, 20.0, -20.0, 88.0, -88.0, 100.0, -100.0, 1e4, -1e4)
# __fdividef(x, y) returns 0 for 2^126 < |y| < 2^128, and x / inf = 0 beyond: where 1 + e^-g >= 2^126 (g < -87.34) the
# kernel's sigmoid is 0 instead of e^g ~ 1e-38; its output there may be 0 (slack = |ref|)
FDIV_FLOOR = 126 * math.log(2) - 1e-3


def _swiglu_ref(g, u, d):
    gd, ud = g.double(), u.double()
    s = torch.sigmoid(gd)
    silu = gd * s
    over = (-gd >= FDIV_FLOOR).double()
    # __expf(x) is within 2 + 1.16|x| ulp (<= (4 + 2.32|g|) U); 1 + e, __fdividef (4 U), g * s and * u or * d: <= 11 U more
    rel = (11 + 2.32 * gd.abs()) * U
    y = silu * ud
    out = {"y": (y, rel * y.abs() + over * y.abs() + FTZ)}
    if d is not None:
        dd = d.double()
        du = dd * silu
        dg = dd * ud * (s + silu * (1 - s))
        # s + silu (1 - s) = s (1 + g (1 - s)) cancels at g ~ -1.28: bound against the magnitudes of its terms (+3 U for
        # 1 - s, the sum and the product with d * u)
        dg_slack = (rel + 3 * U) * (dd * ud).abs() * (s + silu.abs() * (1 - s)) + over * dg.abs() + FTZ
        out["du"] = (du, rel * du.abs() + over * du.abs() + FTZ)
        out["dg"] = (dg, dg_slack)
    return out


@gpu
@pytest.mark.parametrize("T,F", [(8192, 8192), (8192, 14336), (8191, 8200), (37, 192)])
def test_swiglu_fwd_bwd(K, T, F):
    """T*F/8 = 16 (15.5) passes of the grid-stride loop at the flagship shapes, a count that is not a multiple of the grid's
    thread count (8191 x 8200), and one pass; gate values at 0, +-20, +-88, +-100, +-1e4."""
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(T + F)
    gate = (torch.randn(T, F, device="cuda", generator=gen) * 3).bfloat16()
    pos = torch.randint(0, T * F, (4096,), device="cuda", generator=gen)
    special = torch.tensor(SWIGLU_SPECIAL, device="cuda", dtype=torch.bfloat16)
    gate.view(-1)[pos] = special[torch.arange(4096, device="cuda") % len(special)]
    gate[0, : len(SWIGLU_SPECIAL)] = special
    gu = torch.cat([gate, torch.randn(T, F, device="cuda", generator=gen).bfloat16()], 1)
    del gate
    dy = torch.randn(T, F, device="cuda", generator=gen).bfloat16()
    y = torch.empty(T, F, device="cuda", dtype=torch.bfloat16)
    dgu = torch.empty_like(gu)
    K.swiglu_fwd(gu.data_ptr(), y.data_ptr(), T, F, _sp())
    K.swiglu_bwd(dy.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, F, _sp())
    a = gu.clone().requires_grad_()
    ya = fused.swiglu(a)
    ya.backward(dy)
    assert torch.equal(ya, y) and torch.equal(a.grad, dgu)  # the autograd wrapper is the raw launcher
    step = max(1, (1 << 23) // F)
    for lo in range(0, T, step):
        hi = min(T, lo + step)
        ref = _swiglu_ref(gu[lo:hi, :F], gu[lo:hi, F:], dy[lo:hi])
        tag = f"T={T} F={F}"
        assert_close_elementwise(y[lo:hi], ref["y"][0], ulps=1, abs_slack=ref["y"][1], what=f"swiglu y {tag}")
        assert_close_elementwise(dgu[lo:hi, :F], ref["dg"][0], ulps=1, abs_slack=ref["dg"][1], what=f"swiglu dgate {tag}")
        assert_close_elementwise(dgu[lo:hi, F:], ref["du"][0], ulps=1, abs_slack=ref["du"][1], what=f"swiglu dup {tag}")


# ------------------------------------------------------------------ RoPE + q/k/v split
def _table_ref(S, D, theta):
    inv = torch.tensor(theta, dtype=torch.float64) ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
    ang = torch.outer(torch.arange(S, dtype=torch.float64), inv).cuda()
    return torch.stack((ang.cos(), ang.sin()), -1)


def _rot_ref(x, cs64, err, sign):
    """x [n, H, D] (bf16) rotated by the fp64 table rows cs64 [n, D/2, 2]; slack from the fp32 table's own error err."""
    xd = x.double().unflatten(-1, (-1, 2))
    c, s = cs64[:, None, :, 0], sign * cs64[:, None, :, 1]
    x0, x1 = xd[..., 0], xd[..., 1]
    out = torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), -1).flatten(-2)
    # the kernel rotates with the fp32 table (error err per entry) in fp32: 2 roundings of terms <= |x0| + |x1|
    sl = (x0.abs() + x1.abs()) * (err[:, None] + 2 * U)
    return out, torch.stack((sl, sl), -1).flatten(-2) + FTZ


@gpu
@pytest.mark.parametrize("B,S,Hq,Hkv,D,table", [(1, 8192, 32, 8, 64, 8192), (1, 8192, 32, 8, 128, 8192),
                                                  (2, 4096, 32, 8, 64, 4096), (2, 1000, 32, 8, 64, 8192)])
def test_rope_qkv_fwd_bwd(K, B, S, Hq, Hkv, D, table):
    """Positions up to 8191 at theta = 5e5; an 8192-row table used at S = 1000 (the model's cache only grows); backward
    from SDPA-ordered [B, H, S, D] gradients."""
    from torchft_b200.ops import fused

    theta = 5e5
    cs = fused.rope_table(table, D, theta, torch.device("cuda"))
    cs64 = _table_ref(table, D, theta)
    err = (cs.double() - cs64).abs().amax(-1)  # [table, D/2]
    # the table's own error: pow (<= 4 ulp = 8 U), the reciprocal and pos * inv (U each) give an angle error <= 10 U pos;
    # cosf / sinf add <= 2 ulp of a value <= 1 (2 U)
    pos = torch.arange(table, device="cuda", dtype=torch.float64)[:, None]
    assert_close_elementwise(err, torch.zeros_like(err), ulps=0, abs_slack=(10 * pos + 2) * U, what=f"rope table D={D}")
    gen = torch.Generator(device="cuda").manual_seed(S + D)
    row = (Hq + 2 * Hkv) * D
    qkv0 = torch.randn(B * S, row, device="cuda", generator=gen).bfloat16()
    qkv = qkv0.clone().requires_grad_()
    q, k, v = fused.rope_qkv(qkv, cs, B, S, Hq, Hkv, D)
    assert torch.equal(v.reshape(B * S, Hkv * D), qkv0[:, (Hq + Hkv) * D :])
    dq = torch.randn(B, Hq, S, D, device="cuda", generator=gen).bfloat16().transpose(1, 2)
    dk = torch.randn(B, Hkv, S, D, device="cuda", generator=gen).bfloat16().transpose(1, 2)
    dv = torch.randn(B, Hkv, S, D, device="cuda", generator=gen).bfloat16().transpose(1, 2)
    torch.autograd.backward([q, k, v], [dq, dk, dv])
    dqkv = qkv.grad
    # the raw launcher, with v written out (dir 0), must agree bit for bit and copy v exactly
    q2, k2, v2 = (torch.empty(B, S, h, D, device="cuda", dtype=torch.bfloat16) for h in (Hq, Hkv, Hkv))
    K.rope_qkv(qkv0.data_ptr(), row, q2.data_ptr(), k2.data_ptr(), v2.data_ptr(),
               [*q2.stride()[:3], *k2.stride()[:3], *v2.stride()[:3]], cs.data_ptr(), B * S, S, D, Hq, Hkv, 0, _sp())
    assert torch.equal(q2, q) and torch.equal(k2, k) and torch.equal(v2, v)
    assert torch.equal(dqkv[:, (Hq + Hkv) * D :].view(B, S, Hkv, D), dv)  # dv is a plain copy
    tag = f"B={B} S={S} D={D}"
    for b in range(B):
        for lo in range(0, S, 2048):
            hi = min(S, lo + 2048)
            t = slice(b * S + lo, b * S + hi)
            c64, e = cs64[lo:hi], err[lo:hi]
            packed = qkv0[t].view(hi - lo, Hq + 2 * Hkv, D)
            for name, got, x, heads in (("q", q[b, lo:hi], packed[:, :Hq], Hq), ("k", k[b, lo:hi], packed[:, Hq:Hq + Hkv], Hkv)):
                ref, sl = _rot_ref(x, c64, e, 1.0)
                assert_close_elementwise(got, ref, ulps=1, abs_slack=sl, what=f"rope {name} {tag}")
            dpk = dqkv[t].view(hi - lo, Hq + 2 * Hkv, D)
            for name, got, g in (("dq", dpk[:, :Hq], dq[b, lo:hi]), ("dk", dpk[:, Hq:Hq + Hkv], dk[b, lo:hi])):
                ref, sl = _rot_ref(g, c64, e, -1.0)
                assert_close_elementwise(got, ref, ulps=1, abs_slack=sl, what=f"rope {name} {tag}")


# ------------------------------------------------------------------ softmax cross-entropy
def _xent_ref(z, tgt, grad_scale, ignore=-100):
    """Per-row loss and gradient of bf16 logits z [n, V] in fp64, with the kernel's error bounds."""
    n, V = z.shape
    zd = z.double()
    valid = tgt != ignore
    t = torch.where(valid, tgt, 0)
    m = zd.amax(-1, keepdim=True)
    e = torch.exp(zd - m)
    gs = e.sum(-1, keepdim=True)
    lse = m + gs.log()
    p = e / gs
    loss = (lse[:, 0] - zd.gather(1, t[:, None])[:, 0]) * valid
    onehot = torch.zeros_like(zd).scatter_(1, t[:, None], 1.0)
    grad = grad_scale * (p - onehot) * valid[:, None]
    # Each element reaches the row sum through <= P __expf calls whose (negative) arguments add up to x - max: relative
    # error <= (4 P + 2.32 (max - x)) U; the fp32 sum runs along <= C adds (10 per 8-wide vector a thread owns, 10
    # shuffle levels). P and C from the <= nv vectors per thread of 1024.
    nv = math.ceil(V / 8 / 1024) + 1
    P, C = nv + 2, 10 * nv + 10
    gap = m - zd
    d_gs = (4 * P + 2.32 * (p * gap).sum(-1, keepdim=True)) * U + C * U  # relative error of the sum
    # loss = max + __logf(sum) - x_t: __logf is within 2^-21.41 on [0.5, 2], else 3 ulp (6 U relative); two fp32 roundings
    loss_bound = (d_gs[:, 0] + 2.0 ** -21.41 + 6 * U * gs[:, 0].log() + U * (lse[:, 0].abs() + loss.abs())) * valid
    # gradient: __expf(x - max) (4 + 2.32 gap) U, __fdividef 4 U, the product U, plus the sum's error, on p * grad_scale;
    # at the target p - 1 cancels, so this is an absolute slack; 1 ulp covers the rounding to bf16
    grad_slack = grad_scale * p * ((9 + 2.32 * gap) * U + d_gs) * valid[:, None] + FTZ
    return loss, loss_bound, grad, grad_slack


def _xent_logits(rows, V, gen):
    scale = torch.tensor((1.0, 8.0, 30.0), device="cuda")[torch.arange(rows, device="cuda") % 3]
    z = (torch.randn(rows, V, device="cuda", generator=gen) * scale[:, None]).bfloat16()
    z[5] = 0.5  # an all-equal row
    tgt = torch.randint(0, V, (rows,), device="cuda", generator=gen)
    r = torch.arange(rows, device="cuda")
    tgt = torch.where(r % 7 == 0, z.float().argmax(-1), tgt)  # target at the row's max
    tgt = torch.where(r % 7 == 1, z.float().argmin(-1), tgt)  # ... at its min
    tgt = torch.where(r % 11 == 3, torch.full_like(tgt, -100), tgt)  # ignored rows
    return z, tgt


@gpu
def test_xent_flagship_vocab(K):
    from torchft_b200.ops import fused

    rows, V, gsc = 2048, 128256, 1.0 / 2048
    gen = torch.Generator(device="cuda").manual_seed(41)
    z, tgt = _xent_logits(rows, V, gen)
    g_raw = z.clone()
    loss_raw = torch.empty(rows, device="cuda")
    K.xent(g_raw.data_ptr(), tgt.data_ptr(), loss_raw.data_ptr(), rows, V, V, gsc, -100, _sp())
    g = z.clone()
    loss = fused.cross_entropy_inplace(g, tgt, gsc)
    assert torch.equal(loss, loss_raw) and torch.equal(g, g_raw)
    ign = tgt == -100
    assert ign.any() and (loss[ign] == 0).all() and (g[ign] == 0).all()  # ignored rows: exactly zero
    for lo in range(0, rows, 128):
        sl = slice(lo, lo + 128)
        ref, bound, gref, gslack = _xent_ref(z[sl], tgt[sl], gsc)
        assert_close_elementwise(loss[sl], ref, ulps=0, abs_slack=bound, what="xent loss V=128256")
        assert_close_elementwise(g[sl], gref, ulps=1, abs_slack=gslack, what="xent grad V=128256")


@gpu
@pytest.mark.parametrize("V", [1001, 1007])
def test_xent_tail_under_padded_stride(K, V):
    """V % 8 != 0 inside a stride-1008 buffer: the scalar tail loop, with targets in the tail and in the vector body;
    the padding columns are never touched."""
    from torchft_b200.ops import fused

    rows, stride, gsc = 64, 1008, 0.25
    gen = torch.Generator(device="cuda").manual_seed(V)
    buf = (torch.randn(rows, stride, device="cuda", generator=gen) * 4).bfloat16()
    z = buf[:, :V].clone()
    tgt = torch.randint(0, V, (rows,), device="cuda", generator=gen)
    tgt[:6] = torch.tensor([V - 1, 1000, 0, 7, 999, -100], device="cuda")
    tgt[6] = int(z[6].float().argmax())
    pad = buf[:, V:].clone()
    loss = torch.empty(rows, device="cuda")
    b1 = buf.clone()
    K.xent(b1.data_ptr(), tgt.data_ptr(), loss.data_ptr(), rows, V, stride, gsc, -100, _sp())
    b2 = buf.clone()
    loss2 = fused.cross_entropy_inplace(b2[:, :V], tgt, gsc)
    assert torch.equal(loss, loss2) and torch.equal(b1, b2)
    assert torch.equal(b1[:, V:], pad)
    ref, bound, gref, gslack = _xent_ref(z, tgt, gsc)
    assert_close_elementwise(loss, ref, ulps=0, abs_slack=bound, what=f"xent loss tail V={V}")
    assert_close_elementwise(b1[:, :V], gref, ulps=1, abs_slack=gslack, what=f"xent grad tail V={V}")


# ------------------------------------------------------------------ linear cross-entropy
def _lce_ref(h, W, tgt, chunk, n_valid):
    """fp64 loss, dh, dW of mean CE(h @ W^T) over non-ignored targets, with bounds for the kernel path: bf16 logits from
    an fp32-accumulating GEMM, the xent kernel, bf16 dlogits, fp32 GEMMs for dh and dW, and dW accumulated chunk by chunk
    in bf16 (addmm_: one rounding of the running sum per chunk)."""
    T, H = h.shape
    V = W.shape[0]
    Wd, Wa = W.double(), W.double().abs()
    loss = torch.zeros((), dtype=torch.float64, device="cuda")
    loss_bound = torch.zeros_like(loss)
    dh, dh_slack = torch.empty(T, H, dtype=torch.float64, device="cuda"), torch.empty(T, H, dtype=torch.float64, device="cuda")
    dW, dW_slack = torch.zeros(V, H, dtype=torch.float64, device="cuda"), torch.zeros(V, H, dtype=torch.float32, device="cuda")
    gsc = 1.0 / n_valid
    for clo in range(0, T, chunk):
        chi = min(T, clo + chunk)
        for lo in range(clo, chi, 512):
            hi = min(chi, lo + 512)
            hd = h[lo:hi].double()
            z = hd @ Wd.t()
            # a logit is one bf16 rounding (<= 2^-8 relative) of an fp32 sum of H products (<= H U of sum |products|)
            dz = 2.0 ** -8 * z.abs() + H * U * (hd.abs() @ Wa.t())
            valid = tgt[lo:hi] != -100
            l_ref, l_b, g_ref, g_sl = _xent_ref(z, tgt[lo:hi], gsc)
            p = g_ref / gsc + torch.zeros_like(z).scatter_(1, torch.where(valid, tgt[lo:hi], 0)[:, None], 1.0) * valid[:, None]
            t = torch.where(valid, tgt[lo:hi], 0)[:, None]
            # a logit error dz_j moves p_j by p_j (dz_j + sum_i p_i dz_i) and the loss by dz_t + sum_i p_i dz_i
            shift = (p * dz).sum(-1, keepdim=True)
            loss += l_ref.sum()
            loss_bound += (l_b + (dz.gather(1, t)[:, 0] + shift[:, 0]) * valid).sum()
            # dlogits: that, the kernel's own error, and its rounding to bf16 (<= 2^-8 relative)
            E = gsc * p * (dz + shift) * valid[:, None] + g_sl + 2.0 ** -8 * g_ref.abs()
            dh[lo:hi] = g_ref @ Wd
            # dh: the dlogits errors through |W|, and an fp32 sum over V of |dlogits| |W|
            dh_slack[lo:hi] = E @ Wa + V * U * (g_ref.abs() @ Wa)
            dW += g_ref.t() @ hd
            dW_slack += (E.t() @ hd.abs() + (chi - clo) * U * (g_ref.abs().t() @ hd.abs())).float()
            del z, dz, p, E, g_ref, g_sl
        dW_slack += (2.0 ** -8 * dW.abs()).float()  # addmm_ rounds the running sum to bf16 once per chunk
    return loss / n_valid, loss_bound / n_valid, dh, dh_slack, dW, dW_slack


@gpu
@pytest.mark.parametrize("direct", [False, True])
@pytest.mark.parametrize("chunk", [2048, 3000])
def test_linear_cross_entropy_flagship(direct, chunk):
    """T = 8192, H = 2048, V = 128256; chunk 3000 does not divide T; dW written into a flat-gradient slot or a new tensor;
    one target in ten ignored (mean over the rest)."""
    from torchft_b200.ops import fused

    T, H, V = 8192, 2048, 128256
    gen = torch.Generator(device="cuda").manual_seed(chunk + direct)
    h0 = torch.randn(T, H, device="cuda", generator=gen).bfloat16()
    W0 = (torch.randn(V, H, device="cuda", generator=gen) * 0.02).bfloat16()
    tgt = torch.randint(0, V, (T,), device="cuda", generator=gen)
    tgt[torch.randperm(T, device="cuda", generator=gen)[: T // 10]] = -100
    n_valid = int((tgt != -100).sum())
    h, W = h0.clone().requires_grad_(), W0.clone().requires_grad_()
    if direct:
        W._flat_grad = torch.full_like(W0, float("nan"))
    loss = fused.linear_cross_entropy(h, W, tgt, chunk=chunk)
    loss.backward()
    ref, bound, dh, dh_sl, dW, dW_sl = _lce_ref(h0, W0, tgt, chunk, n_valid)
    tag = f"chunk={chunk} direct={direct}"
    # + the fp32 sum of T per-row losses (T U relative) and the division and scaling (2 U)
    assert_close_elementwise(loss.detach(), ref, ulps=0, abs_slack=bound + (T + 2) * U * ref.abs(), what=f"lce loss {tag}")
    assert_close_elementwise(h.grad, dh, ulps=1, abs_slack=dh_sl, what=f"lce dh {tag}")
    # dW: the bound above allows one rounding of the running sum per chunk; on an H100 the worst element exceeded it by
    # 1% (about one extra half-ulp, e.g. cuBLAS splitting a chunk's token dimension), so one more ulp is allowed
    for lo in range(0, V, 16384):
        assert_close_elementwise(W.grad[lo:lo + 16384], dW[lo:lo + 16384], ulps=1, abs_slack=dW_sl[lo:lo + 16384].double(),
                                 what=f"lce dW {tag}")


@gpu
def test_linear_cross_entropy_valid_count_is_exact_and_sync_free():
    """All targets valid: the device count changes nothing, bit for bit. Ignored targets: forward and backward run with
    no host sync."""
    from torchft_b200.ops import fused

    T, H, V = 8192, 2048, 128256
    gen = torch.Generator(device="cuda").manual_seed(7)
    h0 = torch.randn(T, H, device="cuda", generator=gen).bfloat16()
    W0 = (torch.randn(V, H, device="cuda", generator=gen) * 0.02).bfloat16()
    tgt = torch.randint(0, V, (T,), device="cuda", generator=gen)
    out = []
    for count_valid in (False, True):
        h, W = h0.clone().requires_grad_(), W0.clone().requires_grad_()
        loss = fused.linear_cross_entropy(h, W, tgt, chunk=2048, count_valid=count_valid)
        loss.backward()
        out.append((loss.detach(), h.grad, W.grad))
    for a, b in zip(*out):
        assert torch.equal(a, b)
    tgt[::4] = -100
    h, W = h0.clone().requires_grad_(), W0.clone().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = fused.linear_cross_entropy(h, W, tgt, chunk=2048)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    # and the mean is over the 3/4 of the targets that count: exactly the all-rows mean scaled by T / n_valid
    h2, W2 = h0.clone().requires_grad_(), W0.clone().requires_grad_()
    loss_t = fused.linear_cross_entropy(h2, W2, tgt, chunk=2048, count_valid=False)
    n_valid = T - T // 4
    assert abs(loss.item() - loss_t.item() * T / n_valid) <= 4 * U * abs(loss.item())


# ------------------------------------------------------------------ AdamW
@gpu
@pytest.mark.parametrize("n", [7, 8, 10007, (1 << 20) + 3, 40_000_000])
def test_flat_adamw_steps(n):
    """Ten steps from the kernel's own state, each against one fp64 step, at b2 = 0.95 and at b2 = 0.999, where a bias
    correction taken from the double beta instead of the fp32 one the moving averages use is hundreds of ulps off."""
    for b2 in (0.95, 0.999):
        _flat_adamw_steps(n, b2)


def _flat_adamw_steps(n, b2):
    from torchft_b200.ops import fused

    gen = torch.Generator(device="cuda").manual_seed(n % 1000)
    p = torch.randn(n, device="cuda", generator=gen).bfloat16()
    g = torch.zeros_like(p)
    lr, betas, eps, wd, gscale = 1e-3, (0.9, b2), 1e-8, 0.1, 0.37
    opt = fused.FlatAdamW(p, g, lr=lr, betas=betas, eps=eps, weight_decay=wd)
    gate = torch.ones(1, dtype=torch.int32, device="cuda")
    for step in range(1, 11):
        if step > 1:  # a zero gradient at step 1
            g.copy_(torch.randn(n, device="cuda", generator=gen) * (10.0 ** (step % 3 - 1)))
        w0, m0, v0 = opt.master.clone(), opt.m.clone(), opt.v.clone()
        opt.step(grad_scale=gscale, gate=gate)
        w_ref, w_sl, m_ref, m_sl, v_ref, v_sl = _adamw_ref(w0, m0, v0, g, lr, betas[0], betas[1], eps, wd, step, gscale,
                                                                opt.m, opt.v)
        assert_close_elementwise(opt.m, m_ref, ulps=0, abs_slack=m_sl + FTZ, what=f"adamw m n={n} b2={b2}")
        assert_close_elementwise(opt.v, v_ref, ulps=0, abs_slack=v_sl + FTZ, what=f"adamw v n={n} b2={b2}")
        assert_close_elementwise(opt.master, w_ref, ulps=1, abs_slack=w_sl + FTZ, what=f"adamw master n={n} b2={b2}")
        assert torch.equal(p, opt.master.bfloat16())  # p is exactly master rounded to bf16
    state = [t.clone() for t in (p, opt.master, opt.m, opt.v)]
    gate.zero_()
    opt.step(grad_scale=gscale, gate=gate)
    for a, b in zip(state, (p, opt.master, opt.m, opt.v)):
        assert torch.equal(a, b)  # gate 0: nothing moves


@gpu
def test_flat_adamw_step_ranges_matches_step():
    """The overlapped trainer's per-stage update (step_ranges over _compute_stage_ranges of a llama3_debug FlatParams) is
    the same update as step(), bit for bit; a range that does not start on a 16-byte boundary is refused before any launch."""
    from types import SimpleNamespace

    from torchft_b200.models.llama import CONFIGS, FlatParams, Llama
    from torchft_b200.ops import fused
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    model = Llama(CONFIGS["llama3_debug"], device="meta")
    flat = FlatParams(model, device=torch.device("cuda"))
    model.init_weights(0)
    ranges = FaultTolerantTrainer._compute_stage_ranges(SimpleNamespace(flat=flat, model=model))
    gen = torch.Generator(device="cuda").manual_seed(3)
    opts = []
    for _ in range(2):
        p, g = flat.param.clone(), torch.zeros_like(flat.grad)
        opts.append(fused.FlatAdamW(p, g, lr=1e-3))
    stream = torch.cuda.Stream()
    events = [torch.cuda.Event() for _ in ranges]
    for step in range(3):
        gr = torch.randn(flat.numel, device="cuda", generator=gen).bfloat16()
        for o in opts:
            o.g.copy_(gr)
        opts[0].step(grad_scale=0.5)
        stream.wait_stream(torch.cuda.current_stream())
        opts[1].step_ranges(ranges, (stream, events), grad_scale=0.5)
        torch.cuda.current_stream().wait_stream(stream)
        for a, b in zip((opts[0].p, opts[0].master, opts[0].m, opts[0].v), (opts[1].p, opts[1].master, opts[1].m, opts[1].v)):
            assert torch.equal(a, b)
    before = [t.clone() for t in (opts[1].p, opts[1].master, opts[1].m, opts[1].v)]
    t0 = opts[1].t
    with pytest.raises(ValueError, match="multiples of 8"):
        opts[1].step_ranges([(0, 12), (12, flat.numel)], (stream, events[:2]))
    torch.cuda.synchronize()
    assert opts[1].t == t0
    for a, b in zip(before, (opts[1].p, opts[1].master, opts[1].m, opts[1].v)):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ DiLoCo outer step
@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 4099, 10_000_005])
def test_diloco_outer(K, dtype, n):
    """Torch-SGD semantics (momentum mu, optional Nesterov) on the last global weights, then lerp towards the local ones."""
    from _diloco_ref import outer_ref
    from torchft_b200.ops import _native

    gen = torch.Generator(device="cuda").manual_seed(n)
    lr = 0.7
    for mu in (0.0, 0.9):
        for nesterov in (False, True):
            for alpha in (0.0, 0.3, 1.0):
                orig = torch.randn(n, device="cuda", generator=gen).to(dtype)
                param = (orig.float() + 0.1 * torch.randn(n, device="cuda", generator=gen)).to(dtype)
                grad = (0.05 * torch.randn(n, device="cuda", generator=gen)).to(dtype)
                mom = 0.05 * torch.randn(n, device="cuda", generator=gen)
                o0, l0, b0 = orig.clone(), param.clone(), mom.clone()
                K.diloco_outer(param.data_ptr(), orig.data_ptr(), grad.data_ptr(), mom.data_ptr(), n, _native.dtype_code(grad),
                               lr, mu, nesterov, alpha, 0, _sp())
                ref = outer_ref(o0, l0, b0, grad, lr, mu, nesterov, alpha)
                tag = f"{dtype} n={n} mu={mu} nesterov={nesterov} alpha={alpha}"
                if ref.mom_slack is not None:
                    assert_close_elementwise(mom, ref.mom, ulps=0, abs_slack=ref.mom_slack, what=f"diloco mom {tag}")
                else:
                    assert torch.equal(mom, b0)  # no momentum: the buffer is not touched
                assert_close_elementwise(orig, ref.orig, ulps=1, abs_slack=ref.orig_slack, what=f"diloco original {tag}")
                assert_close_elementwise(param, ref.param, ulps=1, abs_slack=ref.param_slack, what=f"diloco param {tag}")
    gate = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = [t.clone() for t in (param, orig, mom)]
    K.diloco_outer(param.data_ptr(), orig.data_ptr(), grad.data_ptr(), mom.data_ptr(), n, _native.dtype_code(grad), lr, 0.9,
                   True, 0.3, gate.data_ptr(), _sp())
    for a, b in zip(before, (param, orig, mom)):
        assert torch.equal(a, b)  # gate 0 changes nothing


# ------------------------------------------------------------------ the whole model
@gpu
@pytest.mark.parametrize("ignored", [False, True])
def test_llama_debug_matches_reference(ignored):
    """llama3_debug at B=2, S=512 against the fp32 eager reference, with all targets valid and with about a quarter
    ignored (-100): the loss is the mean over the targets that count, and so is every gradient."""
    from torchft_b200.models.llama import CONFIGS, Llama
    from torchft_b200.models.reference import reference_loss

    cfg = CONFIGS["llama3_debug"]
    gen = torch.Generator(device="cuda").manual_seed(17)
    m = Llama(cfg, device="cuda")
    m.init_weights(0)
    tok = torch.randint(0, cfg.vocab_size, (2, 512), device="cuda", generator=gen)
    tgt = torch.randint(0, cfg.vocab_size, (2, 512), device="cuda", generator=gen)
    if ignored:
        tgt[torch.rand(2, 512, device="cuda", generator=gen) < 0.25] = -100
    loss = m(tok, tgt)
    loss.backward()
    ref_loss, ref_grads = reference_loss(m, tok, tgt)
    # bf16 activations and weights against an fp32 graph: the loss within 2^-8 relative (one bf16 rounding's worth),
    # every gradient within 2% in norm (at most 0.8% measured on an H100 80GB HBM3 at 400 W, in both cases); a gradient
    # scaled by n_valid / T, as before the loss counted only valid targets, is off by 25%
    assert abs(loss.item() - ref_loss) <= 2.0 ** -8 * abs(ref_loss), (loss.item(), ref_loss)
    for name, p in m.named_parameters():
        r = _rel(p.grad, ref_grads[name])
        print(f"[model] ignored={ignored} {name}: rel {r:.3g}")
        assert r < 0.02, (name, r)
