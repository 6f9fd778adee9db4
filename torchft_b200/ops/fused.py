"""Autograd wrappers over the hand-written sm_90a model kernels.

RMSNorm / SwiGLU / RoPE / chunked linear-cross-entropy / flat AdamW. All take
bf16 CUDA tensors, reduce in fp32 and make one pass over HBM per direction.
There is no PyTorch fallback: on a CUDA box these always run ``_K`` kernels.
"""

from __future__ import annotations

from typing import Optional, Tuple

import torch

from torchft_b200.ops import _native


def _wgrad(dy2: torch.Tensor, x2: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """dW = dy2^T @ x2. When ``W`` lives in a FlatParams buffer and has no gradient yet, the GEMM
    writes STRAIGHT into W's slice of the flat (NVLink-symmetric) gradient buffer and returns that
    view; autograd then adopts it as ``W.grad`` without a copy. This removes the per-step
    zero-fill of the gradient buffer and the read-modify-write accumulation pass (~64 GB of HBM
    traffic per step for an 8B model): the wgrad epilogue IS the bucket write."""

    slot = getattr(W, "_flat_grad", None)
    if slot is not None and W.grad is None and slot.dtype == dy2.dtype:
        return torch.mm(dy2.t(), x2, out=slot.view(W.shape))
    return dy2.t() @ x2


def _chk(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda or t.dtype != torch.bfloat16:
        raise TypeError(f"{name} must be a bf16 CUDA tensor, got {t.dtype} on {t.device}")
    if t.data_ptr() % 16:
        raise ValueError(f"{name} must be 16-byte aligned")


class _RMSNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:  # type: ignore[override]
        K = _native.load()
        x = x.contiguous()
        _chk(x, "x")
        _chk(w, "weight")
        H = x.shape[-1]
        rows = x.numel() // H
        y = torch.empty_like(x)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        K.rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), rows, H, eps, _native.stream_ptr())
        ctx.save_for_backward(x, w, rstd)
        return y

    @staticmethod
    def backward(ctx, dy: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        x, w, rstd = ctx.saved_tensors
        dy = dy.contiguous()
        H = x.shape[-1]
        rows = x.numel() // H
        dx = torch.empty_like(x)
        grid = K.rmsnorm_bwd_grid(rows)
        partial = torch.empty((grid, H), dtype=torch.float32, device=x.device)
        dw = torch.empty_like(w)
        K.rmsnorm_bwd(
            dy.data_ptr(), x.data_ptr(), w.data_ptr(), rstd.data_ptr(), dx.data_ptr(),
            partial.data_ptr(), dw.data_ptr(), False, rows, H, _native.stream_ptr(),
        )
        return dx, dw, None


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """y = x * rsqrt(mean(x^2) + eps) * weight (fp32 statistics, bf16 I/O)."""
    return _RMSNorm.apply(x, weight, eps)


class _SwiGLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gu: torch.Tensor) -> torch.Tensor:  # type: ignore[override]
        K = _native.load()
        gu = gu.contiguous()
        _chk(gu, "gate_up")
        F2 = gu.shape[-1]
        F = F2 // 2
        T = gu.numel() // F2
        y = torch.empty(gu.shape[:-1] + (F,), dtype=gu.dtype, device=gu.device)
        K.swiglu_fwd(gu.data_ptr(), y.data_ptr(), T, F, _native.stream_ptr())
        ctx.save_for_backward(gu)
        return y

    @staticmethod
    def backward(ctx, dy: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        (gu,) = ctx.saved_tensors
        dy = dy.contiguous()
        F2 = gu.shape[-1]
        T = gu.numel() // F2
        dgu = torch.empty_like(gu)
        K.swiglu_bwd(dy.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, F2 // 2, _native.stream_ptr())
        return dgu


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    """silu(gate) * up for a packed ``[..., 2F]`` (gate | up) projection output."""
    return _SwiGLU.apply(gate_up)


def rope_table(seq_len: int, head_dim: int, theta: float, device: torch.device) -> torch.Tensor:
    """(cos, sin) table ``[seq_len, head_dim/2, 2]`` fp32 for interleaved-pair RoPE."""

    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=device) / head_dim))
    ang = torch.outer(torch.arange(seq_len, dtype=torch.float32, device=device), inv)
    return torch.stack((ang.cos(), ang.sin()), dim=-1).contiguous()


class _RoPEQKV(torch.autograd.Function):
    """RoPE on q and k read directly from the fused qkv projection output.

    Returns (q [B,S,Hq,D], k [B,S,Hkv,D] contiguous, v [B,S,Hkv,D] as a view of the projection) so the rotation doubles
    as the q/k/v split: ONE launch. Backward is one launch too: it reads dq/dk/dv in whatever stride order SDPA
    produced them, applies the inverse rotation and writes ONE packed d_qkv buffer (no zero-padded slice gradients,
    no torch.cat, no .contiguous()).
    """

    @staticmethod
    def forward(ctx, qkv: torch.Tensor, cs: torch.Tensor, B: int, S: int, Hq: int, Hkv: int, D: int):  # type: ignore[override]
        K = _native.load()
        assert qkv.is_contiguous() and qkv.dtype == torch.bfloat16
        # the kernel reads the table as fp32: a wrapper that down-casts module inputs (FSDP2's cast_forward_inputs) would
        # make it read garbage and past the end of the buffer
        assert cs.dtype == torch.float32 and cs.is_contiguous() and cs.shape[0] >= S, "rope table must be the fp32 table of rope_table()"
        row = qkv.shape[-1]
        assert row == (Hq + 2 * Hkv) * D
        q = torch.empty((B, S, Hq, D), dtype=qkv.dtype, device=qkv.device)
        k = torch.empty((B, S, Hkv, D), dtype=qkv.dtype, device=qkv.device)
        # one launch rotates q and k out of the packed rows; v stays a strided view of the projection (no copy)
        K.rope_qkv(qkv.data_ptr(), row, q.data_ptr(), k.data_ptr(), 0, [*q.stride()[:3], *k.stride()[:3], 0, 0, 0],
                   cs.data_ptr(), B * S, S, D, Hq, Hkv, 0, _native.stream_ptr())
        v = qkv.view(B * S, row)[:, (Hq + Hkv) * D :].reshape(B, S, Hkv, D)
        ctx.save_for_backward(cs)
        ctx.meta = (B, S, Hq, Hkv, D, row)
        return q, k, v

    @staticmethod
    def backward(ctx, dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        (cs,) = ctx.saved_tensors
        B, S, Hq, Hkv, D, row = ctx.meta

        def usable(t: torch.Tensor) -> torch.Tensor:
            # the kernel takes any (batch, position, head) stride order (SDPA hands back [B, H, S, D]-ordered gradients
            # seen through a transpose) as long as a head vector is contiguous and 16 B aligned
            ok = t.stride(3) == 1 and all(st % 8 == 0 for st in t.stride()[:3]) and t.data_ptr() % 16 == 0
            return t if ok else t.contiguous()

        dq, dk, dv = usable(dq), usable(dk), usable(dv)
        dqkv = torch.empty((B * S, row), dtype=dq.dtype, device=dq.device)
        K.rope_qkv(dqkv.data_ptr(), row, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                   [*dq.stride()[:3], *dk.stride()[:3], *dv.stride()[:3]], cs.data_ptr(), B * S, S, D, Hq, Hkv, 1,
                   _native.stream_ptr())
        return dqkv, None, None, None, None, None, None


def rope_qkv(qkv: torch.Tensor, cs: torch.Tensor, B: int, S: int, Hq: int, Hkv: int, D: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Split a packed ``[B*S, (Hq+2*Hkv)*D]`` projection into q, k, v with RoPE applied to q and k."""
    return _RoPEQKV.apply(qkv, cs, B, S, Hq, Hkv, D)


class _LinearCrossEntropy(torch.autograd.Function):
    """loss = mean CE(h @ W^T, target) without materialising fp32 logits.

    Tokens are processed in chunks: bf16 logits chunk (cuBLAS) -> fused
    softmax/CE kernel that overwrites the chunk with dlogits -> dh chunk and dW
    accumulation (cuBLAS). Peak extra memory = one bf16 logits chunk.
    """

    @staticmethod
    def forward(ctx, h: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, chunk: int, ignore_index: int, count_valid: bool):  # type: ignore[override]
        K = _native.load()
        T, H = h.shape
        V = weight.shape[0]
        # count_valid costs one host sync; training loops with no ignored
        # targets (the synthetic-data bench) pass count_valid=False.
        n_valid = max(int((target != ignore_index).sum().item()), 1) if count_valid else T
        need_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        dh = torch.empty_like(h) if need_grad else None
        slot = getattr(weight, "_flat_grad", None)
        direct = need_grad and slot is not None and weight.grad is None
        dW = (slot.view(weight.shape).zero_() if direct else torch.zeros_like(weight)) if need_grad else None
        ctx.direct = direct
        losses = torch.empty(T, dtype=torch.float32, device=h.device)
        sp = _native.stream_ptr()
        for lo in range(0, T, chunk):
            hi = min(lo + chunk, T)
            hc = h[lo:hi]
            logits = hc @ weight.t()  # [c, V] bf16, cuBLAS
            K.xent(
                logits.data_ptr(), target[lo:hi].data_ptr(), losses[lo:hi].data_ptr(), hi - lo, V,
                logits.stride(0), 1.0 / n_valid, ignore_index, sp,
            )
            if need_grad:
                torch.mm(logits, weight, out=dh[lo:hi])
                dW.addmm_(logits.t(), hc)
            del logits
        ctx.save_for_backward(dh, dW)
        ctx.need = need_grad
        return losses.sum() / n_valid

    @staticmethod
    def backward(ctx, g: torch.Tensor):  # type: ignore[override]
        dh, dW = ctx.saved_tensors
        # g is the upstream scalar (1.0 for a plain loss.backward()); fold it in
        # without a host sync.
        # (dW already sits in the flat gradient buffer when ctx.direct; scale in place)
        return dh * g.to(dh.dtype), (dW.mul_(g.to(dW.dtype)) if ctx.direct else dW * g.to(dW.dtype)), None, None, None, None


def linear_cross_entropy(h: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, chunk: int = 2048,
                         ignore_index: int = -100, count_valid: bool = True) -> torch.Tensor:
    """Mean cross entropy of ``h @ weight.T`` against ``target`` (int64)."""
    assert h.dim() == 2 and target.dim() == 1 and h.shape[0] == target.shape[0]
    return _LinearCrossEntropy.apply(h.contiguous(), weight, target.contiguous(), chunk, ignore_index, count_valid)


def cross_entropy_inplace(logits: torch.Tensor, target: torch.Tensor, grad_scale: float = 1.0, ignore_index: int = -100) -> torch.Tensor:
    """Per-row CE losses; overwrites ``logits`` (bf16, [rows, V]) with grad_scale * dlogits."""

    K = _native.load()
    assert logits.dim() == 2 and logits.stride(1) == 1
    losses = torch.empty(logits.shape[0], dtype=torch.float32, device=logits.device)
    K.xent(logits.data_ptr(), target.data_ptr(), losses.data_ptr(), logits.shape[0], logits.shape[1],
           logits.stride(0), grad_scale, ignore_index, _native.stream_ptr())
    return losses


class FlatAdamW:
    """AdamW over ONE flat bf16 parameter buffer with fp32 master/m/v state.

    The update is a single kernel launch over the whole model. ``gate`` is a
    device int32 tensor: when it holds 0 the launch is a no-op, so the step can
    be enqueued before the host learns the commit verdict (the reference only
    calls ``optim.step()`` after ``should_commit``, torchft/optim.py:52-55).
    """

    def __init__(self, flat_param: torch.Tensor, flat_grad: torch.Tensor, lr: float = 3e-4,
                 betas: Tuple[float, float] = (0.9, 0.95), eps: float = 1e-8, weight_decay: float = 0.1) -> None:
        assert flat_param.dtype == torch.bfloat16 and flat_grad.dtype == torch.bfloat16
        assert flat_param.numel() == flat_grad.numel()
        self.p = flat_param
        self.g = flat_grad
        self.master = flat_param.float()
        self.m = torch.zeros_like(self.master)
        self.v = torch.zeros_like(self.master)
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.t = 0
        self.direct_grads = False
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay, "params": [flat_param]}]

    def zero_grad(self, set_to_none: bool = False) -> None:
        # direct_grads: producers overwrite the whole flat buffer every step
        # (FlatParams.reset_grads + ops.fused._wgrad), so the 2-bytes/param memset is skipped.
        if not self.direct_grads:
            self.g.zero_()

    def step(self, grad_scale: float = 1.0, gate: Optional[torch.Tensor] = None) -> None:
        K = _native.load()
        self.t += 1
        lr = self.param_groups[0]["lr"]
        b1, b2 = self.betas
        K.adamw(
            self.p.data_ptr(), self.master.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.g.data_ptr(),
            self.p.numel(), lr, b1, b2, self.eps, self.weight_decay, 1.0 - b1 ** self.t, 1.0 - b2 ** self.t,
            grad_scale, gate.data_ptr() if gate is not None else 0, _native.stream_ptr(),
        )

    def step_ranges(self, ranges, streams_events, grad_scale: float = 1.0, gate: Optional[torch.Tensor] = None,
                    max_blocks: int = 0) -> None:
        """The same update as :meth:`step`, cut into element ranges ``[(lo, hi), ...]`` that are launched
        in the given order on ``stream``; ``events[i]`` is recorded after range ``i``. Lets the next
        forward start on the first layers while the (HBM-bound) update of later layers is still running
        underneath the (tensor-core-bound) GEMMs. ``streams_events`` = ``(stream, events)``."""
        K = _native.load()
        stream, events = streams_events
        self.t += 1
        lr = self.param_groups[0]["lr"]
        b1, b2 = self.betas
        bc1, bc2 = 1.0 - b1 ** self.t, 1.0 - b2 ** self.t
        gp = gate.data_ptr() if gate is not None else 0
        p, w, m, v, g = (t.data_ptr() for t in (self.p, self.master, self.m, self.v, self.g))
        for (lo, hi), ev in zip(ranges, events):
            K.adamw(p + 2 * lo, w + 4 * lo, m + 4 * lo, v + 4 * lo, g + 2 * lo, hi - lo, lr, b1, b2, self.eps,
                    self.weight_decay, bc1, bc2, grad_scale, gp, stream.cuda_stream, max_blocks)
            ev.record(stream)

    def grad_sumsq(self) -> torch.Tensor:
        K = _native.load()
        out = torch.zeros(1, dtype=torch.float32, device=self.g.device)
        K.sumsq(self.g.data_ptr(), self.g.numel(), out.data_ptr(), _native.stream_ptr())
        return out

    def state_dict(self) -> dict:
        return {"t": self.t, "master": self.master, "m": self.m, "v": self.v}

    def load_state_dict(self, sd: dict) -> None:
        self.t = int(sd["t"])
        self.master.copy_(sd["master"])
        self.m.copy_(sd["m"])
        self.v.copy_(sd["v"])
        self.p.copy_(self.master)


class _NormLinear(torch.autograd.Function):
    """y = rmsnorm(x, g) @ W^T, saving only (x, rstd): the normalised activation
    is recomputed in backward by one extra RMSNorm pass instead of living in HBM
    for the whole forward/backward (64 MB per call at 8k x 4096 bf16)."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, g: torch.Tensor, W: torch.Tensor, eps: float) -> torch.Tensor:  # type: ignore[override]
        K = _native.load()
        x = x.contiguous()
        H = x.shape[-1]
        rows = x.numel() // H
        n = torch.empty_like(x)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), rows, H, eps, _native.stream_ptr())
        y = n.view(rows, H) @ W.t()
        ctx.save_for_backward(x, g, W, rstd)
        ctx.eps = eps
        return y.view(x.shape[:-1] + (W.shape[0],))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        x, g, W, rstd = ctx.saved_tensors
        H = x.shape[-1]
        rows = x.numel() // H
        sp = _native.stream_ptr()
        dy2 = dy.reshape(rows, -1)
        n = torch.empty_like(x)
        K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), rows, H, ctx.eps, sp)
        dW = _wgrad(dy2, n.view(rows, H), W)
        dn = dy2 @ W
        dx = n  # reuse the recompute buffer for dx
        grid = K.rmsnorm_bwd_grid(rows)
        partial = torch.empty((grid, H), dtype=torch.float32, device=x.device)
        dg = torch.empty_like(g)
        K.rmsnorm_bwd(dn.data_ptr(), x.data_ptr(), g.data_ptr(), rstd.data_ptr(), dx.data_ptr(),
                      partial.data_ptr(), dg.data_ptr(), False, rows, H, sp)
        return dx, dg, dW, None


def norm_linear(x: torch.Tensor, norm_weight: torch.Tensor, W: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """``rmsnorm(x, norm_weight) @ W.T`` with the normalised activation recomputed in backward."""
    return _NormLinear.apply(x, norm_weight, W, eps)


class _NormLinearRes(torch.autograd.Function):
    """Pre-norm residual branch point: returns ``(x, rmsnorm(x, g) @ W^T)``.

    The first output IS ``x`` (the residual stream, to be consumed by the ``res=`` argument of
    :func:`linear` / :func:`swiglu_linear`). Routing the residual through this node means its
    gradient arrives here together with the branch gradient, and the RMSNorm backward kernel adds
    it while writing ``dx`` — autograd's separate ``dres + dbranch`` accumulation pass
    (3 x 64 MB of HBM traffic per norm at 8k x 4096) disappears.
    """

    @staticmethod
    def forward(ctx, x: torch.Tensor, g: torch.Tensor, W: torch.Tensor, eps: float):  # type: ignore[override]
        K = _native.load()
        x = x.contiguous()
        H = x.shape[-1]
        rows = x.numel() // H
        n = torch.empty_like(x)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), rows, H, eps, _native.stream_ptr())
        y = n.view(rows, H) @ W.t()
        ctx.save_for_backward(x, g, W, rstd)
        ctx.eps = eps
        return x, y.view(x.shape[:-1] + (W.shape[0],))  # autograd re-wraps the returned input as a new node output

    @staticmethod
    def backward(ctx, dres: Optional[torch.Tensor], dy: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        x, g, W, rstd = ctx.saved_tensors
        H = x.shape[-1]
        rows = x.numel() // H
        sp = _native.stream_ptr()
        dy2 = dy.reshape(rows, -1)
        n = torch.empty_like(x)
        K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), rows, H, ctx.eps, sp)
        dW = _wgrad(dy2, n.view(rows, H), W)
        dn = dy2 @ W
        dx = n  # reuse the recompute buffer for dx
        grid = K.rmsnorm_bwd_grid(rows)
        partial = torch.empty((grid, H), dtype=torch.float32, device=x.device)
        dg = torch.empty_like(g)
        if dres is not None:
            dres = dres.contiguous()
            assert dres.dtype == x.dtype and dres.numel() == x.numel()
        K.rmsnorm_bwd(dn.data_ptr(), x.data_ptr(), g.data_ptr(), rstd.data_ptr(), dx.data_ptr(),
                      partial.data_ptr(), dg.data_ptr(), False, rows, H, sp, dres.data_ptr() if dres is not None else 0)
        return dx, dg, dW, None


def norm_linear_res(x: torch.Tensor, norm_weight: torch.Tensor, W: torch.Tensor, eps: float = 1e-5) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(x, rmsnorm(x, norm_weight) @ W.T)``: like :func:`norm_linear` but also hands back the residual
    stream so that its gradient is accumulated inside the RMSNorm backward kernel."""
    return _NormLinearRes.apply(x, norm_weight, W, eps)


class _SwiGLULinear(torch.autograd.Function):
    """out = swiglu(gu) @ W2^T saving only gu (the [T, F] product is recomputed)."""

    @staticmethod
    def forward(ctx, gu: torch.Tensor, W2: torch.Tensor, res: Optional[torch.Tensor]) -> torch.Tensor:  # type: ignore[override]
        K = _native.load()
        gu = gu.contiguous()
        F2 = gu.shape[-1]
        F = F2 // 2
        T = gu.numel() // F2
        a = torch.empty((T, F), dtype=gu.dtype, device=gu.device)
        K.swiglu_fwd(gu.data_ptr(), a.data_ptr(), T, F, _native.stream_ptr())
        # residual add rides in the GEMM epilogue (beta = 1) instead of a separate elementwise pass
        out = a @ W2.t() if res is None else torch.addmm(res.reshape(T, -1), a, W2.t())
        ctx.save_for_backward(gu, W2)
        ctx.has_res = res is not None
        return out.view(gu.shape[:-1] + (W2.shape[0],))

    @staticmethod
    def backward(ctx, dout: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        gu, W2 = ctx.saved_tensors
        F2 = gu.shape[-1]
        F = F2 // 2
        T = gu.numel() // F2
        sp = _native.stream_ptr()
        d2 = dout.reshape(T, -1)
        a = torch.empty((T, F), dtype=gu.dtype, device=gu.device)
        K.swiglu_fwd(gu.data_ptr(), a.data_ptr(), T, F, sp)
        dW2 = _wgrad(d2, a, W2)
        da = torch.mm(d2, W2, out=a)  # reuse buffer
        dgu = torch.empty_like(gu)
        K.swiglu_bwd(da.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, F, sp)
        return dgu, dW2, (dout if ctx.has_res else None)


def swiglu_linear(gate_up: torch.Tensor, W2: torch.Tensor, res: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``(silu(gate) * up) @ W2.T (+ res)`` with the activation product recomputed in backward."""
    return _SwiGLULinear.apply(gate_up, W2, res)


class _Linear(torch.autograd.Function):
    """y = x @ W^T whose weight gradient is written straight into the flat gradient buffer."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, W: torch.Tensor, res: Optional[torch.Tensor]) -> torch.Tensor:  # type: ignore[override]
        ctx.save_for_backward(x, W)
        ctx.has_res = res is not None
        if res is None:
            return x @ W.t()
        x2 = x.reshape(-1, x.shape[-1])
        return torch.addmm(res.reshape(x2.shape[0], -1), x2, W.t()).view(x.shape[:-1] + (W.shape[0],))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):  # type: ignore[override]
        x, W = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dW = _wgrad(dy2, x.reshape(-1, x.shape[-1]), W)
        return (dy2 @ W).view(x.shape), dW, (dy if ctx.has_res else None)


def linear(x: torch.Tensor, W: torch.Tensor, res: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``x @ W.T (+ res)`` with the wgrad GEMM writing directly into the flat gradient bucket; the
    residual add, when given, is the GEMM's beta=1 epilogue."""
    return _Linear.apply(x, W, res)
