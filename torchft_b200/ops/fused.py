"""Autograd wrappers over the hand-written sm_90a model kernels.

RMSNorm / SwiGLU / RoPE / chunked linear-cross-entropy / flat AdamW. All take
bf16 CUDA tensors, reduce in fp32 and make one pass over HBM per direction.
There is no PyTorch fallback: on a CUDA box these always run ``_K`` kernels.
"""

from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np
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


# ------------------------------------------------------------------------------------------------- fp8 operands
# The fp8 block linears run rowwise torch._scaled_mm: a e4m3 row-major with one fp32 scale per row ([M, 1]), b e4m3
# column-major with one scale per column ([1, N]), fp32 accumulation (use_fast_accum=False), bf16 output. Scales are
# powers of two computed from the tensor at hand on every call (csrc/kernels/fp8.cuh), so there is no scaling state.
E4M3 = torch.float8_e4m3fn


def fp8_rows(x2: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 ``[R, C]`` (any row stride, unit column stride) -> (e4m3 ``[R, C]``, fp32 scale ``[R, 1]``), one scale per
    row. ``C`` must be a multiple of 16 and the rows 16-byte aligned."""
    K = _native.load()
    _chk(x2, "x")
    if x2.dim() != 2 or x2.stride(1) != 1:
        raise ValueError(f"fp8_rows takes a 2-D tensor with unit column stride, got shape {tuple(x2.shape)} strides {x2.stride()}")
    R, C = x2.shape
    q = torch.empty((R, C), dtype=E4M3, device=x2.device)
    scale = torch.empty((R, 1), dtype=torch.float32, device=x2.device)
    K.fp8_rows(x2.data_ptr(), x2.stride(0), q.data_ptr(), scale.data_ptr(), R, C, _native.stream_ptr())
    return q, scale


def fp8_cols_t(W: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 ``W [N, K]`` -> (e4m3 ``W^T [K, N]``, fp32 scale ``[1, K]``), one scale per column of ``W``: ``q.t()`` is the
    column-major ``[N, K]`` operand of the input-gradient GEMM ``dy @ W``."""
    K_ = _native.load()
    W = W.contiguous()
    _chk(W, "W")
    N, Kd = W.shape
    q = torch.empty((Kd, N), dtype=E4M3, device=W.device)
    scale = torch.empty((1, Kd), dtype=torch.float32, device=W.device)
    ws = torch.empty(Kd, dtype=torch.int32, device=W.device)
    K_.fp8_cols_t(W.data_ptr(), N, Kd, q.data_ptr(), scale.data_ptr(), ws.data_ptr(), _native.stream_ptr())
    return q, scale


def _mm_fp8(a: Tuple[torch.Tensor, torch.Tensor], b: Tuple[torch.Tensor, torch.Tensor]) -> torch.Tensor:
    """``a @ b`` of a quantised ``(e4m3 [M, K], scale [M, 1])`` and ``(e4m3 [K, N] column-major, scale [1, N])``."""
    return torch._scaled_mm(a[0], b[0], scale_a=a[1], scale_b=b[1], out_dtype=torch.bfloat16, use_fast_accum=False)


def _fwd_fp8(a: Tuple[torch.Tensor, torch.Tensor], W: torch.Tensor) -> torch.Tensor:
    """Forward GEMM ``a @ W^T``: W quantised per output channel (per row), its row-major copy seen as W^T."""
    qw, sw = fp8_rows(W)
    return _mm_fp8(a, (qw.t(), sw.view(1, -1)))


def _dgrad_fp8(dy2: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """Input-gradient GEMM ``dy @ W``: dy per token row, W per input channel (per column) from its transposed copy."""
    qt, st = fp8_cols_t(W)
    return _mm_fp8(fp8_rows(_rows_ok(dy2)), (qt.t(), st))


def _rows_ok(t: torch.Tensor) -> torch.Tensor:
    """``t`` itself when fp8_rows can read it in place (unit column stride, 16-byte aligned rows), else a copy."""
    ok = t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0
    return t if ok else t.contiguous()


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


def rope_scaled_frequencies(inv: torch.Tensor, scaling: Tuple[float, float, float, int]) -> torch.Tensor:
    """Llama-3.1 frequency scaling of the fp32 inverse frequencies ``inv``, computed in fp64 and rounded once to fp32.
    ``scaling = (factor, low_freq_factor, high_freq_factor, original_max_position)``. With ``w = 2 pi / f``: ``w <
    orig / high`` keeps ``f``; ``w > orig / low`` gives ``f / factor``; in between, with ``s = (orig / w - low) / (high -
    low)``, ``(1 - s) f / factor + s f``."""
    factor, low, high, orig = (float(x) for x in scaling)
    f = inv.double()
    w = 2 * math.pi / f
    s = (orig / w - low) / (high - low)
    out = torch.where(w < orig / high, f, torch.where(w > orig / low, f / factor, (1 - s) * f / factor + s * f))
    return out.float()


def rope_table(seq_len: int, head_dim: int, theta: float, device: torch.device,
               scaling: Optional[Tuple[float, float, float, int]] = None) -> torch.Tensor:
    """(cos, sin) table ``[seq_len, head_dim/2, 2]`` fp32 for interleaved-pair RoPE. ``scaling``: Llama-3.1 frequency
    scaling ``(factor, low_freq_factor, high_freq_factor, original_max_position)`` (:func:`rope_scaled_frequencies`)."""

    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=device) / head_dim))
    if scaling is not None:
        inv = rope_scaled_frequencies(inv, scaling)
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
    def forward(ctx, qkv: torch.Tensor, cs: torch.Tensor, B: int, S: int, Hq: int, Hkv: int, D: int,  # type: ignore[override]
                positions: Optional[torch.Tensor] = None):
        K = _native.load()
        assert qkv.is_contiguous() and qkv.dtype == torch.bfloat16
        # the kernel reads the table as fp32: a wrapper that down-casts module inputs (FSDP2's cast_forward_inputs) would
        # make it read garbage and past the end of the buffer
        assert cs.dtype == torch.float32 and cs.is_contiguous() and cs.shape[0] >= S, "rope table must be the fp32 table of rope_table()"
        if positions is not None:
            # every entry must index the table: data.document_positions of a valid cu_seqlens is < S
            assert (positions.dtype == torch.int32 and positions.is_contiguous() and positions.device == qkv.device
                    and positions.numel() == B * S), "positions must be a contiguous int32 [B*S] tensor on qkv's device"
        row = qkv.shape[-1]
        assert row == (Hq + 2 * Hkv) * D
        q = torch.empty((B, S, Hq, D), dtype=qkv.dtype, device=qkv.device)
        k = torch.empty((B, S, Hkv, D), dtype=qkv.dtype, device=qkv.device)
        pp = positions.data_ptr() if positions is not None else 0
        # one launch rotates q and k out of the packed rows; v stays a strided view of the projection (no copy)
        K.rope_qkv(qkv.data_ptr(), row, q.data_ptr(), k.data_ptr(), 0, [*q.stride()[:3], *k.stride()[:3], 0, 0, 0],
                   cs.data_ptr(), B * S, S, D, Hq, Hkv, 0, _native.stream_ptr(), pp)
        v = qkv.view(B * S, row)[:, (Hq + Hkv) * D :].reshape(B, S, Hkv, D)
        ctx.save_for_backward(cs, positions)
        ctx.meta = (B, S, Hq, Hkv, D, row)
        return q, k, v

    @staticmethod
    def backward(ctx, dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        cs, positions = ctx.saved_tensors
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
                   _native.stream_ptr(), positions.data_ptr() if positions is not None else 0)
        return dqkv, None, None, None, None, None, None, None


def rope_qkv(qkv: torch.Tensor, cs: torch.Tensor, B: int, S: int, Hq: int, Hkv: int, D: int,
             positions: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Split a packed ``[B*S, (Hq+2*Hkv)*D]`` projection into q, k, v with RoPE applied to q and k. Token ``t`` is
    rotated by ``cs[positions[t]]`` when ``positions`` (int32 ``[B*S]`` on the device, e.g. each token's offset in its
    packed document) is given, else by ``cs[t mod S]``; the backward uses the same positions."""
    return _RoPEQKV.apply(qkv, cs, B, S, Hq, Hkv, D, positions)


class _LinearCrossEntropy(torch.autograd.Function):
    """loss = mean CE(h @ W^T, target) without materialising fp32 logits.

    Tokens are processed in chunks: bf16 logits chunk (cuBLAS) -> fused
    softmax/CE kernel that overwrites the chunk with dlogits -> dh chunk and dW
    accumulation (cuBLAS). Peak extra memory = one bf16 logits chunk.
    """

    @staticmethod
    def forward(ctx, h: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, chunk: int, ignore_index: int,  # type: ignore[override]
                count_valid: bool, tied: bool = False):
        T = h.shape[0]
        # count_valid: divide by the number of non-ignored targets, counted on the device (no host sync). The kernels
        # keep grad_scale = 1/T and scale it by the device factor T / n_valid, which is exactly 1.0 when no target is
        # ignored, so that case is bit-identical to count_valid=False (divide by T).
        scale = None
        if count_valid:
            n_valid = (target != ignore_index).sum().clamp_(min=1).float()
            scale = torch.full((), float(T), dtype=torch.float32, device=h.device).div_(n_valid)
        need_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        slot = getattr(weight, "_flat_grad", None)
        losses = torch.empty(T, dtype=torch.float32, device=h.device)
        ctx.tied = None
        if tied:
            link = getattr(weight, "_tied_link", None)
            if link is None or link.mode is not None:
                raise RuntimeError("a tied head needs the weight's tied_embedding node earlier in the same forward")
            if need_grad and slot is not None and weight.grad is not None and weight.grad.data_ptr() == slot.data_ptr():
                # the slot already holds a gradient (reset_grads(zero=True)): the head's dW must be added to it times
                # the upstream scale, which only backward knows, so backward recomputes the chunks (no [V, d] buffer)
                _xent_chunks(h, weight, target, chunk, ignore_index, scale, losses, None, None)
                ctx.save_for_backward(h, weight, target, scale)
                ctx.meta = (chunk, ignore_index)
                link.mode, link.buf = "accumulate", slot.view(weight.shape)
                ctx.tied = link
                loss = losses.sum() / max(T, 1)
                return loss * scale if scale is not None else loss
        dh = torch.empty_like(h) if need_grad else None
        direct = need_grad and slot is not None and weight.grad is None
        dW = (slot.view(weight.shape).zero_() if direct else torch.zeros_like(weight)) if need_grad else None
        ctx.direct = direct
        _xent_chunks(h, weight, target, chunk, ignore_index, scale, losses, dh, dW)
        if tied and need_grad:
            # the embedding node adds its part into dW and hands autograd the sum: the weight's only gradient
            link.mode, link.buf = ("direct" if direct else "own"), dW
            ctx.tied = link
            ctx.save_for_backward(dh)
        else:
            ctx.save_for_backward(dh, dW)
        ctx.need = need_grad
        loss = losses.sum() / max(T, 1)
        return loss * scale if scale is not None else loss

    @staticmethod
    def backward(ctx, g: torch.Tensor):  # type: ignore[override]
        link = ctx.tied
        if link is not None and link.mode == "accumulate":
            h, weight, target, scale = ctx.saved_tensors
            chunk, ignore_index = ctx.meta
            # the upstream scalar rides in the cross-entropy kernel's device factor: dlogits come out scaled by it
            gs = g.float() if scale is None else scale * g.float()
            dh = torch.empty_like(h)
            losses = torch.empty(h.shape[0], dtype=torch.float32, device=h.device)
            _xent_chunks(h, weight, target, chunk, ignore_index, gs, losses, dh, link.buf)
            return dh, None, None, None, None, None, None
        if link is not None:
            (dh,) = ctx.saved_tensors
            link.buf.mul_(g.to(link.buf.dtype))
            return dh * g.to(dh.dtype), None, None, None, None, None, None
        dh, dW = ctx.saved_tensors
        # g is the upstream scalar (1.0 for a plain loss.backward()); fold it in
        # without a host sync.
        # (dW already sits in the flat gradient buffer when ctx.direct; scale in place)
        return (dh * g.to(dh.dtype), (dW.mul_(g.to(dW.dtype)) if ctx.direct else dW * g.to(dW.dtype)), None, None, None,
                None, None)


def _xent_chunks(h: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, chunk: int, ignore_index: int,
                 scale: Optional[torch.Tensor], losses: torch.Tensor, dh: Optional[torch.Tensor],
                 dW: Optional[torch.Tensor]) -> None:
    """The chunk loop of :class:`_LinearCrossEntropy`: per chunk the bf16 logits (cuBLAS), the fused softmax/CE kernel
    that overwrites them with dlogits (``1/T`` times the device factor ``scale``), then ``dh = dlogits @ W`` and ``dW +=
    dlogits^T h`` when ``dh`` is given."""
    K = _native.load()
    T, V = h.shape[0], weight.shape[0]
    sp = _native.stream_ptr()
    for lo in range(0, T, chunk):
        hi = min(lo + chunk, T)
        hc = h[lo:hi]
        logits = hc @ weight.t()  # [c, V] bf16, cuBLAS
        K.xent(
            logits.data_ptr(), target[lo:hi].data_ptr(), losses[lo:hi].data_ptr(), hi - lo, V,
            logits.stride(0), 1.0 / max(T, 1), ignore_index, sp, scale.data_ptr() if scale is not None else 0,
        )
        if dh is not None:
            torch.mm(logits, weight, out=dh[lo:hi])
            dW.addmm_(logits.t(), hc)
        del logits


def linear_cross_entropy(h: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, chunk: int = 2048,
                         ignore_index: int = -100, count_valid: bool = True, tied: bool = False) -> torch.Tensor:
    """Mean cross entropy of ``h @ weight.T`` against ``target`` (int64).

    With ``count_valid`` (the default) the mean is over targets that are not ``ignore_index``, counted on the device
    without a host sync; with ``count_valid=False`` the sum is divided by the number of rows.

    ``tied``: ``weight`` is also the token embedding, read earlier in the same forward through :func:`tied_embedding`.
    This node then returns no gradient for ``weight``: it leaves its part in the buffer that the embedding node adds into
    and hands to autograd, so the weight gets ONE gradient (one post-accumulate-grad event) after both parts. In a
    ``FlatParams`` buffer with the gradient dropped that buffer is the weight's flat slot, written here during the
    forward as the untied head does; with a zeroed slot (``reset_grads(zero=True)``) backward recomputes the chunks and
    adds into the slot; without a flat slot it is a new zeroed gradient."""
    assert h.dim() == 2 and target.dim() == 1 and h.shape[0] == target.shape[0]
    return _LinearCrossEntropy.apply(h.contiguous(), weight, target.contiguous(), chunk, ignore_index, count_valid, tied)


class _TiedLink:
    """What the tied head of one forward left for the embedding node's backward: ``mode`` ``None`` (no tied head ran),
    ``"direct"`` (``buf`` is the flat slot, holding the head's part only), ``"own"`` (``buf`` is a new gradient holding
    the head's part) or ``"accumulate"`` (``buf`` is the flat slot, which is ``p.grad`` and already holds everything
    else)."""

    __slots__ = ("mode", "buf")

    def __init__(self) -> None:
        self.mode: Optional[str] = None
        self.buf: Optional[torch.Tensor] = None


def embedding_bwd(ids: torch.Tensor, dx: torch.Tensor, grad: torch.Tensor) -> torch.Tensor:
    """``grad[v] = bf16(grad[v] + sum of dx[t] over the tokens t with ids[t] = v)`` in place, for every id that occurs;
    the sum is fp32 with one rounding per touched row, and its order depends on the ids alone (bit-identical launches).
    ``ids`` int64 ``[T]`` (any shape, flattened; ids must be in ``[0, V)``, which ``F.embedding`` checked in forward),
    ``dx`` bf16 ``[T, d]`` with unit column stride and 16-byte aligned rows, ``grad`` a contiguous bf16 ``[V, d]``.
    The ids are sorted stably on the current stream (no host sync). Returns ``grad``."""
    K = _native.load()
    if dx.dim() != 2 or grad.dim() != 2 or dx.shape[1] != grad.shape[1]:
        raise ValueError(f"embedding_bwd takes dx [T, d] and grad [V, d], got {tuple(dx.shape)} and {tuple(grad.shape)}")
    T, d = dx.shape
    if d % 8:
        raise ValueError(f"embedding_bwd: the row width must be a multiple of 8, got {d}")
    if ids.dtype != torch.int64 or ids.numel() != T or ids.device != dx.device:
        raise ValueError(f"embedding_bwd: ids must be {T} int64 values on {dx.device}")
    _chk(grad, "grad")
    _chk(dx, "dx")
    if not grad.is_contiguous() or dx.stride(1) != 1 or dx.stride(0) % 8:
        raise ValueError("embedding_bwd: grad must be contiguous and dx rows 16-byte aligned with unit column stride")
    if T == 0:
        return grad
    sid, perm = torch.sort(ids.reshape(-1), stable=True)
    partial = torch.empty((K.embedding_bwd_pieces(T), 2, d), dtype=torch.float32, device=dx.device)
    K.embedding_bwd(sid.data_ptr(), perm.data_ptr(), dx.data_ptr(), dx.stride(0), grad.data_ptr(), partial.data_ptr(),
                    T, d, _native.stream_ptr())
    return grad


# adding -0.0 is the identity on every bf16 value, -0.0 included
_NEG_ZERO = {}


class _TiedEmbedding(torch.autograd.Function):
    """``F.embedding(tokens, W)`` whose backward adds the token gradients into the tied weight's gradient buffer in place
    with :func:`embedding_bwd` (see :func:`linear_cross_entropy` ``tied``)."""

    @staticmethod
    def forward(ctx, tokens: torch.Tensor, W: torch.Tensor) -> torch.Tensor:  # type: ignore[override]
        link = _TiedLink()
        W._tied_link = link  # the tied head of this forward finds it here
        ctx.link = link
        ctx.save_for_backward(tokens, W)
        return torch.nn.functional.embedding(tokens, W)

    @staticmethod
    def backward(ctx, dx: torch.Tensor):  # type: ignore[override]
        tokens, W = ctx.saved_tensors
        link = ctx.link
        d = W.shape[1]
        dx2 = _rows_ok(dx.reshape(-1, d))
        mode, buf = link.mode, link.buf
        link.buf = None  # the buffer handed to autograd must have no other owner, or AccumulateGrad copies it
        if mode is None:  # no tied head in this forward (e.g. the logits path): the embedding's own gradient
            buf = torch.zeros_like(W)
        embedding_bwd(tokens, dx2, buf)
        if mode == "accumulate":
            # p.grad IS the slot and now holds the whole sum; autograd still owes the weight its one event, so it gets
            # a stride-0 -0.0 (no [V, d] allocation) whose in-place add leaves every bit as it is
            key = (W.device, W.dtype)
            if key not in _NEG_ZERO:
                _NEG_ZERO[key] = torch.full((), -0.0, dtype=W.dtype, device=W.device)
            return None, _NEG_ZERO[key].expand(W.shape)
        # "direct": the slot view the head wrote (AccumulateGrad adopts it without a copy); else a gradient of our own
        return None, buf


def tied_embedding(tokens: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """Token embedding of a model whose LM head is ``W`` too (``linear_cross_entropy(..., tied=True)``): the forward is
    ``F.embedding`` (its bounds check is the one check on the ids), the backward the in-place :func:`embedding_bwd`."""
    return _TiedEmbedding.apply(tokens, W)


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
        bc1, bc2 = self._bias_corrections()
        K.adamw(
            self.p.data_ptr(), self.master.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.g.data_ptr(),
            self.p.numel(), lr, b1, b2, self.eps, self.weight_decay, bc1, bc2,
            grad_scale, gate.data_ptr() if gate is not None else 0, _native.stream_ptr(),
        )

    def _bias_corrections(self) -> Tuple[float, float]:
        """1 - b^t of the fp32 betas the kernel's moving averages use (fp64 here, rounded to fp32 by the binding): at
        b2 = 0.999 the double beta's 1 - b^t is hundreds of fp32 ulps away from the fp32 beta's."""
        return tuple(1.0 - float(np.float32(b)) ** self.t for b in self.betas)

    def step_ranges(self, ranges, streams_events, grad_scale: float = 1.0, gate: Optional[torch.Tensor] = None,
                    max_blocks: int = 0) -> None:
        """The same update as :meth:`step`, cut into element ranges ``[(lo, hi), ...]`` that are launched
        in the given order on ``stream``; ``events[i]`` is recorded after range ``i``. Lets the next
        forward start on the first layers while the (HBM-bound) update of later layers is still running
        underneath the (tensor-core-bound) GEMMs. ``streams_events`` = ``(stream, events)``."""
        K = _native.load()
        stream, events = streams_events
        # the kernel's 16-byte vector path needs p + 2*lo to be 16-byte aligned
        bad = [lo for lo, _ in ranges if lo % 8]
        if bad:
            raise ValueError(f"step_ranges: range starts must be multiples of 8 elements, got {bad}")
        self.t += 1
        lr = self.param_groups[0]["lr"]
        b1, b2 = self.betas
        bc1, bc2 = self._bias_corrections()
        gp = gate.data_ptr() if gate is not None else 0
        p, w, m, v, g = (t.data_ptr() for t in (self.p, self.master, self.m, self.v, self.g))
        for (lo, hi), ev in zip(ranges, events):
            K.adamw(p + 2 * lo, w + 4 * lo, m + 4 * lo, v + 4 * lo, g + 2 * lo, hi - lo, lr, b1, b2, self.eps,
                    self.weight_decay, bc1, bc2, grad_scale, gp, stream.cuda_stream, max_blocks)
            ev.record(stream)

    def state_dict(self) -> dict:
        return {"t": self.t, "master": self.master, "m": self.m, "v": self.v}

    def load_state_dict(self, sd: dict) -> None:
        self.t = int(sd["t"])
        self.master.copy_(sd["master"])
        self.m.copy_(sd["m"])
        self.v.copy_(sd["v"])
        self.p.copy_(self.master)


class _NormLinearRes(torch.autograd.Function):
    """Pre-norm residual branch point: returns ``(x, rmsnorm(x, g) @ W^T)``.

    The first output IS ``x`` (the residual stream, to be consumed by the ``res=`` argument of
    :func:`linear` / :func:`swiglu_linear`). Routing the residual through this node means its
    gradient arrives here together with the branch gradient, and the RMSNorm backward kernel adds
    it while writing ``dx`` — autograd's separate ``dres + dbranch`` accumulation pass
    (3 x 64 MB of HBM traffic per norm at 8k x 4096) disappears.

    Of the activations only ``(x, rstd)`` is saved: the normalised activation is recomputed in backward by one extra
    RMSNorm pass instead of living in HBM for the whole forward/backward (64 MB per call at 8k x 4096).

    With ``fp8`` the RMSNorm kernel writes the normalised activation as e4m3 with a scale per row (never as bf16), and
    the forward and input-gradient GEMMs run on fp8 tensor cores; the weight gradient stays the bf16 GEMM.
    """

    @staticmethod
    def forward(ctx, x: torch.Tensor, g: torch.Tensor, W: torch.Tensor, eps: float, fp8: bool = False):  # type: ignore[override]
        K = _native.load()
        x = x.contiguous()
        H = x.shape[-1]
        rows = x.numel() // H
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        if fp8:
            q = torch.empty((rows, H), dtype=E4M3, device=x.device)
            qs = torch.empty((rows, 1), dtype=torch.float32, device=x.device)
            K.rmsnorm_fwd_fp8(x.data_ptr(), g.data_ptr(), q.data_ptr(), qs.data_ptr(), rstd.data_ptr(), rows, H, eps,
                              _native.stream_ptr())
            y = _fwd_fp8((q, qs), W)
        else:
            n = torch.empty_like(x)
            K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), rows, H, eps, _native.stream_ptr())
            y = n.view(rows, H) @ W.t()
        ctx.save_for_backward(x, g, W, rstd)
        ctx.eps = eps
        ctx.fp8 = fp8
        return x, y.view(x.shape[:-1] + (W.shape[0],))  # autograd re-wraps the returned input as a new node output

    @staticmethod
    def backward(ctx, dres: Optional[torch.Tensor], dy: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        x, g, W, rstd = ctx.saved_tensors
        H = x.shape[-1]
        rows = x.numel() // H
        sp = _native.stream_ptr()
        dy2 = dy.reshape(rows, W.shape[0])
        n = torch.empty_like(x)
        K.rmsnorm_fwd(x.data_ptr(), g.data_ptr(), n.data_ptr(), rstd.data_ptr(), rows, H, ctx.eps, sp)
        dW = _wgrad(dy2, n.view(rows, H), W)
        dn = _dgrad_fp8(dy2, W) if ctx.fp8 else dy2 @ W
        dx = n  # reuse the recompute buffer for dx
        grid = K.rmsnorm_bwd_grid(rows)
        partial = torch.empty((grid, H), dtype=torch.float32, device=x.device)
        dg = torch.empty_like(g)
        if dres is not None:
            dres = dres.contiguous()
            assert dres.dtype == x.dtype and dres.numel() == x.numel()
        K.rmsnorm_bwd(dn.data_ptr(), x.data_ptr(), g.data_ptr(), rstd.data_ptr(), dx.data_ptr(),
                      partial.data_ptr(), dg.data_ptr(), False, rows, H, sp, dres.data_ptr() if dres is not None else 0)
        return dx, dg, dW, None, None


def norm_linear_res(x: torch.Tensor, norm_weight: torch.Tensor, W: torch.Tensor, eps: float = 1e-5,
                    fp8: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(x, rmsnorm(x, norm_weight) @ W.T)`` with the normalised activation recomputed in backward. The first output
    is the residual stream, handed back so that its gradient is accumulated inside the RMSNorm backward kernel.
    ``fp8``: the forward and input-gradient GEMMs take row-scaled e4m3 operands (the weight gradient stays bf16)."""
    return _NormLinearRes.apply(x, norm_weight, W, eps, fp8)


class _SwiGLULinear(torch.autograd.Function):
    """out = swiglu(gu) @ W2^T saving only gu (the [T, F] product is recomputed). With ``fp8`` the SwiGLU kernel writes
    the product as e4m3 with a scale per row (never as bf16) for the fp8 forward GEMM."""

    @staticmethod
    def forward(ctx, gu: torch.Tensor, W2: torch.Tensor, res: Optional[torch.Tensor], fp8: bool = False) -> torch.Tensor:  # type: ignore[override]
        K = _native.load()
        gu = gu.contiguous()
        F2 = gu.shape[-1]
        F = F2 // 2
        T = gu.numel() // F2
        if fp8:
            _chk(gu, "gate_up")
            q = torch.empty((T, F), dtype=E4M3, device=gu.device)
            qs = torch.empty((T, 1), dtype=torch.float32, device=gu.device)
            K.fp8_swiglu(gu.data_ptr(), q.data_ptr(), qs.data_ptr(), T, F, _native.stream_ptr())
            out = _fwd_fp8((q, qs), W2)
            if res is not None:
                # _scaled_mm has no beta epilogue: the residual costs one elementwise pass here
                out.add_(res.reshape(T, W2.shape[0]))
        else:
            a = torch.empty((T, F), dtype=gu.dtype, device=gu.device)
            K.swiglu_fwd(gu.data_ptr(), a.data_ptr(), T, F, _native.stream_ptr())
            # residual add rides in the GEMM epilogue (beta = 1) instead of a separate elementwise pass
            out = a @ W2.t() if res is None else torch.addmm(res.reshape(T, W2.shape[0]), a, W2.t())
        ctx.save_for_backward(gu, W2)
        ctx.has_res = res is not None
        ctx.fp8 = fp8
        return out.view(gu.shape[:-1] + (W2.shape[0],))

    @staticmethod
    def backward(ctx, dout: torch.Tensor):  # type: ignore[override]
        K = _native.load()
        gu, W2 = ctx.saved_tensors
        F2 = gu.shape[-1]
        F = F2 // 2
        T = gu.numel() // F2
        sp = _native.stream_ptr()
        d2 = dout.reshape(T, W2.shape[0])
        a = torch.empty((T, F), dtype=gu.dtype, device=gu.device)
        K.swiglu_fwd(gu.data_ptr(), a.data_ptr(), T, F, sp)
        dW2 = _wgrad(d2, a, W2)
        da = _dgrad_fp8(d2, W2) if ctx.fp8 else torch.mm(d2, W2, out=a)  # bf16: reuse buffer
        dgu = torch.empty_like(gu)
        K.swiglu_bwd(da.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, F, sp)
        return dgu, dW2, (dout if ctx.has_res else None), None


def swiglu_linear(gate_up: torch.Tensor, W2: torch.Tensor, res: Optional[torch.Tensor] = None,
                  fp8: bool = False) -> torch.Tensor:
    """``(silu(gate) * up) @ W2.T (+ res)`` with the activation product recomputed in backward. ``fp8``: the forward and
    input-gradient GEMMs take row-scaled e4m3 operands (the weight gradient stays bf16)."""
    return _SwiGLULinear.apply(gate_up, W2, res, fp8)


class _Linear(torch.autograd.Function):
    """y = x @ W^T whose weight gradient is written straight into the flat gradient buffer."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, W: torch.Tensor, res: Optional[torch.Tensor], fp8: bool = False) -> torch.Tensor:  # type: ignore[override]
        ctx.save_for_backward(x, W)
        ctx.has_res = res is not None
        ctx.fp8 = fp8
        if fp8:
            x2 = x.reshape(-1, x.shape[-1])
            y = _fwd_fp8(fp8_rows(_rows_ok(x2)), W)
            if res is not None:
                # _scaled_mm has no beta epilogue: the residual costs one elementwise pass here
                y.add_(res.reshape(x2.shape[0], W.shape[0]))
            return y.view(x.shape[:-1] + (W.shape[0],))
        if res is None:
            return x @ W.t()
        x2 = x.reshape(-1, x.shape[-1])
        return torch.addmm(res.reshape(x2.shape[0], W.shape[0]), x2, W.t()).view(x.shape[:-1] + (W.shape[0],))

    @staticmethod
    def backward(ctx, dy: torch.Tensor):  # type: ignore[override]
        x, W = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dW = _wgrad(dy2, x.reshape(-1, x.shape[-1]), W)
        dx = _dgrad_fp8(dy2, W) if ctx.fp8 else dy2 @ W
        return dx.view(x.shape), dW, (dy if ctx.has_res else None), None


def linear(x: torch.Tensor, W: torch.Tensor, res: Optional[torch.Tensor] = None, fp8: bool = False) -> torch.Tensor:
    """``x @ W.T (+ res)`` with the wgrad GEMM writing directly into the flat gradient bucket; the
    residual add, when given, is the GEMM's beta=1 epilogue. ``fp8``: the forward and input-gradient GEMMs take
    row-scaled e4m3 operands (the weight gradient stays bf16) and the residual is a separate add."""
    return _Linear.apply(x, W, res, fp8)
