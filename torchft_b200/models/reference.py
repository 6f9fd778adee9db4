"""Plain-PyTorch reference of the Llama forward/backward (test oracle only), in fp32 by default.

Numerics tests compare every hand-written kernel path in ``models/llama.py``
against this eager implementation, which shares nothing with it except the
parameter tensors. In fp64 it is the exact model; in bf16 it is an independent
implementation at the fused model's precision.
"""

from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch
import torch.nn.functional as F


def _rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def _scaled(inv: torch.Tensor, scaling, dtype: torch.dtype) -> torch.Tensor:
    """Llama-3.1 frequency scaling of ``inv`` computed in ``dtype`` (at least fp32): a wavelength ``w = 2 pi / f`` below
    ``orig / high`` keeps ``f``, one above ``orig / low`` gets ``f / factor``, and in between ``f`` moves smoothly
    from one to the other with ``s = (orig / w - low) / (high - low)``."""
    factor, low, high, orig = (float(v) for v in scaling)
    f = inv.to(torch.float64 if dtype == torch.float64 else torch.float32)
    w = 2 * torch.pi / f
    out = f.clone()
    long_waves = w > orig / low
    out[long_waves] = f[long_waves] / factor
    band = (w >= orig / high) & ~long_waves
    s = (orig / w[band] - low) / (high - low)
    out[band] = (1 - s) * f[band] / factor + s * f[band]
    return out


def _rope(x: torch.Tensor, theta: float, pos: Optional[torch.Tensor] = None, scaling=None) -> torch.Tensor:
    """Interleaved-pair rotation by the fp32 angles of ``ops.fused.rope_table``; cos and sin in fp64 for an fp64 ``x``,
    else in fp32, and the rotation rounded once to ``x``'s dtype (complex bf16 does not exist). ``pos`` ``[B, S]``: the
    position of each token (default: its offset in its row). ``scaling``: Llama-3.1 frequency scaling, computed in
    ``x``'s dtype (at least fp32); the angles are then the fp32 products of the scaled frequencies, as in the table."""
    B, S, H, D = x.shape
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, device=x.device, dtype=torch.float32) / D))
    if scaling is not None:
        inv = _scaled(inv, scaling, x.dtype).float()
    if pos is None:
        ang = torch.outer(torch.arange(S, device=x.device, dtype=torch.float32), inv)[None]
    else:
        ang = pos.to(x.device, torch.float32)[..., None] * inv  # [B, S, D/2], the same fp32 products as the table's
    if x.dtype in (torch.float32, torch.float64):
        a = ang.to(x.dtype)
        f = torch.polar(torch.ones_like(a), a)
        xc = torch.view_as_complex(x.reshape(B, S, H, D // 2, 2))
        return torch.view_as_real(xc * f[:, :, None, :]).reshape(B, S, H, D)
    c, s = ang.cos()[:, :, None, :], ang.sin()[:, :, None, :]
    x0, x1 = x.float().reshape(B, S, H, D // 2, 2).unbind(-1)
    return torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), -1).reshape(B, S, H, D).to(x.dtype)


def _matmul_t(x: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    return x @ W.t()


def _document_mask_and_positions(cu_seqlens: torch.Tensor, B: int, S: int, device: torch.device
                                 ) -> Tuple[torch.Tensor, torch.Tensor]:
    """From a ``cu_seqlens`` over the ``B*S`` flattened tokens: the boolean attention mask ``[B, 1, S, S]`` (query i
    sees key j iff both lie in the same document and j <= i) and each token's offset in its document ``[B, S]``."""
    t = torch.arange(B * S, device=device)
    cu = cu_seqlens.to(device=device, dtype=torch.int64)
    doc = torch.bucketize(t, cu[1:], right=True)  # index of t's document
    pos = (t - cu[doc]).view(B, S)
    doc = doc.view(B, S)
    same = doc[:, :, None] == doc[:, None, :]
    causal = torch.ones(S, S, dtype=torch.bool, device=device).tril()
    return (same & causal)[:, None], pos


def reference_loss(model, tokens: torch.Tensor, targets: torch.Tensor, dtype: torch.dtype = torch.float32,
                   linear: Optional[Callable[[torch.Tensor, torch.Tensor], torch.Tensor]] = None,
                   cu_seqlens: Optional[torch.Tensor] = None) -> Tuple[float, Dict[str, torch.Tensor]]:
    """Returns (loss, {param_name: grad in ``dtype``}) computed with eager PyTorch in ``dtype``. ``linear(x, W)``, by
    default ``x @ W.T``, computes the four block linears (wqkv, wo, w13, w2), e.g. with quantised operands.
    ``cu_seqlens``: packed documents, attended through an explicit block-diagonal causal mask and rotated by their
    positions in their documents. A config with ``tie_embeddings`` reads ``tok_embeddings`` as the head (autograd adds
    both gradients), and one with ``rope_scaling`` rotates by the scaled frequencies."""

    cfg = model.cfg
    if linear is None:
        linear = _matmul_t
    P = {n: p.detach().to(dtype).requires_grad_() for n, p in model.named_parameters()}
    B, S = tokens.shape
    mask, pos = _document_mask_and_positions(cu_seqlens, B, S, tokens.device) if cu_seqlens is not None else (None, None)
    x = F.embedding(tokens, P["tok_embeddings"])
    Hq, Hkv, D = cfg.n_heads, cfg.n_kv_heads, cfg.head_dim
    for i in range(cfg.n_layers):
        pre = f"layers.{i}."
        n = _rmsnorm(x, P[pre + "attention_norm"], cfg.norm_eps)
        qkv = linear(n, P[pre + "wqkv"]).view(B, S, Hq + 2 * Hkv, D)
        q, k, v = qkv[:, :, :Hq], qkv[:, :, Hq : Hq + Hkv], qkv[:, :, Hq + Hkv :]
        q, k = _rope(q, cfg.rope_theta, pos, cfg.rope_scaling), _rope(k, cfg.rope_theta, pos, cfg.rope_scaling)
        rep = Hq // Hkv
        k = k.repeat_interleave(rep, dim=2)
        v = v.repeat_interleave(rep, dim=2)
        if mask is None:
            o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True)
        else:
            o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=mask)
        o = o.transpose(1, 2).reshape(B, S, cfg.dim)
        h = x + linear(o, P[pre + "wo"])
        n2 = _rmsnorm(h, P[pre + "ffn_norm"], cfg.norm_eps)
        gu = linear(n2, P[pre + "w13"])
        a = F.silu(gu[..., : cfg.ffn_dim]) * gu[..., cfg.ffn_dim :]
        x = h + linear(a, P[pre + "w2"])
    hfin = _rmsnorm(x, P["norm"], cfg.norm_eps)
    logits = hfin @ P["tok_embeddings" if cfg.tie_embeddings else "output"].t()
    loss = F.cross_entropy(logits.view(B * S, -1), targets.reshape(-1))
    loss.backward()
    return float(loss.item()), {n: p.grad for n, p in P.items()}
