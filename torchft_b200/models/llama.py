"""Llama-3 family decoder for the fault-tolerant training benchmarks.

The reference ships no model: its flagship config (BASELINE.json, "Llama-3 8B
fault-tolerant HSDP bf16") borrows torchtitan's. This is our own implementation,
laid out for one-GPU-per-replica training in the 80 GB of an H100:

* every parameter is a view into ONE flat bf16 buffer and every gradient a view
  into ONE flat bf16 gradient buffer that can live in NVLink-symmetric memory,
  so the cross-replica all-reduce kernel reads gradients in place (zero copy)
  and AdamW is a single launch over the whole model;
* q/k/v and gate/up projections are fused GEMMs (cuBLAS);
* RMSNorm, RoPE(+qkv split), SwiGLU, softmax-cross-entropy and AdamW are
  hand-written sm_90a kernels (``torchft_b200/csrc/kernels/model_ops.cu``);
* normalised activations and the SwiGLU product are recomputed in backward
  instead of stored (see ``ops.fused.norm_linear`` / ``swiglu_linear``);
* attention is the SDPA library kernel (flash / cuDNN), causal, GQA.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from torchft_b200.ops import fused


@dataclass
class LlamaConfig:
    """Architecture hyper-parameters (defaults = Llama-3-8B) plus the activation-checkpoint policy and the loss chunk size."""

    dim: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int = 8
    vocab_size: int = 128256
    ffn_dim: int = 14336
    norm_eps: float = 1e-5
    rope_theta: float = 500000.0
    max_seq_len: int = 8192
    # "none": keep activations (fused recompute only); "full": checkpoint every block
    activation_checkpoint: str = "none"
    loss_chunk: int = 2048

    @property
    def head_dim(self) -> int:
        return self.dim // self.n_heads

    def num_params(self) -> int:
        d, f, v = self.dim, self.ffn_dim, self.vocab_size
        qkv = (self.n_heads + 2 * self.n_kv_heads) * self.head_dim * d
        per_layer = qkv + d * d + 2 * f * d + f * d + 2 * d
        return 2 * v * d + self.n_layers * per_layer + d

    def flops_per_token(self, seq_len: int) -> float:
        """Training FLOPs/token: 6 * matmul params + causal attention (fwd+bwd)."""
        d, f, v = self.dim, self.ffn_dim, self.vocab_size
        qkv = (self.n_heads + 2 * self.n_kv_heads) * self.head_dim * d
        mm = self.n_layers * (qkv + d * d + 3 * f * d) + v * d
        attn = self.n_layers * 2 * 2 * seq_len * d / 2  # QK^T and PV, causal half
        return 6.0 * mm + 3.0 * attn


CONFIGS: Dict[str, LlamaConfig] = {
    "llama3_8b": LlamaConfig(),
    "llama3_1b": LlamaConfig(dim=2048, n_layers=16, n_heads=32, n_kv_heads=8, ffn_dim=8192),
    "llama3_debug": LlamaConfig(dim=256, n_layers=2, n_heads=8, n_kv_heads=2, vocab_size=2048, ffn_dim=768, max_seq_len=512),
    "llama3_tiny": LlamaConfig(dim=64, n_layers=2, n_heads=4, n_kv_heads=2, vocab_size=512, ffn_dim=192, max_seq_len=128),
}


class Block(nn.Module):
    """Pre-norm transformer block on the fused kernels: norm+QKV GEMM, RoPE+split, SDPA, output GEMM with the residual in
    its epilogue, norm+gate/up GEMM, SwiGLU+down GEMM with the residual in its epilogue."""

    def __init__(self, cfg: LlamaConfig, device=None, dtype=torch.bfloat16) -> None:
        super().__init__()
        d, hd = cfg.dim, cfg.head_dim
        kw = dict(device=device, dtype=dtype)
        self.cfg = cfg
        self.attention_norm = nn.Parameter(torch.empty(d, **kw))
        self.wqkv = nn.Parameter(torch.empty((cfg.n_heads + 2 * cfg.n_kv_heads) * hd, d, **kw))
        self.wo = nn.Parameter(torch.empty(d, d, **kw))
        self.ffn_norm = nn.Parameter(torch.empty(d, **kw))
        self.w13 = nn.Parameter(torch.empty(2 * cfg.ffn_dim, d, **kw))
        self.w2 = nn.Parameter(torch.empty(d, cfg.ffn_dim, **kw))

    def forward(self, x: torch.Tensor, cs: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        B, S, d = x.shape
        # residual stream is threaded through the norm nodes (norm_linear_res) and added in the
        # projection GEMMs' epilogues: no standalone elementwise add in forward or backward
        x, qkv = fused.norm_linear_res(x, self.attention_norm, self.wqkv, cfg.norm_eps)
        q, k, v = fused.rope_qkv(qkv.view(B * S, -1), cs, B, S, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim)
        o = F.scaled_dot_product_attention(
            q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True,
            enable_gqa=cfg.n_kv_heads != cfg.n_heads,
        )
        o = o.transpose(1, 2).reshape(B, S, d)
        h = fused.linear(o, self.wo, res=x)
        h, gu = fused.norm_linear_res(h, self.ffn_norm, self.w13, cfg.norm_eps)
        return fused.swiglu_linear(gu, self.w2, res=h)


class Llama(nn.Module):
    """Decoder-only Llama-3 style model; ``forward(tokens, targets)`` returns the mean next-token loss through the chunked
    linear-cross-entropy (no fp32 logits), ``forward(tokens)`` returns logits."""

    def __init__(self, cfg: LlamaConfig, device=None, dtype=torch.bfloat16) -> None:
        super().__init__()
        self.cfg = cfg
        kw = dict(device=device, dtype=dtype)
        self.tok_embeddings = nn.Parameter(torch.empty(cfg.vocab_size, cfg.dim, **kw))
        self.layers = nn.ModuleList(Block(cfg, device=device, dtype=dtype) for _ in range(cfg.n_layers))
        self.norm = nn.Parameter(torch.empty(cfg.dim, **kw))
        self.output = nn.Parameter(torch.empty(cfg.vocab_size, cfg.dim, **kw))
        self._cs: Optional[torch.Tensor] = None
        # called with the stage index right before that stage's parameters are first read in forward
        # (stage order = param_stages()); lets an optimizer that updates stage by stage gate the forward
        self.stage_hook: Optional[Callable[[int], None]] = None

    def param_stages(self) -> List[List[nn.Parameter]]:
        """Parameters grouped by first use in forward: [embedding], one group per block, [final norm, output]."""
        return [[self.tok_embeddings], *[list(b.parameters()) for b in self.layers], [self.norm, self.output]]

    @torch.no_grad()
    def init_weights(self, seed: int = 0) -> None:
        """Deterministic random init (same on every replica for a given seed)."""
        gen = torch.Generator(device=self.tok_embeddings.device)
        gen.manual_seed(seed)
        std = 0.02
        for name, p in self.named_parameters():
            if name.endswith("norm"):
                p.fill_(1.0)
            else:
                s = std / math.sqrt(2 * self.cfg.n_layers) if name.endswith(("wo", "w2")) else std
                p.normal_(0.0, s, generator=gen)

    def rope_cache(self, seq_len: int, device: torch.device) -> torch.Tensor:
        if self._cs is None or self._cs.shape[0] < seq_len or self._cs.device != device:
            self._cs = fused.rope_table(max(seq_len, 1), self.cfg.head_dim, self.cfg.rope_theta, device)
        return self._cs

    def hidden(self, tokens: torch.Tensor) -> torch.Tensor:
        B, S = tokens.shape
        cs = self.rope_cache(S, tokens.device)
        hook = self.stage_hook
        if hook is not None:
            hook(0)
        x = F.embedding(tokens, self.tok_embeddings)
        for i, blk in enumerate(self.layers):
            if hook is not None:
                hook(i + 1)
            if self.cfg.activation_checkpoint == "full" and torch.is_grad_enabled():
                from torch.utils.checkpoint import checkpoint

                x = checkpoint(blk, x, cs, use_reentrant=False)
            else:
                x = blk(x, cs)
        return x

    def forward(self, tokens: torch.Tensor, targets: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Returns the mean next-token loss when ``targets`` is given, else logits."""
        x = self.hidden(tokens)
        B, S, d = x.shape
        if self.stage_hook is not None:
            self.stage_hook(len(self.layers) + 1)
        if targets is None:
            return fused.rmsnorm(x, self.norm, self.cfg.norm_eps) @ self.output.t()
        h = fused.rmsnorm(x, self.norm, self.cfg.norm_eps).view(B * S, d)
        return fused.linear_cross_entropy(h, self.output, targets.reshape(-1), chunk=self.cfg.loss_chunk, count_valid=False)


class FlatParams:
    """Re-home a module's parameters (and gradients) into two flat bf16 buffers.

    ``grad_alloc(numel) -> Tensor`` lets the caller place the gradient buffer in
    NVLink-symmetric memory (``ProcessGroupB200.alloc_symmetric``); buckets for
    the overlapped cross-replica all-reduce are contiguous slices of it.
    Parameters are laid out in reverse FORWARD order (``module.param_stages()`` when the module
    provides it, else reverse registration order) so that buckets fill front-to-back in the
    order backward produces gradients.
    """

    ALIGN = 128  # elements; keeps every view 256 B aligned

    def __init__(self, module: nn.Module, grad_alloc: Optional[Callable[[int], torch.Tensor]] = None,
                 device: Optional[torch.device] = None,
                 param_alloc: Optional[Callable[[int], torch.Tensor]] = None) -> None:
        named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        assert named, "module has no parameters"
        dev, dt = named[0][1].device, named[0][1].dtype
        meta = dev.type == "meta"
        if meta:
            # module built on the meta device: materialise straight into the flat
            # buffer (no transient second copy of the weights); caller initialises after.
            assert device is not None, "pass device= when flattening a meta module"
            dev = torch.device(device)
        # Gradient-production order = reverse of first use in forward. Registration order is only a proxy
        # (a module's own parameters are listed before its children's), so a model that knows its forward
        # order says so through ``param_stages()``: for Llama that puts the LM head and final norm FIRST
        # (their gradients exist at the very start of backward and their all-reduce then hides under the
        # rest of it) and the embedding last.
        if hasattr(module, "param_stages"):
            name_of = {id(p): n for n, p in named}
            fwd = [p for stage in module.param_stages() for p in stage if id(p) in name_of]
            assert len({id(p) for p in fwd}) == len(named), "param_stages() must cover every parameter exactly once"
            order = [(name_of[id(p)], p) for p in reversed(fwd)]
        else:
            order = list(reversed(named))
        offs, total = [], 0
        for _, p in order:
            offs.append(total)
            total += (p.numel() + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.numel = total
        # ``param_alloc`` places the weights in peer-visible memory too (FT-ZeRO-1: the holder of a slice stores
        # the updated bf16 weights straight into every replica's parameter buffer)
        self.param = param_alloc(total)[:total] if param_alloc is not None else torch.zeros(total, dtype=dt, device=dev)
        assert self.param.numel() == total and self.param.dtype == dt
        self.grad = grad_alloc(total) if grad_alloc is not None else torch.zeros(total, dtype=dt, device=dev)
        assert self.grad.numel() >= total and self.grad.dtype == dt
        self.grad = self.grad[:total]
        self.params: List[nn.Parameter] = []
        self.offsets: List[int] = offs
        with torch.no_grad():
            for (name, p), o in zip(order, offs):
                v = self.param[o : o + p.numel()].view(p.shape)
                if meta:
                    q = nn.Parameter(v, requires_grad=True)
                    owner = module
                    *path, leaf = name.split(".")
                    for part in path:
                        owner = getattr(owner, part)
                    setattr(owner, leaf, q)
                    p = q
                else:
                    v.copy_(p.data)
                    p.data = v
                p._flat_grad = self.grad[o : o + p.numel()].view(p.shape)  # wgrad GEMMs write here directly
                p.grad = p._flat_grad
                self.params.append(p)

    def reset_grads(self, zero: bool = False) -> None:
        """Start a step: with ``zero=False`` every ``p.grad`` is dropped so producers write their
        gradient straight into the flat buffer (no memset, no accumulate pass); ``zero=True`` keeps
        the classic zeroed-views behaviour (needed for gradient accumulation over micro-batches)."""
        if zero:
            self.grad.zero_()
            for p in self.params:
                p.grad = p._flat_grad
        else:
            for p in self.params:
                p.grad = None

    def adopt_grad(self, p: nn.Parameter) -> None:
        """Make sure ``p.grad`` IS its slice of the flat buffer (copy if autograd produced it elsewhere)."""
        g = p.grad
        slot = p._flat_grad
        if g is None:
            slot.zero_()
        elif g.data_ptr() != slot.data_ptr():
            slot.copy_(g)
        p.grad = slot

    def buckets_from_ranges(self, ranges) -> List[Tuple[int, int, List[nn.Parameter]]]:
        """(start, end, params) for caller-chosen element ranges (each parameter must fall inside exactly one)."""
        out: List[Tuple[int, int, List[nn.Parameter]]] = []
        for lo, hi in ranges:
            ps = [p for p, o in zip(self.params, self.offsets) if lo <= o < hi]
            assert all(o + p.numel() <= hi for p, o in zip(self.params, self.offsets) if lo <= o < hi), "parameter straddles a range"
            out.append((int(lo), int(hi), ps))
        assert sum(len(b[2]) for b in out) == len(self.params), "ranges must cover every parameter exactly once"
        return out

    def buckets(self, bucket_elems: int) -> List[Tuple[int, int, List[nn.Parameter]]]:
        """Contiguous (start, end, params) buckets in gradient-production order."""
        out: List[Tuple[int, int, List[nn.Parameter]]] = []
        start, cur = 0, []
        for i, (p, o) in enumerate(zip(self.params, self.offsets)):
            cur.append(p)
            end = self.offsets[i + 1] if i + 1 < len(self.params) else self.numel
            if end - start >= bucket_elems or i + 1 == len(self.params):
                out.append((start, end, cur))
                start, cur = end, []
        return out
