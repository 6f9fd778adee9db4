"""FP8 (e4m3) quantisation primitives -- sm_90a CUDA kernels, not Triton.

API parity with the reference's ``torchft/quantization.py`` (three host
functions around five Triton kernels): :func:`fused_quantize_into_fp8`,
:func:`fused_dequantize_from_fp8`, :func:`fused_reduce_fp8`. The wire format is
ours ("Q8G", see ``csrc/kernels/quant.cu``): per tensor, groups of 512 elements
with one fp32 scale each, padded so the group count divides ``world_size`` and
rank ``r`` owns the ``r``-th contiguous run of groups.

A list of tensors is laid out back to back; every tensor's region starts at a
16-byte boundary. The all-in-one fused collective that never materialises this
buffer outside peer memory is ``SymmetricComm.q8_allreduce_``.
"""

from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
from torch.distributed import ReduceOp

from torchft_b200.ops import _native

GROUP = 512


def _check(t: torch.Tensor) -> None:
    if not t.is_cuda:
        raise ValueError("quantization kernels need CUDA tensors")
    if t.dtype not in _native.DTYPE_CODE:
        raise TypeError(f"unsupported dtype {t.dtype} (need fp32/bf16/fp16)")
    if not t.is_contiguous() or t.data_ptr() % 16:
        raise ValueError("tensor must be contiguous and 16-byte aligned")


def q8_bytes(numel: int, world_size: int) -> int:
    return _native.load().q8_buffer_bytes(numel, world_size)


def quantize_q8(x: torch.Tensor, world_size: int = 1, subtract: torch.Tensor | None = None) -> torch.Tensor:
    """Quantise ``x`` (optionally ``x - subtract``) into a fresh uint8 Q8G buffer."""

    K = _native.load()
    _check(x)
    buf = torch.empty(K.q8_buffer_bytes(x.numel(), world_size), dtype=torch.uint8, device=x.device)
    K.q8_quantize(x.data_ptr(), subtract.data_ptr() if subtract is not None else 0, x.numel(),
                  K.q8_ngroups(x.numel(), world_size), _native.dtype_code(x), buf.data_ptr(), _native.stream_ptr())
    return buf


def dequantize_q8(buf: torch.Tensor, numel: int, dtype: torch.dtype, world_size: int = 1,
                  out: torch.Tensor | None = None) -> torch.Tensor:
    K = _native.load()
    if out is None:
        out = torch.empty(numel, dtype=dtype, device=buf.device)
    _check(out)
    K.q8_dequantize(buf.data_ptr(), K.q8_ngroups(numel, world_size), out.data_ptr(), numel, _native.DTYPE_CODE[dtype],
                    _native.stream_ptr())
    return out


def _layout(inputs: Sequence[torch.Tensor], world_size: int) -> Tuple[List[int], int]:
    offs, total = [], 0
    for t in inputs:
        offs.append(total)
        total += (q8_bytes(t.numel(), world_size) + 15) // 16 * 16
    return offs, total


def fused_quantize_into_fp8(inputs: List[torch.Tensor], world_size: int) -> torch.Tensor:
    """Quantise a list of tensors into one uint8 buffer (reference: quantization.py:531-588)."""

    K = _native.load()
    offs, total = _layout(inputs, world_size)
    buf = torch.empty(total, dtype=torch.uint8, device=inputs[0].device)
    sp = _native.stream_ptr()
    for t, o in zip(inputs, offs):
        t = t.contiguous()
        _check(t)
        K.q8_quantize(t.data_ptr(), 0, t.numel(), K.q8_ngroups(t.numel(), world_size), _native.dtype_code(t),
                      buf.data_ptr() + o, sp)
    return buf


def fused_dequantize_from_fp8(inputs: List[torch.Tensor], quantized: torch.Tensor, world_size: int) -> None:
    """Dequantise ``quantized`` back into ``inputs`` in place (reference: quantization.py:591-635)."""

    K = _native.load()
    offs, total = _layout(inputs, world_size)
    assert quantized.numel() >= total
    sp = _native.stream_ptr()
    for t, o in zip(inputs, offs):
        g = K.q8_ngroups(t.numel(), world_size)
        if not t.is_contiguous():
            tmp = torch.empty_like(t, memory_format=torch.contiguous_format)
            K.q8_dequantize(quantized.data_ptr() + o, g, tmp.data_ptr(), t.numel(), _native.dtype_code(t), sp)
            t.copy_(tmp)
        else:
            _check(t)
            K.q8_dequantize(quantized.data_ptr() + o, g, t.data_ptr(), t.numel(), _native.dtype_code(t), sp)


def fused_reduce_fp8(inputs: List[torch.Tensor], all_buffers: List[torch.Tensor], world_size: int, rank: int,
                     reduce_op: ReduceOp = ReduceOp.SUM) -> None:
    """Reduce rank ``rank``'s slice of ``world_size`` quantised buffers.

    ``all_buffers[p]`` is the buffer received from peer ``p`` (same layout as
    :func:`fused_quantize_into_fp8` output); the reduced + requantised slice is
    written into ``all_buffers[rank]`` (reference: quantization.py:638-686, where
    the buffers are the rows of the all-to-all output).
    """

    K = _native.load()
    if reduce_op not in (ReduceOp.SUM, ReduceOp.AVG):
        raise NotImplementedError(f"unsupported reduce op {reduce_op}")
    assert len(all_buffers) == world_size
    offs, _ = _layout(inputs, world_size)
    post = 1.0 / world_size if reduce_op == ReduceOp.AVG else 1.0
    sp = _native.stream_ptr()
    dev = inputs[0].device
    for t, o in zip(inputs, offs):
        ptrs = torch.tensor([b.data_ptr() + o for b in all_buffers], dtype=torch.int64, device=dev)
        g = K.q8_ngroups(t.numel(), world_size)
        sl = g // world_size
        # the sum starts at this rank's own buffer and wraps, over the groups of this rank's slice
        K.q8_reduce(ptrs.data_ptr(), world_size, rank, g, rank * sl, (rank + 1) * sl, post,
                    all_buffers[rank].data_ptr() + o, sp)



def rank_slice_views(inputs: Sequence[torch.Tensor], buf: torch.Tensor, world_size: int, rank: int) -> List[torch.Tensor]:
    """uint8 views of the parts of a :func:`fused_quantize_into_fp8` buffer that rank ``rank`` owns:
    per tensor, its run of fp32 scales and its run of 512-byte payload groups."""

    K = _native.load()
    offs, _ = _layout(inputs, world_size)
    views = []
    for t, o in zip(inputs, offs):
        g = K.q8_ngroups(t.numel(), world_size)
        sl = g // world_size
        poff = (g * 4 + 15) & ~15
        views.append(buf[o + rank * sl * 4: o + (rank + 1) * sl * 4])
        views.append(buf[o + poff + rank * sl * GROUP: o + poff + (rank + 1) * sl * GROUP])
    return views


def copy_rank_slice(inputs: Sequence[torch.Tensor], dst: torch.Tensor, src: torch.Tensor, world_size: int, rank: int) -> None:
    """``dst[slice of rank] = src[slice of rank]`` for every tensor region (the all-gather step of a
    quantised all-reduce when it is emulated on one device, e.g. in tests)."""
    for d, s in zip(rank_slice_views(inputs, dst, world_size, rank), rank_slice_views(inputs, src, world_size, rank)):
        d.copy_(s)
