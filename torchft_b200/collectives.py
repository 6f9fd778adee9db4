"""Quantised (fp8) collectives over ANY reconfigurable process group.

API parity with upstream torchft/collectives.py (``allreduce_quantized``,
``reduce_scatter_quantized``, ``get_padded_sizes``, ``allocate_reduce_scatter_output``).
This is the *generic* path (used when the group is NCCL/Gloo-backed): our sm_90a
quantise / reduce / dequantise kernels around the group's ``alltoall_base`` and
``allgather``. On :class:`ProcessGroupB200` the whole pipeline is a single fused
kernel instead -- these functions detect that and delegate.
"""

from __future__ import annotations

from datetime import timedelta
from typing import Any, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch.distributed import ReduceOp, Work
from torch.distributed.distributed_c10d import AllgatherOptions, AllreduceOptions, AllToAllOptions, ReduceScatterOptions
from torch.futures import Future

from torchft_b200 import quantization as Q
from torchft_b200.ops import _native


def _op_of(opts: Any) -> ReduceOp:
    return opts.reduceOp if isinstance(opts, (AllreduceOptions, ReduceScatterOptions)) else opts


class _StreamWork(Work):
    """Completed-on-stream work: ``wait`` joins ``stream`` into the caller's current stream."""

    def __init__(self, stream: Optional[torch.cuda.Stream], result: Any) -> None:
        super().__init__()
        self._event = stream.record_event() if stream is not None else None
        self._fut: Future = Future()
        self._fut.set_result(result)

    def wait(self, timeout: Optional[timedelta] = None) -> bool:
        if self._event is not None:
            torch.cuda.current_stream().wait_event(self._event)
        return True

    def get_future(self) -> Future:
        return self._fut


def get_padded_sizes(tensors: List[torch.Tensor], world_size: int) -> List[torch.Size]:
    """Shapes with dim 0 rounded up to a multiple of ``world_size`` (reference: collectives.py:51-75)."""

    out = []
    for t in tensors:
        s = list(t.shape) if t.dim() > 0 else [1]
        s[0] = (s[0] + world_size - 1) // world_size * world_size
        out.append(torch.Size(s))
    return out


def allocate_reduce_scatter_output(tensors: List[torch.Tensor], world_size: int) -> Tuple[torch.Tensor, List[torch.Size]]:
    """One flat output buffer holding this rank's 1/world_size row-slice of every (padded) tensor."""

    padded = get_padded_sizes(tensors, world_size)
    dt, dev = tensors[0].dtype, tensors[0].device
    for t in tensors:
        if t.dtype != dt or t.device != dev:
            raise ValueError("all tensors must share dtype and device")
    chunk = sum(s.numel() // world_size for s in padded)
    return torch.zeros(chunk, dtype=dt, device=dev), padded


def _check(tensors: List[torch.Tensor], op: ReduceOp) -> None:
    if op not in (ReduceOp.SUM, ReduceOp.AVG):
        raise NotImplementedError(f"quantized collectives support SUM and AVG only, got {op}")
    if not tensors or not all(t.is_cuda for t in tensors):
        raise ValueError("quantized collectives need CUDA tensors")


def _rank_of(pg: Any) -> int:
    r = getattr(pg, "rank", None)
    if callable(r):
        try:
            return int(r())
        except Exception:  # noqa: BLE001
            pass
    inner = getattr(pg, "_rank", None)
    if isinstance(inner, int):
        return inner
    return dist.get_rank(pg)


class _SlicePlan:
    """Per-tensor slicing of a flat message into ``world`` equal slices, each quantised as a
    standalone Q8G chunk (fp32 scale per 512 elements + e4m3 payload) so that chunk ``r`` of every
    tensor can be concatenated into ONE contiguous all-to-all segment for rank ``r``."""

    def __init__(self, tensors: List[torch.Tensor], world: int, slice_elems: Optional[List[int]] = None) -> None:
        self.world = world
        self.slice_elems: List[int] = []
        self.groups: List[int] = []
        self.offsets: List[int] = []
        off = 0
        for i, t in enumerate(tensors):
            if slice_elems is not None:
                se = slice_elems[i]
            else:
                se = (t.numel() + world - 1) // world
                se = (se + 7) // 8 * 8  # slice starts stay 16 B aligned for every dtype we support
            g = (se + Q.GROUP - 1) // Q.GROUP
            self.slice_elems.append(se)
            self.groups.append(g)
            self.offsets.append(off)
            off += ((g * 4 + 15) // 16 * 16) + g * Q.GROUP
        self.chunk_bytes = (off + 15) // 16 * 16


def _quantize_slices(tensors: List[torch.Tensor], plan: _SlicePlan, send: torch.Tensor) -> None:
    K = _native.load()
    sp = _native.stream_ptr()
    for t, se, g, off in zip(tensors, plan.slice_elems, plan.groups, plan.offsets):
        es, n = t.element_size(), t.numel()
        for r in range(plan.world):
            valid = max(0, min(se, n - r * se))
            src = t.data_ptr() + r * se * es if valid > 0 else t.data_ptr()
            K.q8_quantize_raw(src, 0, valid, g, _native.dtype_code(t), send[r].data_ptr() + off, sp)


def _reduce_slices(tensors: List[torch.Tensor], plan: _SlicePlan, recv: torch.Tensor, out_chunk: torch.Tensor,
                   rank: int, post_scale: float) -> None:
    K = _native.load()
    sp = _native.stream_ptr()
    for g, off in zip(plan.groups, plan.offsets):
        ptrs = torch.tensor([recv[p].data_ptr() + off for p in range(plan.world)], dtype=torch.int64, device=recv.device)
        K.q8_reduce_raw(ptrs.data_ptr(), plan.world, rank, g, 0, g, post_scale, out_chunk.data_ptr() + off, sp)


def allreduce_quantized(tensors: List[torch.Tensor], opts: AllreduceOptions | ReduceOp, process_group: dist.ProcessGroup,
                        sync_stream: Optional[torch.cuda.Stream] = None) -> Work:
    """In-place fp8 all-reduce of ``tensors`` (SUM or AVG).

    quantize -> all-to-all of per-rank slices -> fp32 reduce + requantize of the local slice ->
    all-gather -> dequantize, all enqueued on ``sync_stream`` (a side stream by default).
    Expected mean relative error <= 0.04 (reference tolerance, collectives_test.py:186).
    """

    op = _op_of(opts)
    _check(tensors, op)
    world = process_group.size()
    fused = getattr(process_group, "allreduce_q8", None)
    if fused is not None:  # ProcessGroupB200: one kernel per tensor, no NCCL
        scale = 1.0 / world if op == ReduceOp.AVG else 1.0
        works = [fused(t, t, None, scale=scale) for t in tensors]
        for w in works[:-1]:
            w.wait()
        return works[-1]
    rank = _rank_of(process_group)
    K = _native.load()
    stream = sync_stream if sync_stream is not None else torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    contig = [t if (t.is_contiguous() and t.data_ptr() % 16 == 0) else t.contiguous() for t in tensors]
    with torch.cuda.stream(stream):
        plan = _SlicePlan(contig, world)
        dev = contig[0].device
        send = torch.zeros((world, plan.chunk_bytes), dtype=torch.uint8, device=dev)
        _quantize_slices(contig, plan, send)
        recv = torch.empty_like(send)
        process_group.alltoall_base(recv.view(-1), send.view(-1), [], [], AllToAllOptions()).wait()
        mine = torch.zeros(plan.chunk_bytes, dtype=torch.uint8, device=dev)
        _reduce_slices(contig, plan, recv, mine, rank, 1.0 / world if op == ReduceOp.AVG else 1.0)
        gathered = torch.empty((world, plan.chunk_bytes), dtype=torch.uint8, device=dev)
        process_group.allgather([list(gathered.unbind(0))], [mine], AllgatherOptions()).wait()
        sp = _native.stream_ptr()
        for t, se, g, off in zip(contig, plan.slice_elems, plan.groups, plan.offsets):
            es, n = t.element_size(), t.numel()
            for r in range(world):
                valid = max(0, min(se, n - r * se))
                if valid > 0:
                    K.q8_dequantize_raw(gathered[r].data_ptr() + off, g, t.data_ptr() + r * se * es, valid,
                                        _native.dtype_code(t), sp)
        for t, c in zip(tensors, contig):
            if t.data_ptr() != c.data_ptr():
                t.copy_(c)
            t.record_stream(stream)
    return _StreamWork(stream, tensors)


def reduce_scatter_quantized(output: torch.Tensor, inputs: List[torch.Tensor], opts: ReduceScatterOptions | ReduceOp,
                             process_group: dist.ProcessGroup, sync_stream: Optional[torch.cuda.Stream] = None) -> Work:
    """fp8 reduce-scatter: ``output`` receives this rank's row-slice of every (row-padded) input,
    concatenated (layout of :func:`allocate_reduce_scatter_output`): quantize -> all-to-all ->
    fp32 reduce -> dequantize own slice. No all-gather."""

    op = _op_of(opts)
    _check(inputs, op)
    world = process_group.size()
    rank = _rank_of(process_group)
    K = _native.load()
    stream = sync_stream if sync_stream is not None else torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    padded = get_padded_sizes(inputs, world)
    with torch.cuda.stream(stream):
        work_tensors, slices = [], []
        for t, ps in zip(inputs, padded):
            rows = t.shape[0] if t.dim() else 1
            p = torch.zeros(ps, dtype=t.dtype, device=t.device)
            p.view(ps[0], -1)[:rows].copy_(t.reshape(rows, -1))
            work_tensors.append(p)
            slices.append(p.numel() // world)
        es = work_tensors[0].element_size()
        fused = getattr(process_group, "reduce_scatter_q8", None)
        aligned = not any((s * es) % 16 for s in slices) and output.is_contiguous()
        if fused is not None and aligned and world > 1 and all((sum(slices[:i]) * es) % 16 == 0 for i in range(len(slices))) \
                and output.data_ptr() % 16 == 0:
            # ProcessGroupB200: one kernel per tensor does quantise + exchange + reduce; no alltoall, no temporaries
            scale = 1.0 / world if op == ReduceOp.AVG else 1.0
            off = 0
            for p, s in zip(work_tensors, slices):
                fused(output[off: off + s], p.view(-1), s, scale=scale).wait()
                off += s
        elif any((s * es) % 16 for s in slices):
            # rows too narrow for aligned slices: reduce everything, keep our rows
            allreduce_quantized(work_tensors, op, process_group, stream).wait()
            off = 0
            for p, s in zip(work_tensors, slices):
                output[off : off + s].copy_(p.view(-1)[rank * s : (rank + 1) * s])
                off += s
        else:
            plan = _SlicePlan(work_tensors, world, slices)
            dev = work_tensors[0].device
            send = torch.zeros((world, plan.chunk_bytes), dtype=torch.uint8, device=dev)
            _quantize_slices(work_tensors, plan, send)
            recv = torch.empty_like(send)
            process_group.alltoall_base(recv.view(-1), send.view(-1), [], [], AllToAllOptions()).wait()
            mine = torch.zeros(plan.chunk_bytes, dtype=torch.uint8, device=dev)
            _reduce_slices(work_tensors, plan, recv, mine, rank, 1.0 / world if op == ReduceOp.AVG else 1.0)
            sp = _native.stream_ptr()
            off = 0
            aligned_out = output.data_ptr() % 16 == 0 and output.is_contiguous()
            for p, s, g, coff in zip(work_tensors, plan.slice_elems, plan.groups, plan.offsets):
                dst = output[off : off + s]
                if aligned_out and (off * es) % 16 == 0:
                    K.q8_dequantize_raw(mine.data_ptr() + coff, g, dst.data_ptr(), s, _native.dtype_code(p), sp)
                else:
                    tmp = torch.empty(s, dtype=p.dtype, device=dev)
                    K.q8_dequantize_raw(mine.data_ptr() + coff, g, tmp.data_ptr(), s, _native.dtype_code(p), sp)
                    dst.copy_(tmp)
                off += s
        output.record_stream(stream)
    return _StreamWork(stream, output)
