"""Fault-tolerant data parallelism across replica groups.

* :class:`DistributedDataParallel` / :class:`PureDistributedDataParallel` -- API
  parity with upstream torchft/ddp.py:31-104 (torch DDP bucket hook /
  per-parameter hooks feeding ``Manager.allreduce``).
* :class:`FlatDistributedDataParallel` -- the native path: all gradients live
  in ONE flat bf16 buffer inside NVLink-symmetric memory; backward fills it
  front-to-back and each bucket is all-reduced IN PLACE by the fused P2P kernel
  on the process group's comm stream the moment its last gradient lands, so the
  cross-replica reduction overlaps the rest of backward with zero copies.
"""

import os
from typing import TYPE_CHECKING, Any, Dict, List, Tuple

import torch
import torch.distributed as dist
from torch import nn
from torch.nn import parallel

from torchft_b200.process_group import ProcessGroupDummy

if TYPE_CHECKING:
    from torchft_b200.manager import Manager


class DistributedDataParallel(parallel.DistributedDataParallel):
    """torch DDP whose bucket all-reduce goes through the fault-tolerant Manager.

    The module is wrapped over a world-size-1 dummy group (which also absorbs
    DDP's constructor broadcast); ``find_unused_parameters`` keeps the bucket
    layout static so every replica issues identical collectives even when the
    quorum changes.
    """

    def __init__(self, manager: "Manager", module: nn.Module, **kwargs: Any) -> None:
        pg = ProcessGroupDummy(0, 1)
        kwargs.setdefault("find_unused_parameters", True)
        super().__init__(module, process_group=pg, **kwargs)
        self.register_comm_hook(manager, self._comm_hook)

    @staticmethod
    def _comm_hook(state: "Manager", bucket: dist.GradBucket) -> torch.futures.Future[torch.Tensor]:
        # NOTE: no `from __future__ import annotations` in this module -- torch DDP
        # validates the hook's *runtime* annotations (bucket must be dist.GradBucket).
        buf = bucket.buffer()
        work = state.allreduce(buf)
        work.wait()  # stream dependency (and continuation callbacks); never raises
        fut: torch.futures.Future[torch.Tensor] = torch.futures.Future()
        fut.set_result(buf)
        return fut


class PureDistributedDataParallel(nn.Module):
    """Minimal DDP: one ``Manager.allreduce`` per parameter gradient, no bucketing
    (slow; mirrors reference ddp.py:81-104)."""

    def __init__(self, manager: "Manager", module: nn.Module) -> None:
        super().__init__()
        self.module = module

        def post_grad_hook(p: torch.Tensor) -> None:
            if p.grad is not None:
                manager.allreduce(p.grad).wait()

        for p in module.parameters():
            p.register_post_accumulate_grad_hook(post_grad_hook)

    def forward(self, *args: object, **kwargs: object) -> object:
        return self.module(*args, **kwargs)


class FlatDistributedDataParallel(nn.Module):
    """Bucketed, overlapped, zero-copy gradient all-reduce over a flat symmetric buffer.

    Args:
        manager: the fault-tolerant manager
        module: model whose parameters were (or will be) flattened
        flat: a ``FlatParams`` (``torchft_b200.models.llama.FlatParams``); its gradient
            buffer should come from ``pg.alloc_symmetric`` for the zero-copy path
        bucket_mb: bucket size; buckets are contiguous slices of the flat gradient
        should_quantize: use the fused fp8 all-reduce (communication-bound links)

    Call :meth:`finish` (or ``manager.should_commit`` via the optimizer wrapper after
    :meth:`finish`) once backward is done to join the comm stream.
    """

    def __init__(self, manager: "Manager", module: nn.Module, flat: Any, bucket_mb: float = 256.0,
                 should_quantize: bool = False, bucket_ranges: Any = None, reduce_fn: Any = None) -> None:
        """``bucket_ranges`` (element ranges tiling the flat buffer) overrides the size-based bucketing and
        ``reduce_fn(bucket_index, start, end) -> Work`` replaces the plain ``manager.allreduce`` -- the FT-ZeRO-1
        trainer passes one bucket per optimizer unit and a reduce-scatter."""
        super().__init__()
        self.module = module
        self._manager = manager
        self._flat = flat
        self._quantize = should_quantize
        self._reduce_fn = reduce_fn
        bucket_elems = max(1, int(bucket_mb * (1 << 20)) // flat.grad.element_size())
        self._buckets: "List[Tuple[int, int, List[nn.Parameter]]]" = (
            flat.buckets_from_ranges(bucket_ranges) if bucket_ranges is not None else flat.buckets(bucket_elems))
        self._pending: List[int] = []
        self._works: List[Any] = []
        self._param_bucket: Dict[int, int] = {}
        for bi, (_, _, params) in enumerate(self._buckets):
            for p in params:
                self._param_bucket[id(p)] = bi
        self._reset()
        for p in flat.params:
            p.register_post_accumulate_grad_hook(self._on_grad)

    def _reset(self) -> None:
        self._pending = [len(params) for _, _, params in self._buckets]
        self._works = []

    def _on_grad(self, p: torch.Tensor) -> None:
        self._flat.adopt_grad(p)  # no-op when the producer already wrote into the flat buffer
        bi = self._param_bucket[id(p)]
        self._pending[bi] -= 1
        if self._pending[bi] == 0:
            self._works.append(self._reduce(bi))

    def _reduce(self, bi: int) -> Any:
        start, end, _ = self._buckets[bi]
        if self._reduce_fn is not None:
            return self._reduce_fn(bi, start, end)
        return self._manager.allreduce(self._flat.grad[start:end], should_quantize=self._quantize)

    def forward(self, *args: object, **kwargs: object) -> object:
        return self.module(*args, **kwargs)

    def finish(self, wait: bool = True) -> None:
        """Make the current stream wait for every bucket reduction issued by this backward (``wait=False``:
        only issue the missing ones; whoever consumes the gradients orders itself behind the comm stream)."""
        # parameters that received no gradient this step still need their bucket reduced
        for bi, left in enumerate(self._pending):
            if left > 0:
                start, end, params = self._buckets[bi]
                for q in params:
                    if q.grad is None:
                        self._flat.adopt_grad(q)  # unused parameter this step: contributes zeros
                self._works.append(self._reduce(bi))
        if wait:
            for w in self._works:
                w.wait()
        self._reset()

    @property
    def num_buckets(self) -> int:
        return len(self._buckets)
