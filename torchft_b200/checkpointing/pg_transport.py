"""Live-checkpoint transport over the fault-tolerant process group's send/recv.

Parity target: upstream torchft/checkpointing/pg_transport.py:32-305.
Protocol (one pair of messages for the header, then one per tensor):

    tag 1: int64 length of the pickled header
    tag 2: uint8[length] pickled ``_Header`` (step, treespec, per-leaf records)
    tag 3+i: raw bytes of tensor i (contiguous, viewed as uint8)

Unlike the reference we ship only the bytes that back each tensor (its
contiguous form), not the whole underlying storage, and the receiver can write
*in place* into tensors supplied by the ``state_dict`` callable (no allocation,
no host bounce). DTensors travel as their local shard plus placement spec.
"""

from __future__ import annotations

import logging
import pickle
import time
from dataclasses import dataclass
from datetime import timedelta
from typing import Any, Callable, Generic, List, Optional, TypeVar

import torch
from torch.utils import _pytree as pytree

from torchft_b200.checkpointing.transport import CheckpointTransport

try:  # DTensor is optional at import time
    from torch.distributed.tensor import DTensor
except Exception:  # pragma: no cover
    DTensor = None  # type: ignore[assignment,misc]

logger = logging.getLogger(__name__)
T = TypeVar("T")


@dataclass
class _TensorRec:
    shape: torch.Size
    dtype: torch.dtype
    nbytes: int
    dtensor_spec: Any = None  # DTensorSpec when the leaf was a DTensor


@dataclass
class _Header:
    step: int
    treespec: Any
    leaves: List[Any]  # _TensorRec for tensors, the object itself otherwise


def _as_bytes(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(-1).view(torch.uint8)


class PGTransport(CheckpointTransport[T], Generic[T]):
    """Send/recv the state_dict over ``pg`` (any of our ProcessGroups).

    Args:
        pg: process group spanning the replicas (the Manager's FT group)
        timeout: per-operation timeout
        device: device tensors are staged on for the wire (cuda for NCCL, cpu for gloo)
        state_dict: optional callable returning the receiver's current state_dict;
            matching tensors are received in place.
    """

    def __init__(self, pg: Any, timeout: timedelta, device: torch.device,
                 state_dict: Optional[Callable[[], T]] = None) -> None:
        self._pg = pg
        self._timeout = timeout
        self._device = torch.device(device)
        self._state_dict = state_dict

    def metadata(self) -> str:
        return "<n/a>"

    def disallow_checkpoint(self) -> None:
        pass

    def _wait(self, work: Any, timeout: timedelta) -> None:
        try:
            work.wait(timeout)
        except TypeError:
            work.wait()

    def send_checkpoint(self, dst_ranks: List[int], step: int, state_dict: T, timeout: timedelta) -> None:
        t0 = time.perf_counter()
        leaves, spec = pytree.tree_flatten(state_dict)
        recs: List[Any] = []
        payloads: List[torch.Tensor] = []
        for leaf in leaves:
            if isinstance(leaf, torch.Tensor):
                dspec = None
                local = leaf
                if DTensor is not None and isinstance(leaf, DTensor):
                    dspec = leaf._spec
                    local = leaf.to_local()
                local = local.detach()
                b = _as_bytes(local)
                recs.append(_TensorRec(local.shape, local.dtype, b.numel(), dspec))
                payloads.append(b)
            else:
                recs.append(leaf)
        blob = pickle.dumps(_Header(step, spec, recs))
        hdr = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(self._device)
        ln = torch.tensor([hdr.numel()], dtype=torch.int64, device=self._device)
        for dst in dst_ranks:
            works = [self._pg.send([ln], dst, 1), self._pg.send([hdr], dst, 2)]
            for w in works:
                self._wait(w, timeout)
        for i, b in enumerate(payloads):
            if b.numel() == 0:
                continue
            wire = b if b.device == self._device else b.to(self._device)
            works = [self._pg.send([wire], dst, 3 + i) for dst in dst_ranks]
            for w in works:
                self._wait(w, timeout)
        logger.info("send_checkpoint took %.3fs", time.perf_counter() - t0)

    def recv_checkpoint(self, src_rank: int, metadata: str, step: int, timeout: timedelta) -> T:
        t0 = time.perf_counter()
        ln = torch.zeros(1, dtype=torch.int64, device=self._device)
        self._wait(self._pg.recv([ln], src_rank, 1), timeout)
        hdr = torch.empty(int(ln.item()), dtype=torch.uint8, device=self._device)
        self._wait(self._pg.recv([hdr], src_rank, 2), timeout)
        header: _Header = pickle.loads(bytes(hdr.cpu().numpy().tobytes()))
        if header.step != step:
            raise RuntimeError(f"checkpoint step mismatch: expected {step}, sender has {header.step}")
        # in-place targets are matched by key path (a restarted replica's state_dict can be structurally
        # smaller than the sender's, e.g. lazily created optimizer state); unmatched leaves are allocated
        inplace: Optional[List[Any]] = None
        if self._state_dict is not None:
            targets = {pytree.keystr(kp): leaf for kp, leaf in pytree.tree_flatten_with_path(self._state_dict())[0]}
            index_tree = pytree.tree_unflatten(list(range(len(header.leaves))), header.treespec)
            inplace = [None] * len(header.leaves)
            for kp, idx in pytree.tree_flatten_with_path(index_tree)[0]:
                inplace[idx] = targets.get(pytree.keystr(kp))
        out: List[Any] = []
        ti = 0
        for i, rec in enumerate(header.leaves):
            if not isinstance(rec, _TensorRec):
                out.append(rec)
                continue
            dst_leaf = inplace[i] if inplace is not None else None
            target: Optional[torch.Tensor] = None
            if isinstance(dst_leaf, torch.Tensor):
                cand = dst_leaf.to_local() if (DTensor is not None and isinstance(dst_leaf, DTensor)) else dst_leaf
                if cand.is_contiguous() and cand.dtype == rec.dtype and cand.shape == rec.shape:
                    target = cand
            if target is None:
                target = torch.empty(rec.shape, dtype=rec.dtype, device=self._device if dst_leaf is None or not isinstance(dst_leaf, torch.Tensor) else dst_leaf.device)
                dst_leaf = None
            if rec.nbytes:
                wire = target.view(-1).view(torch.uint8)
                if wire.device != self._device:
                    tmp = torch.empty(rec.nbytes, dtype=torch.uint8, device=self._device)
                    self._wait(self._pg.recv([tmp], src_rank, 3 + ti), timeout)
                    wire.copy_(tmp)
                else:
                    self._wait(self._pg.recv([wire], src_rank, 3 + ti), timeout)
            ti += 1
            if dst_leaf is not None:
                out.append(dst_leaf)
            elif rec.dtensor_spec is not None and DTensor is not None:
                sp = rec.dtensor_spec
                out.append(DTensor.from_local(target, sp.mesh, sp.placements, run_check=False))
            else:
                out.append(target)
        logger.info("recv_checkpoint took %.3fs", time.perf_counter() - t0)
        return pytree.tree_unflatten(out, header.treespec)
