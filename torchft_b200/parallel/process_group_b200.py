"""``ProcessGroupB200`` -- the native fault-tolerant process group.

Where the reference re-creates an NCCL communicator per quorum
(upstream torchft/process_group.py:435-471,848-873) and funnels every
gradient byte through NCCL (manager.py:466-468), this group

* keeps CUDA context, streams, symmetric segments and signal pads alive across
  quorums and only *remaps peer handles* in ``configure`` (sub-millisecond);
* runs every collective as ONE hand-written sm_90a kernel over NVLink peer memory (P2P loads +
  stores, epoch-tagged flags, bounded abortable spins) on a dedicated comm stream: all-reduce
  (one-/two-shot, NVLS) with the 1/N scale, dtype handling and the non-participant zero
  contribution fused; all-gather, broadcast and all-to-all (equal or per-peer splits) as a push exchange
  through staging slots; reduce-scatter; send / recv through per-pair mailboxes -- each moving exactly the
  algorithmic bytes (``csrc/kernels/{allreduce,allreduce_nvls,collectives,quant,zero1}.cu``);
* surfaces peer death as a latched ``errored()`` (kernel spin timeout / abort
  flag), the in-kernel analogue of ``ncclCommAbort``;
* exposes ``alloc_symmetric`` so gradient buckets can live in peer-visible memory
  and be reduced with zero copies.

What the kernels cannot express (CPU tensors, non-contiguous views, integer reductions) goes to a lazily created NCCL *sidecar* group over the same store, so the
full c10d surface keeps working; nothing on the training or heal paths uses it.
"""

from __future__ import annotations

import logging
import threading
from datetime import timedelta
from typing import Any, List, Optional

import torch
from torch.distributed import PrefixStore, ReduceOp, Work
from torch.futures import Future

from torchft_b200.ops import _native
from torchft_b200.parallel.symm_mem import SymmetricComm
from torchft_b200.process_group import (
    ProcessGroup,
    ProcessGroupGloo,
    ProcessGroupNCCL,
    _reduce_op,
    create_store_client,
)

logger = logging.getLogger(__name__)

_NATIVE_DTYPES = (torch.float32, torch.bfloat16, torch.float16)


def _native_op(op: Any) -> Optional[tuple]:
    """``(kernel op code, is_avg)`` for reduce ops the kernels implement, else ``None``. Compared with ``==``:
    ``opts.reduceOp`` is a ``ReduceOp`` OBJECT whose hash differs from the ``ReduceOp.SUM`` enum member, so a dict
    lookup silently misses (and used to send plain SUM all-reduces to the NCCL sidecar)."""
    for member, code in ((ReduceOp.SUM, _native.OP_SUM), (ReduceOp.MAX, _native.OP_MAX), (ReduceOp.MIN, _native.OP_MIN)):
        if op == member:
            return code, False
    if op == ReduceOp.AVG:
        return _native.OP_SUM, True
    return None


class StreamWork(Work):
    """Work for a kernel enqueued on the group's comm stream.

    ``wait()`` makes the CALLER's current stream wait for the kernel (no host
    block), exactly like c10d NCCL work; ``synchronize`` blocks the host.
    """

    def __init__(self, event: Optional[torch.cuda.Event], result: object) -> None:
        super().__init__()
        self._event = event
        self._result = result
        self._fut: Optional[Future] = None

    def wait(self, timeout: Optional[timedelta] = None) -> bool:
        if self._event is not None:
            torch.cuda.current_stream().wait_event(self._event)
            if timeout is not None:
                self._event.synchronize()
        return True

    def block_current_stream(self) -> None:
        self.wait()

    def synchronize(self) -> None:
        if self._event is not None:
            self._event.synchronize()

    def is_completed(self) -> bool:
        return self._event is None or self._event.query()

    def get_future(self) -> Future:
        # Stream-ordered completion: the future is ready immediately and
        # consumers must call wait() (or chain through _ManagedWork, which does)
        # before touching the tensor on another stream -- same contract as NCCL.
        if self._fut is None:
            self._fut = Future()
            self._fut.set_result(self._result)
        return self._fut


class ProcessGroupB200(ProcessGroup):
    """Fault-tolerant process group over NVLink peer memory (see the module docstring).

    Args:
        timeout: spin budget of every in-kernel wait and of store operations.
        staging_bytes: size of the staging buffer used for tensors outside symmetric memory (default 64 MB).
        device: CUDA device of this rank (default: current device).
    """

    # every member maps every other member's memory: the group is confined to one NVSwitch domain / host,
    # so the Manager may default to the NVLink heal transport and to liveness-driven aborts
    single_host = True
    supports_liveness_abort = True

    def __init__(self, timeout: timedelta = timedelta(seconds=60), staging_bytes: Optional[int] = None,
                 device: Optional[torch.device] = None) -> None:
        super().__init__(0, 1)
        if not torch.cuda.is_available():
            raise RuntimeError("ProcessGroupB200 needs a CUDA device (sm_90a); use ProcessGroupGloo on CPU")
        self._timeout = timeout
        self._device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._comm = SymmetricComm(self._device, staging_bytes=staging_bytes, timeout=timeout)
        self._stream = torch.cuda.Stream(device=self._device, priority=-1)
        self._send_stream = torch.cuda.Stream(device=self._device, priority=-1)
        self._recv_stream = torch.cuda.Stream(device=self._device, priority=-1)
        self._rank = 0
        self._world = 1
        self._store_addr: Optional[str] = None
        self._cfg: Optional[tuple] = None
        self._sidecar: Optional[ProcessGroup] = None
        self._sidecar_lock = threading.Lock()
        self._aborted: Optional[Exception] = None
        self._configure_hooks: List[Any] = []

    # ------------------------------------------------------------- lifecycle
    def add_configure_hook(self, fn: Any) -> None:
        """``fn(store, rank, world, quorum_id)`` runs at the end of every :meth:`configure` with the quorum-scoped
        store, after the peer map is in place (used by the FT-ZeRO-1 optimizer to re-shard its state)."""
        self._configure_hooks.append(fn)

    def configure(self, store_addr: str, replica_id: str, rank: int, world_size: int, quorum_id: Optional[int] = None,
                  group_rank: Optional[int] = None, group_world_size: Optional[int] = None,
                  global_ranks: Optional[List[int]] = None) -> None:
        with torch.cuda.device(self._device):
            store = create_store_client(store_addr, self._timeout)
            self._comm.configure(PrefixStore("b200", store), rank, world_size, int(quorum_id or 0))
            for hook in self._configure_hooks:
                hook(PrefixStore("b200hook", store), rank, world_size, int(quorum_id or 0))
        self._rank, self._world = rank, world_size
        self._store_addr = store_addr
        self._cfg = (replica_id, rank, world_size, quorum_id, group_rank, group_world_size, global_ranks)
        self._aborted = None
        old, self._sidecar = self._sidecar, None
        if old is not None:
            try:
                old.abort()
            except Exception:  # noqa: BLE001
                pass

    def alloc_symmetric(self, name: str, nbytes: int) -> torch.Tensor:
        """Peer-visible uint8 buffer; tensors carved from it are reduced in place with zero copies.
        Call on every replica with identical arguments BEFORE the next ``configure``."""
        return self._comm.alloc(name, nbytes)

    def set_timeout(self, timeout: timedelta) -> None:
        self._timeout = timeout
        self._comm.set_timeout(timeout)

    def abort(self) -> None:
        self._aborted = RuntimeError("aborted")
        self._comm.abort()
        if self._sidecar is not None:
            try:
                self._sidecar.abort()
            except Exception:  # noqa: BLE001
                pass

    def errored(self) -> Optional[Exception]:
        self._stream.synchronize()
        e = self._comm.errored()
        if e is not None:
            return e
        if self._aborted is not None:
            return self._aborted
        return self._sidecar.errored() if self._sidecar is not None else None

    def shutdown(self) -> None:
        self._comm.shutdown()
        if self._sidecar is not None:
            self._sidecar.shutdown()
            self._sidecar = None

    def size(self) -> int:
        return self._world

    def rank(self) -> int:
        return self._rank

    def getBackendName(self) -> str:
        return "torchft-b200"

    @property
    def comm(self) -> SymmetricComm:
        return self._comm

    @property
    def comm_stream(self) -> torch.cuda.Stream:
        return self._stream

    # -------------------------------------------------------------- helpers
    def _native_ok(self, t: torch.Tensor) -> bool:
        return t.is_cuda and t.dtype in _NATIVE_DTYPES and t.is_contiguous() and t.data_ptr() % 16 == 0

    def _launch(self, fn: Any, result: object) -> Work:
        # an earlier kernel already timed out / was aborted: fail fast on the host instead of
        # queueing more collectives against a peer set that needs reconfiguring
        latched = self._comm.errored() or self._aborted
        if latched is not None:
            raise latched
        cur = torch.cuda.current_stream(self._device)
        self._stream.wait_stream(cur)
        with torch.cuda.stream(self._stream):
            fn(self._stream)
            ev = self._stream.record_event()
        stack = [result]
        while stack:  # results may be nested lists (allgather)
            t = stack.pop()
            if isinstance(t, (list, tuple)):
                stack.extend(t)
            elif isinstance(t, torch.Tensor):
                t.record_stream(self._stream)
        return StreamWork(ev, result)

    def _get_sidecar(self) -> ProcessGroup:
        with self._sidecar_lock:
            if self._sidecar is None:
                assert self._cfg is not None and self._store_addr is not None, "configure() first"
                side = ProcessGroupNCCL(timeout=self._timeout)
                rid, rank, world, qid, gr, gws, ranks = self._cfg
                side.configure(self._store_addr + "/sidecar", rid, rank, world, qid, gr, gws, ranks)
                self._sidecar = side
            return self._sidecar

    # ------------------------------------------------------------ collectives
    def allreduce_native(self, tensor: torch.Tensor, op: int = _native.OP_SUM, scale: float = 1.0,
                         contribute: bool = True) -> Work:
        """Fused all-reduce: ``tensor = scale * reduce(op, contributions)``; ``contribute=False``
        adds zeros for this replica (healing / spare) without a separate zero_() pass."""
        return self._launch(lambda s: self._comm.allreduce_(tensor, op=op, scale=scale, contribute=contribute, stream=s), tensor)

    def allreduce_q8(self, out: torch.Tensor, a: torch.Tensor, b: Optional[torch.Tensor] = None, scale: float = 1.0,
                     contribute: bool = True) -> Work:
        """Fused fp8 all-reduce of ``a - b`` (``b`` optional) into ``out``; one kernel, no NCCL."""
        return self._launch(lambda s: self._comm.q8_allreduce_(out, a, b, scale=scale, contribute=contribute, stream=s), out)

    def reduce_scatter_q8(self, out: torch.Tensor, inp: torch.Tensor, slice_elems: int, scale: float = 1.0) -> Work:
        """Fused fp8 reduce-scatter: ``out`` = this rank's ``slice_elems``-element slice of ``inp`` reduced over the
        quorum (quantise + exchange + fp32 reduce in one kernel; no all-to-all call, no temporaries)."""
        return self._launch(lambda s: self._comm.q8_reduce_scatter_(out, inp, slice_elems, scale=scale, stream=s), out)

    def allreduce(self, tensors: List[torch.Tensor], opts: Any) -> Work:
        kind = _native_op(_reduce_op(opts))
        if kind is not None and all(self._native_ok(t) for t in tensors):
            code, scale = kind[0], (1.0 / self._world if kind[1] else 1.0)

            def run(s: torch.cuda.Stream) -> None:
                for t in tensors:
                    self._comm.allreduce_(t, op=code, scale=scale, stream=s)

            return self._launch(run, tensors)
        return self._get_sidecar().allreduce(tensors, opts)

    def allreduce_coalesced(self, tensors: List[torch.Tensor], opts: Any) -> Work:
        return self.allreduce(tensors, opts)

    # Everything below is ONE push-exchange / reduce-scatter / p2p kernel per tensor (csrc/kernels/collectives.cu):
    # algorithmic bytes over NVLink, no zero-padded all-reduce emulation, no NCCL. Only what the kernels cannot
    # express (CPU tensors, non-contiguous views, integer reductions) goes to the sidecar.
    @staticmethod
    def _raw_ok(t: torch.Tensor) -> bool:
        return t.is_cuda and t.is_contiguous()

    def broadcast(self, tensor_list: List[torch.Tensor], opts: Any) -> Work:
        root = opts.rootRank
        if all(self._raw_ok(t) for t in tensor_list):
            def run(s: torch.cuda.Stream) -> None:
                for t in tensor_list:
                    self._comm.broadcast_(t, root, stream=s)

            return self._launch(run, tensor_list)
        return self._get_sidecar().broadcast(tensor_list, opts)

    def barrier(self, opts: Any = None) -> Work:
        # a 16-byte all-reduce in the staging segment; the flag lives as long as the work (ADVICE r1: it used to be
        # freed while the comm-stream kernel still read it)
        with torch.cuda.stream(self._stream):
            flag = torch.zeros(4, dtype=torch.float32, device=self._device)
        return self._launch(lambda s: self._comm.allreduce_(flag, stream=s), flag)

    def allgather(self, output_tensors: List[List[torch.Tensor]], input_tensor: List[torch.Tensor], opts: Any) -> Work:
        if (all(self._raw_ok(t) for t in input_tensor) and all(len(o) == self._world for o in output_tensors)
                and all(self._raw_ok(t) for o in output_tensors for t in o)):
            def run(s: torch.cuda.Stream) -> None:
                for outs, inp in zip(output_tensors, input_tensor):
                    # gather straight into the caller's tensors when they are one contiguous block, else through a flat buffer
                    n = inp.numel() * inp.element_size()
                    base = outs[0].data_ptr()
                    if all(o.data_ptr() == base + r * n and o.numel() * o.element_size() == n for r, o in enumerate(outs)):
                        from torchft_b200.parallel.symm_mem import tensor_from_ptr

                        flat = tensor_from_ptr(base, n * self._world, self._device)
                        self._comm.allgather_(flat, inp, stream=s)
                    else:
                        flat = torch.empty(self._world * inp.numel(), dtype=inp.dtype, device=inp.device)
                        self._comm.allgather_(flat, inp, stream=s)
                        for r, o in enumerate(outs):
                            o.copy_(flat[r * inp.numel():(r + 1) * inp.numel()].view_as(o))

            return self._launch(run, [t for o in output_tensors for t in o])
        return self._get_sidecar().allgather(output_tensors, input_tensor, opts)

    def allgather_into_tensor_coalesced(self, output_tensors: List[torch.Tensor], input_tensors: List[torch.Tensor], opts: Any) -> Work:
        if all(self._raw_ok(t) for t in input_tensors) and all(self._raw_ok(t) for t in output_tensors):
            def run(s: torch.cuda.Stream) -> None:
                for out, inp in zip(output_tensors, input_tensors):
                    assert out.numel() == inp.numel() * self._world
                    self._comm.allgather_(out, inp, stream=s)

            return self._launch(run, output_tensors)
        return self._get_sidecar().allgather_into_tensor_coalesced(output_tensors, input_tensors, opts)

    def _reduce_kind(self, opts: Any, tensors: List[torch.Tensor]) -> Optional[tuple]:
        kind = _native_op(_reduce_op(opts))
        if kind is not None and all(self._raw_ok(t) and t.dtype in _NATIVE_DTYPES for t in tensors):
            return kind[0], (1.0 / self._world if kind[1] else 1.0)
        return None

    def reduce_scatter(self, output_tensors: List[torch.Tensor], input_tensors: List[List[torch.Tensor]], opts: Any) -> Work:
        flat_in = [t for ins in input_tensors for t in ins]
        kind = self._reduce_kind(opts, flat_in + list(output_tensors))
        if kind is not None:
            code, scale = kind

            def run(s: torch.cuda.Stream) -> None:
                for out, ins in zip(output_tensors, input_tensors):
                    n = out.numel() * out.element_size()
                    base = ins[0].data_ptr()
                    if all(t.data_ptr() == base + r * n for r, t in enumerate(ins)):
                        from torchft_b200.parallel.symm_mem import tensor_from_ptr

                        buf = tensor_from_ptr(base, n * self._world, self._device).view(out.dtype)
                    else:
                        buf = torch.cat([t.reshape(-1) for t in ins])
                    self._comm.reduce_scatter_(out, buf, op=code, scale=scale, stream=s)

            return self._launch(run, output_tensors)
        return self._get_sidecar().reduce_scatter(output_tensors, input_tensors, opts)

    def reduce_scatter_tensor_coalesced(self, output_tensors: List[torch.Tensor], input_tensors: List[torch.Tensor], opts: Any) -> Work:
        kind = self._reduce_kind(opts, list(input_tensors) + list(output_tensors))
        if kind is not None:
            code, scale = kind

            def run(s: torch.cuda.Stream) -> None:
                for out, inp in zip(output_tensors, input_tensors):
                    self._comm.reduce_scatter_(out, inp, op=code, scale=scale, stream=s)

            return self._launch(run, output_tensors)
        return self._get_sidecar().reduce_scatter_tensor_coalesced(output_tensors, input_tensors, opts)

    def alltoall_base(self, output_buffer: torch.Tensor, input_buffer: torch.Tensor, output_split_sizes: List[int],
                      input_split_sizes: List[int], opts: Any) -> Work:
        w = self._world
        equal = ((not output_split_sizes or len(set(output_split_sizes)) == 1) and (not input_split_sizes or len(set(input_split_sizes)) == 1)
                 and input_buffer.numel() % max(w, 1) == 0
                 and input_buffer.numel() * input_buffer.element_size() == output_buffer.numel() * output_buffer.element_size())
        if equal and self._raw_ok(output_buffer) and self._raw_ok(input_buffer):
            return self._launch(lambda s: self._comm.alltoall_(output_buffer, input_buffer, stream=s), output_buffer)
        if self._raw_ok(output_buffer) and self._raw_ok(input_buffer) and output_buffer.dim() >= 1 and input_buffer.dim() >= 1:
            # unequal splits (in rows of dim 0): the ranks agree on the number of staging rounds with one tiny MAX
            # all-reduce, then run the same push exchange with per-peer lengths
            def rows_to_bytes(buf: torch.Tensor, splits: List[int]) -> List[int]:
                row = (buf.numel() // max(buf.shape[0], 1)) * buf.element_size()
                if not splits:
                    assert buf.shape[0] % w == 0, "alltoall_base: dim 0 must divide by the world size when no splits are given"
                    splits = [buf.shape[0] // w] * w
                assert len(splits) == w and sum(splits) == buf.shape[0], "alltoall_base: splits must cover dim 0"
                return [int(x) * row for x in splits]

            ob, ib = rows_to_bytes(output_buffer, output_split_sizes), rows_to_bytes(input_buffer, input_split_sizes)
            return self._launch(lambda s: self._comm.alltoallv_(output_buffer, input_buffer, ob, ib, stream=s), output_buffer)
        return self._get_sidecar().alltoall_base(output_buffer, input_buffer, output_split_sizes, input_split_sizes, opts)

    def _p2p_launch(self, stream: torch.cuda.Stream, fn: Any, tensors: List[torch.Tensor]) -> Work:
        latched = self._comm.errored() or self._aborted
        if latched is not None:
            raise latched
        stream.wait_stream(torch.cuda.current_stream(self._device))
        with torch.cuda.stream(stream):
            fn(stream)
            ev = stream.record_event()
        for t in tensors:
            t.record_stream(stream)
        return StreamWork(ev, tensors)

    def send(self, tensors: List[torch.Tensor], dst_rank: int, tag: int) -> Work:
        """Per-pair FIFO over the receiver's mailbox (tags are not matched, like NCCL). Sends and receives run on
        two dedicated streams, so a rank that posts ``send`` then ``recv`` cannot dead-lock against a peer doing the same."""
        if all(self._raw_ok(t) for t in tensors):
            def run(s: torch.cuda.Stream) -> None:
                for t in tensors:
                    self._comm.send_(t, dst_rank, stream=s)

            return self._p2p_launch(self._send_stream, run, tensors)
        return self._get_sidecar().send(tensors, dst_rank, tag)

    def recv(self, tensors: List[torch.Tensor], src_rank: int, tag: int) -> Work:
        if all(self._raw_ok(t) for t in tensors):
            def run(s: torch.cuda.Stream) -> None:
                for t in tensors:
                    self._comm.recv_(t, src_rank, stream=s)

            return self._p2p_launch(self._recv_stream, run, tensors)
        return self._get_sidecar().recv(tensors, src_rank, tag)

    def __repr__(self) -> str:
        return f"ProcessGroupB200(rank={self._rank}, world={self._world})"
