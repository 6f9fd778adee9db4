"""Process groups hosted in a killable subprocess ("Baby" PGs).

Why: a wedged NCCL/Gloo collective can only be reliably cancelled by killing the
process that issued it. Hosting the real group in a child lets the trainer kill
and respawn it on ``configure``/``abort`` without losing its own CUDA context or
model state (reference: upstream torchft/process_group.py:1356-2118; costs
documented there -- ~1 GB extra CUDA context per child, no comm/compute overlap --
apply equally). ``ProcessGroupB200`` does not need this: its kernels are abortable.

Design (ours): one request pipe + one response pipe and a strictly serial child
loop. Every collective is ``("run", op_id, method, args)``; completion is observed
with ``("wait", op_id)`` round trips issued either by ``Work.wait`` or by a single
parent-side waiter thread that resolves ``get_future()`` futures. CPU tensors
travel through shared memory, CUDA tensors through CUDA IPC (torch.multiprocessing
reductions); options objects are flattened to plain dicts.
"""

from __future__ import annotations

import logging
import queue
import threading
from dataclasses import dataclass
from datetime import timedelta
from typing import Any, Callable, Dict, List, Optional, Tuple, Type

import torch
import torch.multiprocessing as mp
from torch.distributed import ReduceOp, Work
from torch.distributed.distributed_c10d import (
    AllgatherOptions,
    AllreduceCoalescedOptions,
    AllreduceOptions,
    AllToAllOptions,
    BarrierOptions,
    BroadcastOptions,
    ReduceScatterOptions,
)
from torch.futures import Future

from torchft_b200.multiprocessing import MonitoredPipe, failure_of
from torchft_b200.process_group import _FORWARDED, ProcessGroup, ProcessGroupGloo, ProcessGroupNCCL, ProcessGroupXCCL

logger = logging.getLogger(__name__)

_OPTION_TYPES: Dict[str, type] = {
    c.__name__: c
    for c in (AllgatherOptions, AllreduceOptions, AllreduceCoalescedOptions, AllToAllOptions, BarrierOptions,
              BroadcastOptions, ReduceScatterOptions)
}
_OPTION_FIELDS = ("reduceOp", "rootRank", "rootTensor", "timeout", "asyncOp")


@dataclass
class _FlatOptions:
    """Picklable image of a c10d ``*Options`` object."""

    kind: str
    fields: Dict[str, Any]

    @classmethod
    def flatten(cls, opts: Any) -> Any:
        kind = type(opts).__name__
        if kind not in _OPTION_TYPES:
            if isinstance(opts, (ReduceOp, ReduceOp.RedOpType)):
                return cls("ReduceOp", {"value": _redop_to_int(opts)})
            return opts
        fields: Dict[str, Any] = {}
        for f in _OPTION_FIELDS:
            if hasattr(opts, f):
                v = getattr(opts, f)
                if f == "reduceOp":
                    v = _redop_to_int(v)
                fields[f] = v
        return cls(kind, fields)

    def rebuild(self) -> Any:
        if self.kind == "ReduceOp":
            return _int_to_redop(self.fields["value"])
        opts = _OPTION_TYPES[self.kind]()
        for f, v in self.fields.items():
            if f == "reduceOp":
                v = _int_to_redop(v)
            try:
                setattr(opts, f, v)
            except Exception:  # noqa: BLE001 - read-only / version specific fields
                pass
        return opts


_REDOPS = [ReduceOp.SUM, ReduceOp.AVG, ReduceOp.PRODUCT, ReduceOp.MIN, ReduceOp.MAX, ReduceOp.BAND, ReduceOp.BOR, ReduceOp.BXOR]


def _redop_to_int(op: Any) -> int:
    for i, r in enumerate(_REDOPS):
        if op == r:
            return i
    raise ValueError(f"unsupported reduce op {op}")


def _int_to_redop(i: int) -> ReduceOp:
    return _REDOPS[i]


def _share(obj: Any) -> Any:
    """Move CPU tensors to shared memory (in place) so the child sees the same storage."""
    if isinstance(obj, torch.Tensor):
        if obj.device.type == "cpu" and not obj.is_shared():
            obj.share_memory_()
        return obj
    if isinstance(obj, (list, tuple)):
        return type(obj)(_share(o) for o in obj)
    return _FlatOptions.flatten(obj)


def _unflatten(obj: Any) -> Any:
    if isinstance(obj, _FlatOptions):
        return obj.rebuild()
    if isinstance(obj, (list, tuple)):
        return type(obj)(_unflatten(o) for o in obj)
    return obj


def _child_main(pg_factory: Callable[[timedelta], ProcessGroup], store_addr: str, cfg: Tuple[Any, ...],
                timeout_s: float, device: int, req: Any, resp: Any) -> None:
    """Serial command loop of the subprocess."""

    try:
        if device >= 0 and torch.cuda.is_available():
            torch.cuda.set_device(device)
        pg = pg_factory(timedelta(seconds=timeout_s))
        pg.configure(store_addr, *cfg)
        resp.send(("ready",))
    except Exception as e:  # noqa: BLE001
        resp.send(failure_of(e))
        return
    works: Dict[int, Work] = {}
    while True:
        try:
            cmd = req.recv()
        except (EOFError, OSError):
            return
        try:
            op = cmd[0]
            if op == "run":
                _, op_id, name, args = cmd
                works[op_id] = getattr(pg, name)(*_unflatten(args))
                resp.send(("launched", op_id))
            elif op == "wait":
                _, op_id, wait_timeout = cmd
                w = works.pop(op_id, None)
                if w is not None:
                    w.wait() if wait_timeout is None else w.wait(timedelta(seconds=wait_timeout))
                    if torch.cuda.is_available() and device >= 0:
                        torch.cuda.current_stream().synchronize()
                resp.send(("done", op_id))
            elif op == "drop":
                works.pop(cmd[1], None)
                resp.send(("dropped", cmd[1]))
            elif op == "num_active_work":
                resp.send(("count", len(works)))
            elif op == "exit":
                resp.send(("bye",))
                return
            else:
                raise ValueError(f"unknown command {op}")
        except Exception as e:  # noqa: BLE001
            try:
                resp.send(failure_of(e))
            except Exception:  # noqa: BLE001
                return


class _BabyWork(Work):
    def __init__(self, pg: "ProcessGroupBaby", op_id: int, result: object) -> None:
        super().__init__()
        self._pg, self._op_id, self._result = pg, op_id, result
        self._done = False

    def wait(self, timeout: Optional[timedelta] = None) -> bool:
        if not self._done:
            self._pg._wait(self._op_id, timeout)
            self._done = True
        return True

    def synchronize(self) -> None:
        self.wait()

    def get_future(self) -> Future:
        return self._pg._future(self, self._result)

    def __del__(self) -> None:
        if not self._done:
            try:
                self._pg._drop(self._op_id)
            except Exception:  # noqa: BLE001
                pass


class ProcessGroupBaby(ProcessGroup):
    """Base for subprocess-hosted groups; subclasses name the real group class."""

    PG_CLASS: Type[ProcessGroup]

    def __init__(self, timeout: timedelta | float = 60.0) -> None:
        super().__init__(0, 1)
        self._timeout = timeout if isinstance(timeout, timedelta) else timedelta(seconds=timeout)
        self._world = -1
        self._rank = -1
        self._proc: Optional[Any] = None
        self._req: Optional[Any] = None
        self._resp: Optional[MonitoredPipe] = None
        self._lock = threading.RLock()
        self._next_op = 0
        self._error: Optional[Exception] = None
        self._waiter: Optional[threading.Thread] = None
        self._fut_q: "queue.Queue[Optional[Tuple[_BabyWork, Future, object]]]" = queue.Queue()

    @classmethod
    def _make_pg(cls, timeout: timedelta) -> ProcessGroup:
        return cls.PG_CLASS(timeout=timeout)

    def _mp_context(self) -> Any:
        return mp.get_context("spawn")

    # ------------------------------------------------------------- lifecycle
    def configure(self, store_addr: str, replica_id: str, rank: int, world_size: int, quorum_id: Optional[int] = None,
                  group_rank: Optional[int] = None, group_world_size: Optional[int] = None,
                  global_ranks: Optional[List[int]] = None) -> None:
        self._kill()
        self._error = None
        self._rank, self._world = rank, world_size
        ctx = self._mp_context()
        req_child, req_parent = ctx.Pipe(duplex=False)
        resp_parent, resp_child = ctx.Pipe(duplex=False)
        device = torch.cuda.current_device() if torch.cuda.is_available() else -1
        cfg = (replica_id, rank, world_size, quorum_id, group_rank, group_world_size, global_ranks)
        self._proc = ctx.Process(
            target=_child_main,
            args=(type(self)._make_pg, store_addr, cfg, self._timeout.total_seconds(), device, req_child, resp_child),
            daemon=True,
        )
        self._proc.start()
        self._req, self._resp = req_parent, MonitoredPipe(resp_parent, alive=getattr(self._proc, "is_alive", None))
        # the child's PG creation is a rendezvous with its peers: allow the full timeout (+ process start)
        msg = self._resp.recv(self._timeout + timedelta(seconds=30))
        assert msg == ("ready",), msg
        self._waiter = threading.Thread(target=self._waiter_loop, name="tft_baby_futures", daemon=True)
        self._waiter.start()

    def _kill(self) -> None:
        with self._lock:
            self._fut_q.put(None)
            if self._proc is not None:
                try:
                    self._proc.kill()
                    self._proc.join(timeout=5)
                except Exception:  # noqa: BLE001
                    pass
            for p in (self._req, self._resp):
                try:
                    if p is not None:
                        p.close()
                except Exception:  # noqa: BLE001
                    pass
            self._proc = self._req = self._resp = None
            self._fut_q = queue.Queue()

    def abort(self) -> None:
        self._error = RuntimeError("aborted")
        self._kill()

    def shutdown(self) -> None:
        self._kill()

    def errored(self) -> Optional[Exception]:
        return self._error

    def set_timeout(self, timeout: timedelta) -> None:
        self._timeout = timeout

    def size(self) -> int:
        return self._world

    def getBackendName(self) -> str:
        return f"torchft-baby-{self.PG_CLASS.__name__.replace('ProcessGroup', '').lower()}"

    # -------------------------------------------------------------- plumbing
    def _rpc(self, cmd: Tuple[Any, ...], timeout: timedelta) -> Any:
        with self._lock:
            if self._req is None or self._resp is None:
                raise RuntimeError("process group not initialized (or aborted)")
            try:
                self._req.send(cmd)
                return self._resp.recv(timeout)
            except Exception as e:  # noqa: BLE001
                self._error = e
                if isinstance(e, (TimeoutError, EOFError, BrokenPipeError, OSError)):
                    self._kill()  # wedged or dead child: only a respawn (configure) recovers
                raise

    def _run(self, name: str, args: Tuple[Any, ...]) -> Work:
        if torch.cuda.is_available() and any(isinstance(a, torch.Tensor) and a.is_cuda for a in _flat(args)):
            torch.cuda.current_stream().synchronize()  # child works on its own streams
        with self._lock:
            op_id = self._next_op
            self._next_op += 1
            self._rpc(("run", op_id, name, _share(args)), self._timeout)
        return _BabyWork(self, op_id, args[0] if args else None)

    def _wait(self, op_id: int, timeout: Optional[timedelta]) -> None:
        t = timeout or self._timeout
        self._rpc(("wait", op_id, t.total_seconds()), t + timedelta(seconds=1))

    def _drop(self, op_id: int) -> None:
        if self._req is not None:
            self._rpc(("drop", op_id), timedelta(seconds=5))

    def num_active_work(self) -> int:
        return int(self._rpc(("num_active_work",), self._timeout)[1])

    def _future(self, work: _BabyWork, result: object) -> Future:
        fut: Future = Future()
        self._fut_q.put((work, fut, result))
        return fut

    def _waiter_loop(self) -> None:
        q = self._fut_q
        while True:
            item = q.get()
            if item is None:
                return
            work, fut, result = item
            try:
                work.wait()
                fut.set_result(result)
            except Exception as e:  # noqa: BLE001
                fut.set_exception(e)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(rank={self._rank}, world={self._world})"


def _flat(obj: Any) -> List[Any]:
    if isinstance(obj, (list, tuple)):
        out: List[Any] = []
        for o in obj:
            out.extend(_flat(o))
        return out
    return [obj]


def _install() -> None:
    def make(name: str) -> Callable[..., Work]:
        def op(self: ProcessGroupBaby, *args: Any) -> Work:
            return self._run(name, args)

        op.__name__ = name
        return op

    for name in _FORWARDED:
        setattr(ProcessGroupBaby, name, make(name))

    def barrier(self: ProcessGroupBaby, opts: Any = None) -> Work:
        return self._run("barrier", (opts if opts is not None else BarrierOptions(),))

    ProcessGroupBaby.barrier = barrier  # type: ignore[method-assign]


_install()


class ProcessGroupBabyGloo(ProcessGroupBaby):
    """Gloo in a subprocess (CPU tensors via shared memory)."""

    PG_CLASS = ProcessGroupGloo

    def reduce_scatter(self, *a: Any) -> Work:
        raise RuntimeError("ProcessGroupBabyGloo does not support reduce_scatter.")

    def reduce_scatter_tensor_coalesced(self, *a: Any) -> Work:
        raise RuntimeError("ProcessGroupBabyGloo does not support reduce_scatter_tensor_coalesced.")


class ProcessGroupBabyXCCL(ProcessGroupBaby):
    """XCCL in a subprocess (reference: process_group.py:2081+). API parity for Intel XPUs; see ``ProcessGroupXCCL``."""

    PG_CLASS = ProcessGroupXCCL


class ProcessGroupBabyNCCL(ProcessGroupBaby):
    """NCCL in a subprocess (CUDA tensors via CUDA IPC). Tensors must stay alive until the work is waited on."""

    PG_CLASS = ProcessGroupNCCL
