"""Reconfigurable, fault-tolerant process groups.

Every class here is a ``torch.distributed.ProcessGroup`` whose membership can
change at runtime through :meth:`ProcessGroup.configure` (one call per quorum
change) and whose failures surface as a *latched error* (:meth:`errored`)
instead of a crashed process. API parity: upstream torchft/process_group.py.

=========================  =====================================================
``ProcessGroupB200``       native: collectives are hand-written sm_90a
                           kernels over NVLink peer memory; ``configure`` remaps
                           peer handles instead of re-creating a
                           communicator; no NCCL on the hot path.
``ProcessGroupNCCL``       reference-equivalent baseline: stock c10d NCCL
                           destroyed/re-created per quorum, user-space timeouts
                           + ``abort`` (reference :780-891).
``ProcessGroupGloo``       CPU / plumbing path (reference :643-711).
``ProcessGroupBaby*``      the real PG hosted in a killable subprocess
                           (reference :1356-2118).
``ProcessGroupDummy``      world-size-1 no-op (reference :1005-1134).
wrappers                   ``ErrorSwallowingProcessGroupWrapper``,
                           ``FakeProcessGroupWrapper`` (fault injection),
                           ``ManagedProcessGroup`` (HSDP replicate dimension).
=========================  =====================================================

Intel XPU twins (``ProcessGroupXCCL``) are intentionally absent: this framework
targets sm_90a only.
"""

from __future__ import annotations

import logging
import os
from contextlib import contextmanager
from datetime import timedelta
from typing import TYPE_CHECKING, Any, Callable, Dict, Generator, List, Optional, Tuple, TypeVar

import torch
import torch.distributed as dist
from torch.distributed import PrefixStore, ReduceOp, Store, TCPStore, Work
from torch.distributed import ProcessGroup as BaseProcessGroup
from torch.distributed.distributed_c10d import AllgatherOptions, BarrierOptions, BroadcastOptions
from torch.futures import Future

from torchft_b200.futures import context_timeout, stream_timeout
from torchft_b200.utils import synchronize
from torchft_b200.work import DummyWork

if TYPE_CHECKING:
    from torchft_b200.manager import Manager

logger = logging.getLogger(__name__)
T = TypeVar("T")

TORCH_NCCL_DEBUG_INFO_PIPE_FILE_ENV_VAR = "TORCH_NCCL_DEBUG_INFO_PIPE_FILE"
TRIGGER_FR_ON_ABORT_ENV = "TORCHFT_TRIGGER_FR_ON_ABORT"


def create_store_client(store_addr: str, timeout: timedelta) -> Store:
    """``host:port/some/prefix`` -> ``PrefixStore("some/prefix", TCPStore(host, port))`` client."""
    hostport, _, prefix = store_addr.partition("/")
    host, _, port = hostport.rpartition(":")
    store = TCPStore(host_name=host, port=int(port), is_master=False, wait_for_workers=False, timeout=timeout)
    return PrefixStore(prefix, store)


def trigger_nccl_fr_trace_through_pipe(rank: int) -> bool:
    """Ask the NCCL flight recorder to dump through its named pipe (reference :92-106)."""

    prefix = os.environ.get(TORCH_NCCL_DEBUG_INFO_PIPE_FILE_ENV_VAR, "")
    if not prefix:
        logger.info("[rank %d] flight-recorder pipe not enabled", rank)
        return False
    try:
        with open(f"{prefix}{rank}.pipe", "w") as f:
            f.write("1\n")
        return True
    except OSError as e:  # pragma: no cover
        logger.warning("[rank %d] could not trigger flight recorder dump: %s", rank, e)
        return False


def _reduce_op(opts: Any) -> ReduceOp:
    if isinstance(opts, ReduceOp) or isinstance(opts, ReduceOp.RedOpType):
        return opts  # type: ignore[return-value]
    return opts.reduceOp


# --------------------------------------------------------------------------- base
class ProcessGroup(BaseProcessGroup):
    """Base class: c10d collectives + the reconfiguration / error-latch protocol."""

    def __init__(self, *args: Any, **kwargs: Any) -> None:
        super().__init__(*args, **kwargs)
        self._group_name: Optional[str] = None

    # collectives: subclasses override what they support
    def _unsupported(self, what: str) -> Work:
        raise NotImplementedError(f"{type(self).__name__} does not implement {what}")

    def allgather(self, output_tensors: List[List[torch.Tensor]], input_tensor: List[torch.Tensor], opts: Any) -> Work:
        return self._unsupported("allgather")

    def allgather_into_tensor_coalesced(self, output_tensors: List[torch.Tensor], input_tensors: List[torch.Tensor], opts: Any) -> Work:
        return self._unsupported("allgather_into_tensor_coalesced")

    def allreduce(self, tensors: List[torch.Tensor], opts: Any) -> Work:
        return self._unsupported("allreduce")

    def allreduce_coalesced(self, tensors: List[torch.Tensor], opts: Any) -> Work:
        return self._unsupported("allreduce_coalesced")

    def alltoall_base(self, output_buffer: torch.Tensor, input_buffer: torch.Tensor, output_split_sizes: List[int],
                      input_split_sizes: List[int], opts: Any) -> Work:
        return self._unsupported("alltoall_base")

    def barrier(self, opts: Any = None) -> Work:
        return self._unsupported("barrier")

    def broadcast(self, tensor_list: List[torch.Tensor], opts: Any) -> Work:
        return self._unsupported("broadcast")

    def broadcast_one(self, tensor: torch.Tensor, root: int) -> Work:
        opts = BroadcastOptions()
        opts.rootRank = root
        return self.broadcast([tensor], opts)

    def recv(self, tensors: List[torch.Tensor], src_rank: int, tag: int) -> Work:
        return self._unsupported("recv")

    def reduce_scatter(self, output_tensors: List[torch.Tensor], input_tensors: List[List[torch.Tensor]], opts: Any) -> Work:
        return self._unsupported("reduce_scatter")

    def reduce_scatter_tensor_coalesced(self, output_tensors: List[torch.Tensor], input_tensors: List[torch.Tensor], opts: Any) -> Work:
        return self._unsupported("reduce_scatter_tensor_coalesced")

    def send(self, tensors: List[torch.Tensor], dst_rank: int, tag: int) -> Work:
        return self._unsupported("send")

    # reconfiguration protocol
    def configure(self, store_addr: str, replica_id: str, rank: int, world_size: int, quorum_id: Optional[int] = None,
                  group_rank: Optional[int] = None, group_world_size: Optional[int] = None,
                  global_ranks: Optional[List[int]] = None) -> None:
        """Re-form the group over a new membership.

        ``store_addr`` (``host:port/prefix``) must be unique per quorum; blocks until
        the group is usable and raises on failure.
        """
        raise NotImplementedError("configure")

    def size(self) -> int:
        raise NotImplementedError("size")

    def getBackendName(self) -> str:
        raise NotImplementedError("getBackendName")

    def abort(self) -> None:
        """Cancel in-flight collectives; the group needs ``configure`` afterwards."""

    def shutdown(self) -> None:
        """Release resources."""

    def errored(self) -> Optional[Exception]:
        """The latched asynchronous error, if any (requires reconfiguration)."""
        return None

    def set_timeout(self, timeout: timedelta) -> None:
        raise NotImplementedError("set_timeout")

    # c10d registry interop (DeviceMesh / functional collectives / FSDP hooks)
    def _register(self, name: str) -> str:
        group_name = f"{self.getBackendName()}:{name}"
        me = self

        def _factory(prefix_store: PrefixStore, rank: int, world_size: int, timeout: float) -> "ProcessGroup":
            return me

        devices = ["cpu"] + (["cuda"] if torch.cuda.is_available() else [])
        dist.Backend.register_backend(group_name, _factory, devices=devices)
        return group_name

    def register(self, name: str) -> "ProcessGroup":
        """Register with the global c10d registry under a unique ``name`` (call once).

        Resizable worlds do not fit DeviceMesh, so the registered group is a
        world-size-1 ``new_group`` whose backend factory returns ``self``.
        """
        group_name = self._register(name)
        return dist.new_group(ranks=[dist.get_rank()], backend=group_name, group_desc=group_name,
                              timeout=timedelta(seconds=60))

    def unregister(self) -> None:
        dist.destroy_process_group(self)

    @property
    def group_name(self) -> str:
        if self._group_name is None:
            raise ValueError("ProcessGroup name not set")
        return self._group_name

    def _set_group_name(self, name: str) -> None:
        self._group_name = name

    def __repr__(self) -> str:
        return f"{type(self).__name__}()"


# ------------------------------------------------------------------------ wrapper
# name -> does the last positional argument carry an options object?
_FORWARDED: Dict[str, bool] = {
    "allgather": True,
    "allgather_into_tensor_coalesced": True,
    "allreduce": True,
    "allreduce_coalesced": True,
    "alltoall_base": True,
    "barrier": True,
    "broadcast": True,
    "reduce_scatter": True,
    "reduce_scatter_tensor_coalesced": True,
    "recv": False,
    "send": False,
}


class ProcessGroupWrapper(ProcessGroup):
    """Holds an inner c10d group that is thrown away and rebuilt on ``configure``.

    Subclasses implement ``_create_pg`` and may customise three hooks applied to
    every forwarded collective: ``_run_context`` (around the call), ``_opts_hook``
    (rewrite options) and ``_wrap_work`` (decorate the returned Work).
    """

    def __init__(self, timeout: timedelta = timedelta(seconds=60), pg: Optional[BaseProcessGroup] = None) -> None:
        super().__init__(0, 1)
        self._pg: Optional[BaseProcessGroup] = pg
        self._timeout = timeout
        self._replica_id: Optional[str] = None
        self._rank: Optional[int] = None
        self._quorum_id: Optional[int] = None
        self._group_rank: Optional[int] = None
        self._group_world_size: Optional[int] = None
        self._global_ranks: Optional[List[int]] = None
        self.errors_logger: logging.Logger = logging.getLogger("torchft_errors")

    @property
    def parent(self) -> BaseProcessGroup:
        if self._pg is None:  # after abort() the group stays unusable until the next configure()
            raise RuntimeError("process group not initialized (or aborted)")
        return self._pg

    def getBackendName(self) -> str:
        if isinstance(self._pg, ProcessGroup):
            return self._pg.getBackendName()
        raise NotImplementedError("getBackendName")

    def size(self) -> int:
        return self.parent.size()

    def set_timeout(self, timeout: timedelta) -> None:
        self._timeout = timeout

    def configure(self, store_addr: str, replica_id: str, rank: int, world_size: int, quorum_id: Optional[int] = None,
                  group_rank: Optional[int] = None, group_world_size: Optional[int] = None,
                  global_ranks: Optional[List[int]] = None) -> None:
        self._replica_id, self._rank, self._quorum_id = replica_id, rank, quorum_id
        self._group_rank, self._group_world_size, self._global_ranks = group_rank, group_world_size, global_ranks
        inner = self._pg
        if isinstance(inner, ProcessGroup):  # wrapping one of ours: delegate
            inner.configure(store_addr, replica_id, rank, world_size, quorum_id, group_rank, group_world_size, global_ranks)
            return
        self.abort(errored=False)
        self._pg = self._create_pg(create_store_client(store_addr, self._timeout), rank, world_size)

    def _log_abort(self) -> None:
        self.errors_logger.info("", extra={
            "job_id": os.environ.get("JOB_ID", "unknown"), "replica_id": self._replica_id, "rank": self._rank,
            "quorum_id": self._quorum_id, "error": "process_group_abort"})

    def abort(self, errored: bool = True) -> None:
        if errored:
            self._log_abort()
        inner, self._pg = self._pg, None
        if inner is None:
            return
        if hasattr(inner, "abort"):
            inner.abort()
            return
        backend = None
        try:
            if torch.cuda.is_available():
                backend = inner._get_backend(torch.device("cuda"))
        except RuntimeError:
            backend = None
        if backend is not None and hasattr(backend, "abort"):
            backend.abort()

    def shutdown(self) -> None:
        self._pg = None

    def _create_pg(self, store: Store, rank: int, world_size: int) -> BaseProcessGroup:
        raise NotImplementedError("_create_pg")

    # hooks
    def _wrap_work(self, work: Work, opts: Any) -> Work:
        return work

    def _opts_hook(self, opts: T) -> T:
        return opts

    @contextmanager
    def _run_context(self) -> Generator[None, None, None]:
        yield

    def _forward(self, name: str, has_opts: bool, args: Tuple[Any, ...]) -> Work:
        opts = args[-1] if has_opts and args else None
        if has_opts and args:
            args = args[:-1] + (self._opts_hook(opts),)
        with self._run_context():
            return self._wrap_work(getattr(self.parent, name)(*args), opts)

    def __repr__(self) -> str:
        return f"{type(self).__name__}(pg={self._pg})"


def _install_forwarders() -> None:
    def make(name: str, has_opts: bool) -> Callable[..., Work]:
        def fwd(self: ProcessGroupWrapper, *args: Any) -> Work:
            return self._forward(name, has_opts, args)

        fwd.__name__ = name
        fwd.__doc__ = f"Forward ``{name}`` to the current inner process group."
        return fwd

    for name, has_opts in _FORWARDED.items():
        setattr(ProcessGroupWrapper, name, make(name, has_opts))


_install_forwarders()


def _barrier_with_default(self: ProcessGroupWrapper, opts: Any = None) -> Work:
    return self._forward("barrier", True, (opts if opts is not None else BarrierOptions(),))


ProcessGroupWrapper.barrier = _barrier_with_default  # type: ignore[method-assign]


# --------------------------------------------------------------------------- gloo
class ProcessGroupGloo(ProcessGroupWrapper):
    """Reconfigurable Gloo group (CPU tensors; also registered for CUDA tensors)."""

    def _create_pg(self, store: Store, rank: int, world_size: int) -> BaseProcessGroup:
        from torch.distributed import ProcessGroupGloo as _Gloo

        pg = BaseProcessGroup(store, rank, world_size)
        pg._set_default_backend(BaseProcessGroup.BackendType.GLOO)
        backend = _Gloo(store, rank, world_size, self._timeout)
        backend._set_sequence_number_for_group()
        if self._global_ranks:
            backend.options.global_ranks_in_group = self._global_ranks
        if self._group_rank is not None and self._group_world_size:
            backend.options.group_name = f"torchft_quorum_{self._quorum_id}_rank_{self._group_rank % self._group_world_size}"
        pg._register_backend(torch.device("cpu"), BaseProcessGroup.BackendType.GLOO, backend)
        if torch.cuda.is_available():
            pg._register_backend(torch.device("cuda"), BaseProcessGroup.BackendType.GLOO, backend)
        return pg

    def getBackendName(self) -> str:
        return "torchft-gloo"

    def reduce_scatter(self, output_tensors: Any, input_tensors: Any, opts: Any) -> Work:
        raise RuntimeError("ProcessGroupGloo does not support reduce_scatter.")

    def reduce_scatter_tensor_coalesced(self, output_tensors: Any, input_tensors: Any, opts: Any) -> Work:
        raise RuntimeError("ProcessGroupGloo does not support reduce_scatter_tensor_coalesced.")


# --------------------------------------------------------------------------- nccl
class _WorkAcceleratorTimeout(Work):
    """NCCL work whose completion is policed by OUR timers (abort the communicator)
    rather than by the NCCL watchdog (which would kill the process)."""

    def __init__(self, pg: "ProcessGroup", work: Work, timeout: timedelta) -> None:
        super().__init__()
        self._pg, self._work, self._timeout = pg, work, timeout

    @staticmethod
    @contextmanager
    def _guard(pg: "ProcessGroup", timeout: timedelta) -> Generator[None, None, None]:
        def on_timeout() -> None:
            logger.error("collective exceeded %s: aborting process group", timeout)
            pg.abort()

        with context_timeout(on_timeout, timeout):  # host-side blocking (e.g. barrier)
            yield
        stream_timeout(on_timeout, timeout)  # device-side: stream must drain in time

    def wait(self, timeout: Optional[timedelta] = None) -> bool:
        with self._guard(self._pg, timeout or self._timeout):
            if self._work is not None and not self._work.wait():
                return False
            if timeout is not None:
                torch.cuda.synchronize()
            return True

    def get_future(self) -> Future:
        fut = self._work.get_future()
        pg, timeout = self._pg, self._timeout

        def on_done(f: Future) -> None:
            try:
                with _WorkAcceleratorTimeout._guard(pg, timeout):
                    f.wait()
            except Exception as e:  # noqa: BLE001
                logger.error("collective future failed: %s", e)

        fut.add_done_callback(on_done)
        return fut


class ProcessGroupNCCL(ProcessGroupWrapper):
    """Reconfigurable NCCL group = the reference's data plane, kept as baseline/fallback.

    ``configure`` aborts the old communicator and builds a new non-blocking one
    (``ncclCommInitRank`` via ``eager_connect_single_device``); per-op user-space
    timeouts call ``abort`` (``ncclCommAbort``, NCCL >= 2.25) so a dead peer
    yields a latched error instead of a watchdog crash.
    """

    def __init__(self, timeout: timedelta = timedelta(seconds=60.0)) -> None:
        super().__init__(timeout)
        self._use_abort = torch.cuda.nccl.version() >= (2, 25) if torch.cuda.is_available() else False
        self._errored: Optional[Exception] = None
        env = "TORCH_NCCL_NONBLOCKING_TIMEOUT"
        if env not in os.environ:
            os.environ[env] = str(timeout.total_seconds())

    def _opts_hook(self, opts: T) -> T:
        if self._use_abort and hasattr(opts, "timeout"):
            opts.timeout = AllgatherOptions().timeout  # type: ignore[attr-defined]  # c10d default = "unset"
        return opts

    def _wrap_work(self, work: Work, opts: Any) -> Work:
        if not self._use_abort:
            return work
        timeout = self._timeout
        if hasattr(opts, "timeout") and opts.timeout.total_seconds() > 0:
            timeout = opts.timeout
        return _WorkAcceleratorTimeout(self, work, timeout)

    @contextmanager
    def _run_context(self) -> Generator[None, None, None]:
        timeout = self._timeout

        def on_timeout() -> None:
            logger.error("collective launch exceeded %s: aborting process group", timeout)
            self.abort()

        with context_timeout(on_timeout, timeout):
            yield

    def _create_pg(self, store: Store, rank: int, world_size: int) -> BaseProcessGroup:
        from torch.distributed import ProcessGroupNCCL as _NCCL

        self._errored = None
        opts = _NCCL.Options()
        opts.config.blocking = False
        if self._global_ranks:
            opts.global_ranks_in_group = self._global_ranks
        if self._group_rank is not None and self._group_world_size:
            opts.group_name = f"torchft_quorum_{self._quorum_id}_rank_{self._group_rank % self._group_world_size}"
        pg = BaseProcessGroup(store, rank, world_size)
        pg._set_default_backend(BaseProcessGroup.BackendType.NCCL)
        backend = _NCCL(store, rank, world_size, opts)
        backend._set_sequence_number_for_group()
        backend.eager_connect_single_device(torch.device("cuda", torch.cuda.current_device()))
        pg._register_backend(torch.device("cuda"), BaseProcessGroup.BackendType.NCCL, backend)
        return pg

    def alltoall_base(self, output_buffer: torch.Tensor, input_buffer: torch.Tensor, output_split_sizes: List[int],
                      input_split_sizes: List[int], opts: Any) -> Work:
        """All-to-all as ONE coalesced group of send/recv.

        torch's NCCL all-to-all helper ends its group without the non-blocking retry loop, so on the
        non-blocking communicators this class creates it fails with ``ncclInProgress`` ("NCCL Error 7",
        seen on NCCL 2.28 / torch 2.11); the coalescing path of ``ProcessGroupNCCL`` polls correctly.
        """
        pg = self.parent
        world, rank = pg.size(), pg.rank()

        def cut(buf: torch.Tensor, sizes: List[int]) -> List[torch.Tensor]:
            if sizes:
                return list(torch.split(buf, list(sizes), dim=0))
            if buf.shape[0] % world:
                raise ValueError("alltoall_base: dim 0 must divide evenly by the world size")
            return list(torch.split(buf, buf.shape[0] // world, dim=0))

        ins, outs = cut(input_buffer, input_split_sizes), cut(output_buffer, output_split_sizes)
        dev = input_buffer.device
        with self._run_context():
            outs[rank].copy_(ins[rank])
            pg._start_coalescing(dev)
            for p in range(world):
                if p != rank:
                    pg.send([ins[p]], p, 0)
                    pg.recv([outs[p]], p, 0)
            work = pg._end_coalescing(dev)
        return self._wrap_work(work, self._opts_hook(opts))

    def abort(self, errored: bool = True) -> None:
        if os.environ.get(TRIGGER_FR_ON_ABORT_ENV, "false") == "true":
            trigger_nccl_fr_trace_through_pipe(dist.get_rank() if dist.is_initialized() else 0)
        # latch BEFORE aborting so errored() is already set when the stream unblocks
        self._errored = RuntimeError("aborted")
        super().abort(errored=errored)

    def errored(self) -> Optional[Exception]:
        synchronize()  # all enqueued work has either finished or been aborted
        return self._errored

    def getBackendName(self) -> str:
        return "torchft-nccl"


# --------------------------------------------------------------------------- xccl
class ProcessGroupXCCL(ProcessGroupWrapper):
    """Reconfigurable XCCL group for Intel XPUs (reference: process_group.py:894-1002).

    API-parity component only: this package's compute and collective kernels are sm_90a CUDA and nothing here is
    exercised on an H100. The wrapper follows the reference's shape -- per-quorum communicator over the prefixed store,
    user-space timeouts that call ``abort`` -- and needs a torch build with XCCL (``torch.distributed.is_xccl_available()``);
    ``configure`` raises a clear error otherwise.
    """

    def __init__(self, timeout: timedelta = timedelta(seconds=60.0)) -> None:
        super().__init__(timeout)
        self._errored: Optional[Exception] = None

    @staticmethod
    def available() -> bool:
        fn = getattr(dist, "is_xccl_available", None)
        return bool(fn and fn()) and hasattr(torch, "xpu") and torch.xpu.is_available()

    def _wrap_work(self, work: Work, opts: Any) -> Work:
        return _WorkAcceleratorTimeout(self, work, self._timeout)

    def _create_pg(self, store: Store, rank: int, world_size: int) -> BaseProcessGroup:
        if not self.available():
            raise RuntimeError("ProcessGroupXCCL needs a PyTorch build with XCCL and an Intel XPU; on NVIDIA H100 use "
                               "ProcessGroupB200 (native NVLink kernels) or ProcessGroupNCCL")
        from torch.distributed import ProcessGroupXCCL as _XCCL  # type: ignore[attr-defined]

        self._errored = None
        opts = _XCCL.Options()
        if self._global_ranks and hasattr(opts, "global_ranks_in_group"):
            opts.global_ranks_in_group = self._global_ranks
        if self._group_rank is not None and self._group_world_size and hasattr(opts, "group_name"):
            opts.group_name = f"torchft_quorum_{self._quorum_id}_rank_{self._group_rank % self._group_world_size}"
        pg = BaseProcessGroup(store, rank, world_size)
        pg._set_default_backend(BaseProcessGroup.BackendType.XCCL)
        backend = _XCCL(store, rank, world_size, opts)
        backend._set_sequence_number_for_group()
        pg._register_backend(torch.device("xpu"), BaseProcessGroup.BackendType.XCCL, backend)
        return pg

    def abort(self, errored: bool = True) -> None:
        self._errored = RuntimeError("aborted")
        super().abort(errored=errored)

    def errored(self) -> Optional[Exception]:
        if hasattr(torch, "xpu") and torch.xpu.is_available():
            torch.xpu.synchronize()
        return self._errored

    def getBackendName(self) -> str:
        return "torchft-xccl"


# -------------------------------------------------------------------------- dummy
class ProcessGroupDummy(ProcessGroup):
    """World-size-1 group: every collective copies input to output and completes.

    Soaks up torch DDP's constructor broadcast and is handy in tests; counts calls.
    """

    def __init__(self, rank: int, world: int) -> None:
        super().__init__(rank, world)
        assert rank == 0 and world == 1
        self._rank, self._world = rank, world
        self.wait_count = 0
        self.get_future_count = 0
        self._work: List[Work] = []
        self.configure_count = 0

    def configure(self, store_addr: str, replica_id: str, rank: int, world_size: int, quorum_id: Optional[int] = None,
                  group_rank: Optional[int] = None, group_world_size: Optional[int] = None,
                  global_ranks: Optional[List[int]] = None) -> None:
        self.configure_count += 1

    def _done(self, result: object) -> Work:
        pg = self

        class _Counted(DummyWork):
            def wait(self, timeout: Optional[timedelta] = None) -> bool:
                pg.wait_count += 1
                return True

            def get_future(self) -> Future:
                pg.get_future_count += 1
                return super().get_future()

        w = _Counted(result)
        self._work.append(w)
        return w

    def allgather(self, output_tensors: Any, input_tensor: Any, opts: Any) -> Work:
        for outs, inp in zip(output_tensors, input_tensor):
            for o in outs:
                o.copy_(inp)
        return self._done(output_tensors)

    def allgather_into_tensor_coalesced(self, output_tensors: Any, input_tensors: Any, opts: Any) -> Work:
        for o, i in zip(output_tensors, input_tensors):
            o.copy_(i)
        return self._done(output_tensors)

    def allreduce(self, tensors: Any, opts: Any) -> Work:
        return self._done(tensors)

    def allreduce_coalesced(self, tensors: Any, opts: Any) -> Work:
        return self._done(tensors)

    def alltoall_base(self, output_buffer: Any, input_buffer: Any, output_split_sizes: Any, input_split_sizes: Any, opts: Any) -> Work:
        output_buffer.copy_(input_buffer)
        return self._done([output_buffer])

    def barrier(self, opts: Any = None) -> Work:
        return self._done(None)

    def broadcast(self, tensor_list: Any, opts: Any) -> Work:
        return self._done(tensor_list)

    def recv(self, tensors: Any, src_rank: int, tag: int) -> Work:
        return self._done(tensors)

    def reduce_scatter(self, output_tensors: Any, input_tensors: Any, opts: Any) -> Work:
        for o, ins in zip(output_tensors, input_tensors):
            o.copy_(ins[0])
        return self._done(output_tensors)

    def reduce_scatter_tensor_coalesced(self, output_tensors: Any, input_tensors: Any, opts: Any) -> Work:
        for o, i in zip(output_tensors, input_tensors):
            o.copy_(i)
        return self._done(output_tensors)

    def send(self, tensors: Any, dst_rank: int, tag: int) -> Work:
        return self._done(tensors)

    def size(self) -> int:
        return self._world

    def getBackendName(self) -> str:
        return "torchft-dummy"


# ----------------------------------------------------------------------- wrappers
class _ErrorSwallowingWork(Work):
    def __init__(self, pg: "ErrorSwallowingProcessGroupWrapper", work: Work, default: object) -> None:
        super().__init__()
        self._pg, self._work, self._default = pg, work, default

    def wait(self, timeout: Optional[timedelta] = None) -> bool:
        try:
            self._work.wait() if timeout is None else self._work.wait(timeout)
        except Exception as e:  # noqa: BLE001
            self._pg.report_error(e)
        return True

    def get_future(self) -> Future:
        fut = self._work.get_future()
        pg, default = self._pg, self._default

        def swallow(f: Future) -> object:
            try:
                return f.value()
            except Exception as e:  # noqa: BLE001
                pg.report_error(e)
                return default

        return fut.then(swallow)


class ErrorSwallowingProcessGroupWrapper(ProcessGroupWrapper):
    """Latch the first error; afterwards collectives are no-ops until ``configure`` (reference :1137-1249)."""

    def __init__(self, pg: ProcessGroup) -> None:
        super().__init__(pg=pg)
        self._error: Optional[Exception] = None

    def configure(self, *args: Any, **kwargs: Any) -> None:
        self._error = None
        super().configure(*args, **kwargs)

    def report_error(self, e: Exception) -> None:
        self._error = e

    def error(self) -> Optional[Exception]:
        return self._error

    def errored(self) -> Optional[Exception]:
        return self._error or (self._pg.errored() if isinstance(self._pg, ProcessGroup) else None)

    def _forward(self, name: str, has_opts: bool, args: Tuple[Any, ...]) -> Work:
        result = args[0] if args else None
        if self._error is not None:
            return DummyWork(result)
        try:
            return _ErrorSwallowingWork(self, super()._forward(name, has_opts, args), result)
        except Exception as e:  # noqa: BLE001
            self.report_error(e)
            return DummyWork(result)


class FakeProcessGroupWrapper(ProcessGroupWrapper):
    """Fault injection: ``report_future_error(e)`` makes the NEXT collective's future raise ``e``
    (reference :1252-1317); used by the EventInjector-driven integration tests."""

    def __init__(self, pg: ProcessGroup) -> None:
        super().__init__(pg=pg)
        self._future_error: Optional[Exception] = None

    def configure(self, *args: Any, **kwargs: Any) -> None:
        self._future_error = None
        super().configure(*args, **kwargs)

    def report_future_error(self, e: Exception) -> None:
        self._future_error = e

    def _forward(self, name: str, has_opts: bool, args: Tuple[Any, ...]) -> Work:
        work = super()._forward(name, has_opts, args)
        if self._future_error is None:
            return work
        err, self._future_error = self._future_error, None
        fut: Future = Future()
        fut.set_exception(err)

        class _Failing(Work):
            def wait(self, timeout: Optional[timedelta] = None) -> bool:
                raise err

            def get_future(self) -> Future:
                return fut

        return _Failing()


class ManagedProcessGroup(ProcessGroup):
    """The Manager as a process group: ``allreduce`` is fault tolerant and ``size()`` is the
    live participant count. This is what HSDP installs as its replicate dimension
    (reference :1320-1353)."""

    def __init__(self, manager: "Manager") -> None:
        super().__init__(0, 1)
        self._manager = manager

    def allreduce(self, tensors: List[torch.Tensor], opts: Any) -> Work:
        assert len(tensors) == 1, "ManagedProcessGroup.allreduce takes exactly one tensor"
        op = _reduce_op(opts) if opts is not None else ReduceOp.SUM
        return self._manager.allreduce(tensors[0], reduce_op=op)

    def size(self) -> int:
        return self._manager.num_participants()

    def getBackendName(self) -> str:
        pg = self._manager._pg
        return pg.getBackendName() if isinstance(pg, ProcessGroup) else "torchft-managed"


# The subprocess-hosted groups live in torchft_b200.baby (which imports this module); the reference exposes
# them from process_group.py, so resolve those names lazily here for import compatibility.
_BABY_NAMES = ("ProcessGroupBaby", "ProcessGroupBabyGloo", "ProcessGroupBabyNCCL")


def __getattr__(name: str) -> Any:
    if name in _BABY_NAMES:
        from torchft_b200 import baby

        return getattr(baby, name)
    if name == "ProcessGroupB200":
        from torchft_b200.parallel.process_group_b200 import ProcessGroupB200

        return ProcessGroupB200
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
