"""Per-rank fault-tolerance state machine.

One ``Manager`` per training process. A training step is three calls (semantics of
upstream torchft/manager.py:148-1053, SURVEY.md 3.2 and 7.4):

1. ``start_quorum()``  -- async by default (overlaps the forward pass): intra-group barrier + Lighthouse
   quorum through the C++ ``ManagerServer``; when the quorum id changed the process group is
   *reconfigured* (a peer-memory remap on ``ProcessGroupB200``); replicas behind ``max_step`` heal from
   an up-to-date peer through the checkpoint transport.
2. ``allreduce()`` / ``guarded()`` -- fault-tolerant collectives: errors never raise, the first one is
   latched, later calls become no-ops and the step is discarded.
3. a commit decision, in one of two forms:

   * ``should_commit()`` -- the reference's host-synchronous form: drain the stream, AND over the ranks
     of the group through the ManagerServer, return a bool.
   * ``commit_on_device(committer)`` -- native form for replica groups of ONE rank: the verdict is
     computed by a kernel (``zero1_commit_kernel``: AND of "no latched error, enough participants" over
     the quorum through the NVLink signal pads), lands in a device gate word that the fused optimizer
     kernels test, and the host learns it LAZILY -- on the quorum thread at the next ``start_quorum``,
     or whenever ``current_step()`` is asked. No ``cudaStreamSynchronize`` and no RPC on the step's
     critical path (the reference does both every step, manager.py:884-903).

Bookkeeping (step counter, batches committed, consecutive failures, structured commit log) lives in
``_StepLedger`` and is identical for both forms. A ``_LivenessWatch`` thread turns "the Lighthouse no
longer hears replica X" into ``pg.abort()`` so kernels spinning on a dead peer bail out after the
heartbeat timeout instead of the (much longer) collective timeout.
"""

from __future__ import annotations

import concurrent.futures
import logging
import os
import socket
import threading
import traceback
import uuid
import weakref
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from datetime import timedelta
from enum import Enum
from typing import TYPE_CHECKING, Any, Callable, Dict, List, Optional, TypeVar, cast

import torch
from torch.distributed import ReduceOp, TCPStore, Work
from torch.distributed.distributed_c10d import AllreduceOptions
from torch.futures import Future

from torchft_b200._C import ManagerClient, ManagerServer
from torchft_b200.checkpointing._rwlock import RWLock
from torchft_b200.checkpointing.transport import CheckpointTransport
from torchft_b200.futures import future_timeout
from torchft_b200.utils import get_stream_context, synchronize
from torchft_b200.work import DummyWork

if TYPE_CHECKING:
    from torchft_b200.process_group import ProcessGroup

MANAGER_ADDR_KEY = "manager_addr"
MANAGER_PORT_ENV = "TORCHFT_MANAGER_PORT"
REPLICA_ID_KEY = "replica_id"

# env overrides win over constructor arguments (reference: manager.py:78-87,251-268)
TIMEOUT_SEC_ENV = "TORCHFT_TIMEOUT_SEC"
QUORUM_TIMEOUT_SEC_ENV = "TORCHFT_QUORUM_TIMEOUT_SEC"
CONNECT_TIMEOUT_SEC_ENV = "TORCHFT_CONNECT_TIMEOUT_SEC"
QUORUM_RETRIES_ENV = "TORCHFT_QUORUM_RETRIES"
TORCH_FR_DUMP_TEMP_FILE_ENV = "TORCH_FR_DUMP_TEMP_FILE"
LIVENESS_ENV = "TORCHFT_B200_LIVENESS_ABORT"

T = TypeVar("T")
S = TypeVar("S")


def get_timeout(timeout_sec_env: Optional[str], default_timeout: timedelta) -> timedelta:
    """Environment value (integer seconds) if present, else the default."""
    return timedelta(seconds=int(timeout_sec_env)) if timeout_sec_env is not None else default_timeout


def extract_trailing_digits(s: str) -> int:
    """``"replica_12"`` -> 12; 0 when the string does not end in digits."""
    n = len(s)
    while n > 0 and s[n - 1].isdigit():
        n -= 1
    return int(s[n:]) if n < len(s) else 0


class WorldSizeMode(Enum):
    """How the reduction is normalised when more than ``min_replica_size`` replicas are alive.

    DYNAMIC: use every healthy replica, divide by the live count.
    FIXED_WITH_SPARES: exactly ``min_replica_size`` replicas contribute; the rest are
    hot spares that add zeros.
    """

    DYNAMIC = 0
    FIXED_WITH_SPARES = 1


class ExceptionWithTraceback(Exception):
    """The first error reported in a step, with the traceback that was live when it was reported."""

    def __init__(self, e: Exception) -> None:
        self.original_exception = e
        self.stack_trace = traceback.format_exc()
        super().__init__(f"{e}\n{self.stack_trace}")


# --------------------------------------------------------------------------- small state holders
@dataclass
class _Participation:
    """Who reduces with whom this step, derived from one quorum result."""

    rank: Optional[int] = None   # this replica's index among the contributors (None: spare / behind)
    world: int = 0               # number of contributors (the AVG divisor)

    @staticmethod
    def derive(quorum: Any, everyone_counts: bool, mode: WorldSizeMode, cap: int) -> "_Participation":
        # async quorum (or healing disabled): only replicas already at max_step contribute; a replica
        # that heals eagerly (sync quorum) counts right away
        rank, world = ((quorum.replica_rank, quorum.replica_world_size) if everyone_counts
                       else (quorum.max_replica_rank, quorum.max_world_size))
        if mode == WorldSizeMode.FIXED_WITH_SPARES:
            world = min(world, cap)
            if rank is not None and rank >= cap:
                rank = None
        return _Participation(rank, world)


class _StepLedger:
    """Step counter, committed batches and consecutive commit failures + the structured commit log."""

    def __init__(self, max_retries: Optional[int]) -> None:
        self.step = 0
        self.batches = 0
        self.failures = 0
        self._max_retries = max_retries
        self._log = logging.getLogger("torchft_commits")

    def record(self, committed: bool, participants: int, tags: Dict[str, object]) -> None:
        self._log.info("", extra={**tags, "step": self.step, "commit_result": committed})
        if committed:
            self.step += 1
            self.batches += participants
            self.failures = 0
            return
        self.failures += 1
        if self._max_retries is not None and self.failures > self._max_retries:
            raise RuntimeError(f"should_commit failed {self.failures} times consecutively, exceeding max_retries={self._max_retries}")


@dataclass
class _DeferredCommit:
    committer: Any
    seq: int
    participants: int
    tags: Dict[str, object]


class _LivenessWatch(threading.Thread):
    """Polls the Lighthouse's heartbeat table and calls ``on_dead`` when a member of the current quorum
    stopped heart-beating -- the data plane's spins are then released by ``pg.abort()`` within about one
    heartbeat timeout (the reference's analogue: user-space timeout -> ``ncclCommAbort``,
    process_group.py:738-763, which only fires after the full collective timeout)."""

    def __init__(self, lighthouse_addr: str, members: Callable[[], List[str]], on_dead: Callable[[str], None]) -> None:
        super().__init__(name="torchft_liveness", daemon=True)
        self._addr = lighthouse_addr
        self._members = members
        self._on_dead = on_dead
        self._halt = threading.Event()
        self.period_s = 0.5

    def run(self) -> None:
        from torchft_b200.coordination import lighthouse_status

        while not self._halt.wait(self.period_s):
            members = self._members()  # the OTHER members of the current quorum
            if not members:
                continue
            try:
                st = lighthouse_status(self._addr, timedelta(seconds=2))
            except Exception:  # noqa: BLE001 - the lighthouse being away is not a peer failure
                continue
            self.period_s = max(0.05, min(1.0, float(st.get("heartbeat_timeout_ms", 5000)) / 4000.0))
            beats = st.get("heartbeats", {})
            for rid in members:
                hb = beats.get(rid)
                if hb is not None and not hb.get("alive", True):
                    self._on_dead(rid)
                    break

    def stop(self) -> None:
        self._halt.set()


# --------------------------------------------------------------------------- the manager
class Manager:
    """Fault-tolerant training-loop manager (see module docstring).

    The replica group's TCPStore (``store_addr:store_port`` or ``MASTER_ADDR`` /
    ``MASTER_PORT``) must already be running. When you persist periodic
    checkpoints, save and restore :meth:`state_dict` alongside the model.
    """

    def __init__(
        self,
        pg: "ProcessGroup",
        load_state_dict: Optional[Callable[[T], None]],
        state_dict: Optional[Callable[[], T]],
        min_replica_size: int,
        use_async_quorum: bool = True,
        timeout: timedelta = timedelta(seconds=60),
        quorum_timeout: timedelta = timedelta(seconds=60),
        connect_timeout: timedelta = timedelta(seconds=60),
        rank: Optional[int] = None,
        world_size: Optional[int] = None,
        world_size_mode: WorldSizeMode = WorldSizeMode.DYNAMIC,
        store_addr: Optional[str] = None,
        store_port: Optional[int] = None,
        lighthouse_addr: Optional[str] = None,
        replica_id: Optional[str] = None,
        port: Optional[int] = None,
        hostname: str = socket.gethostname(),
        heartbeat_interval: timedelta = timedelta(milliseconds=100),
        checkpoint_transport: Optional[CheckpointTransport[Dict[str, T]]] = None,
        init_sync: bool = True,
        max_retries: Optional[int] = None,
        quorum_retries: int = 0,
    ) -> None:
        """
        Args:
            pg: reconfigurable process group spanning the replica dimension
            load_state_dict / state_dict: user state hooks used to heal a recovering replica
            min_replica_size: minimum number of participating replicas for a step to commit
            use_async_quorum: compute the quorum in the background during the forward pass
            timeout: default timeout for collectives, should_commit, checkpoint ops, wrap_future
            quorum_timeout: how long to wait for a quorum (set ~1h for LocalSGD/DiLoCo)
            connect_timeout: timeout for establishing control-plane connections
            rank / world_size: rank and size WITHIN the replica group (env RANK / WORLD_SIZE)
            store_addr / store_port: the replica group's TCPStore (env MASTER_ADDR / MASTER_PORT)
            lighthouse_addr: (group rank 0) lighthouse address (env TORCHFT_LIGHTHOUSE)
            replica_id: (group rank 0) human-readable id; a uuid suffix makes restarts unique
            port: (group rank 0) manager server port (env TORCHFT_MANAGER_PORT, else ephemeral)
            checkpoint_transport: heal transport; default NVLink P2P when ``pg`` is a ``ProcessGroupB200``
                (one NVSwitch domain by construction), HTTP otherwise (works across hosts)
            init_sync: force a step-0 weight sync from the primary replica
            max_retries: raise after this many consecutive failed commits (None = never)
            quorum_retries: lighthouse quorum retries before the manager gives up
        """
        self.quorum_logger = logging.getLogger("torchft_quorums")
        self.commits_logger = logging.getLogger("torchft_commits")
        self.errors_logger = logging.getLogger("torchft_errors")

        self._replica_id = replica_id
        self._timeout = get_timeout(os.environ.get(TIMEOUT_SEC_ENV), timeout)
        self._quorum_timeout = get_timeout(os.environ.get(QUORUM_TIMEOUT_SEC_ENV), quorum_timeout)
        self._connect_timeout = get_timeout(os.environ.get(CONNECT_TIMEOUT_SEC_ENV), connect_timeout)
        self._quorum_retries = int(os.environ.get(QUORUM_RETRIES_ENV, str(quorum_retries)))
        self._original_fr_dump_temp_file = os.environ.get(TORCH_FR_DUMP_TEMP_FILE_ENV)

        # user state: key -> (load, save); reads of it (heal sends) are fenced by a reader-writer lock
        self._state_fns: Dict[str, tuple] = {}
        self._state_dict_lock = RWLock(timeout=self._timeout.total_seconds())
        self._state_reads_allowed = True
        if load_state_dict and state_dict:
            self.register_state_dict_fn("default", load_state_dict, state_dict)

        self._pg = pg
        self._use_async_quorum = use_async_quorum
        self._world_size_mode = world_size_mode
        self._init_sync = init_sync
        self._min_replica_size = min_replica_size
        self._ledger = _StepLedger(max_retries)
        self._ledger_lock = threading.RLock()
        self._deferred: Optional[_DeferredCommit] = None

        store_addr = store_addr or os.environ["MASTER_ADDR"]
        store_port = store_port or int(os.environ["MASTER_PORT"])
        self._group_rank = rank if rank is not None else int(os.environ["RANK"])
        self._group_world_size = world_size or int(os.environ["WORLD_SIZE"])

        self._checkpoint_transport: CheckpointTransport[Dict[str, T]] = (
            checkpoint_transport if checkpoint_transport is not None else self._default_transport())

        self._executor = ThreadPoolExecutor(max_workers=1, thread_name_prefix="async_quorum")
        self._quorum_future: Optional[concurrent.futures.Future] = None
        self._store = TCPStore(host_name=store_addr, port=store_port, is_master=False, wait_for_workers=False)
        self._manager: Optional[ManagerServer] = None
        self._recovery_stream: Optional[torch.cuda.Stream] = torch.cuda.Stream() if torch.cuda.is_available() else None
        self._recovery_event: Optional[torch.cuda.Event] = None
        self._commit_gate: Optional[torch.Tensor] = None
        self._liveness: Optional[_LivenessWatch] = None
        self._reported_dead: set = set()

        if self._group_rank == 0:
            if port is None:
                port = int(os.environ.get(MANAGER_PORT_ENV, 0))
            lighthouse_addr = lighthouse_addr or os.environ["TORCHFT_LIGHTHOUSE"]
            # uuid suffix: a fast restart must not be mistaken for the old incarnation
            suffix = str(uuid.uuid4())
            replica_id = suffix if not replica_id else f"{replica_id}:{suffix}"
            self._manager = ManagerServer(
                replica_id=replica_id,
                lighthouse_addr=lighthouse_addr,
                hostname=hostname,
                bind=f"[::]:{port}",
                store_addr=f"{store_addr}:{store_port}",
                world_size=self._group_world_size,
                heartbeat_interval=heartbeat_interval,
                connect_timeout=self._connect_timeout,
                quorum_retries=self._quorum_retries,
            )
            self._store.set(MANAGER_ADDR_KEY, self._manager.address())
            self._store.set(REPLICA_ID_KEY, replica_id)

        addr = self._store.get(MANAGER_ADDR_KEY).decode("utf-8")
        self._client = ManagerClient(addr, connect_timeout=self._connect_timeout)
        self._full_replica_id = self._store.get(REPLICA_ID_KEY).decode("utf-8")
        self._logger = _ManagerLogger(self, self._full_replica_id or "", self._group_rank)

        self._quorum_id = -1
        self._quorum_members: List[str] = []
        self._errored: Optional[ExceptionWithTraceback] = None
        self._healing = False
        self._serving_heal = False
        self._pending_state_dict: Optional[Dict[str, object]] = None
        self._participation = _Participation()

        self._global_rank = (
            self._group_rank
            if self._replica_id is None
            else extract_trailing_digits(self._replica_id) * self._group_world_size + self._group_rank
        )
        self._update_fr_path()

        want_watch = os.environ.get(LIVENESS_ENV)
        if (want_watch != "0" and lighthouse_addr and getattr(pg, "supports_liveness_abort", False) is True) or want_watch == "1":
            if lighthouse_addr:
                self._liveness = _LivenessWatch(lighthouse_addr, self._peers_in_quorum, self._peer_died)
                self._liveness.start()

    # ------------------------------------------------------------------ transports / state hooks
    def _default_transport(self) -> CheckpointTransport[Dict[str, T]]:
        # CUDA-IPC handles only open on the exporting host: pick the NVLink transport only when the process
        # group itself is confined to one NVSwitch domain (ProcessGroupB200); everything else gets the HTTP
        # transport, which works across hosts like the reference's default (manager.py:277-281)
        choice = os.environ.get("TORCHFT_B200_TRANSPORT", "auto")
        same_host = getattr(self._pg, "single_host", False) is True
        if torch.cuda.is_available() and (choice == "p2p" or (choice == "auto" and same_host)):
            from torchft_b200.checkpointing.p2p_transport import P2PTransport

            # receive IN PLACE into the live tensors: a heal allocates nothing
            return P2PTransport(timeout=self._timeout, state_dict=self._heal_targets)
        from torchft_b200.checkpointing.http_transport import HTTPTransport

        return HTTPTransport(timeout=self._timeout, num_chunks=0)

    def _heal_targets(self) -> Dict[str, object]:
        """Same pytree shape as ``_manager_state_dict`` (destinations for an in-place heal)."""
        return {"user": {k: save() for k, (_, save) in self._state_fns.items()}, "torchft": self.state_dict()}

    def register_state_dict_fn(self, key: str, load_state_dict: Callable[[T], None], state_dict: Callable[[], T]) -> None:
        """Add a named piece of user state that travels with live heals."""
        assert key not in self._state_fns, f"duplicate state_dict key {key}"
        self._state_fns[key] = (cast(Callable[[object], None], load_state_dict), state_dict)

    def set_state_dict_fns(self, load_state_dict: Callable[[T], None], state_dict: Callable[[], T]) -> None:
        self._logger.warn("`set_state_dict_fns` is deprecated, please use `register_state_dict_fn` instead")
        self.register_state_dict_fn("set_state_dict_fns", load_state_dict, state_dict)

    def allow_state_dict_read(self) -> None:
        """Let heal senders read the user state again (after an optimizer step)."""
        if self._state_reads_allowed:
            return
        self._state_reads_allowed = True
        self._state_dict_lock.w_release()

    def disallow_state_dict_read(self) -> None:
        """Fence heal senders out while the user state is being modified."""
        if not self._state_reads_allowed:
            return
        self._state_reads_allowed = False
        self._state_dict_lock.w_acquire()

    def _manager_state_dict(self) -> Dict[str, object]:
        with self._state_dict_lock.r_lock():
            assert self._state_fns, "user state_dict is not initialized."
            return {"user": {k: save() for k, (_, save) in self._state_fns.items()}, "torchft": self.state_dict()}

    def shutdown(self, wait: bool = True) -> None:
        """Stop the liveness watch, the checkpoint transport, the manager server and the quorum thread."""
        if self._liveness is not None:
            self._liveness.stop()
        self._checkpoint_transport.shutdown(wait=wait)
        if self._manager is not None:
            self._manager.shutdown()
        self._executor.shutdown(wait=wait)

    # ------------------------------------------------------------------ collectives
    def guarded(self, launch: Callable[[], Optional[Work]], value: object = None) -> Work:
        """Run ``launch()`` (which enqueues a collective of the fault-tolerant group and returns its ``Work``)
        under this step's error latch: after a first error nothing is launched any more, an exception is
        latched instead of raised, and the returned work's ``wait()`` never raises."""
        if self.errored():
            return DummyWork(value)
        self.wait_quorum()
        try:
            work = launch()
            return DummyWork(value) if work is None else _ManagedWork(self, work, value)
        except Exception as e:  # noqa: BLE001
            self._logger.exception(f"got exception in collective -- skipping remaining: {e}")
            self.report_error(e)
            return DummyWork(value)

    @torch.profiler.record_function("torchft::manager::allreduce")
    def allreduce(self, tensor: torch.Tensor, should_quantize: bool = False, reduce_op: ReduceOp = ReduceOp.AVG) -> Work:
        """Fault-tolerant all-reduce across the participating replicas.

        AVG divides by ``num_participants()``. Errors never raise: the first one is
        latched (``errored()``), the returned work completes, later calls are
        no-ops, and the commit decision will be negative so the (possibly
        corrupted) tensor is discarded.
        """
        if reduce_op == ReduceOp.AVG and not torch.is_floating_point(tensor):
            raise ValueError("average reduce op is only supported for floating point tensors")

        def launch() -> Work:
            n, contributing = self.num_participants(), self.is_participating()
            fused = self._fused_allreduce(tensor, should_quantize, reduce_op, n, contributing)
            if fused is not None:
                return fused
            # generic process group: zero a non-contributor, SUM, divide afterwards
            if not contributing:
                tensor.zero_()
            wire_op = ReduceOp.SUM if reduce_op == ReduceOp.AVG else reduce_op
            if should_quantize and tensor.is_cuda:
                from torchft_b200.collectives import allreduce_quantized

                return allreduce_quantized([tensor], wire_op, self._pg, torch.cuda.current_stream())
            opts = AllreduceOptions()
            opts.reduceOp = wire_op
            return self._pg.allreduce([tensor], opts)

        fused_path = self._has_fused_path(tensor, reduce_op)
        work = self.guarded(launch, tensor)
        if reduce_op == ReduceOp.AVG and not fused_path and isinstance(work, _ManagedWork):
            n = self.num_participants()

            @torch.profiler.record_function("torchft::manager::allreduce::callback")
            def normalize(fut: Future) -> torch.Tensor:
                tensor.div_(n)
                return tensor

            work.get_future().then(normalize)
        return work

    _FUSED_OPS = (ReduceOp.SUM, ReduceOp.AVG, ReduceOp.MAX, ReduceOp.MIN)

    def _has_fused_path(self, tensor: torch.Tensor, reduce_op: ReduceOp) -> bool:
        pg = self._pg
        return (getattr(pg, "allreduce_native", None) is not None and tensor.is_cuda and reduce_op in self._FUSED_OPS
                and pg._native_ok(tensor))  # type: ignore[attr-defined]

    def _fused_allreduce(self, tensor: torch.Tensor, should_quantize: bool, reduce_op: ReduceOp,
                         num_participants: int, participating: bool) -> Optional[Work]:
        """ProcessGroupB200: 1/num_participants and the zero contribution live inside the kernel."""
        if not self._has_fused_path(tensor, reduce_op):
            return None
        from torchft_b200.ops import _native

        pg = self._pg
        scale = 1.0 / max(num_participants, 1) if reduce_op == ReduceOp.AVG else 1.0
        if should_quantize and reduce_op in (ReduceOp.SUM, ReduceOp.AVG):
            return pg.allreduce_q8(tensor, tensor, None, scale=scale, contribute=participating)  # type: ignore[attr-defined]
        code = {ReduceOp.MAX: _native.OP_MAX, ReduceOp.MIN: _native.OP_MIN}.get(reduce_op, _native.OP_SUM)
        return pg.allreduce_native(tensor, op=code, scale=scale, contribute=participating)  # type: ignore[attr-defined]

    def alloc_symmetric(self, name: str, nbytes: int) -> Optional[torch.Tensor]:
        """Peer-visible buffer from the process group (``ProcessGroupB200.alloc_symmetric``) or ``None``
        when the group has no such memory. Tensors carved from it are all-reduced in place, zero-copy."""
        fn = getattr(self._pg, "alloc_symmetric", None)
        return fn(name, nbytes) if callable(fn) else None

    def supports_fused_delta(self) -> bool:
        """True when ``allreduce_delta`` runs as ONE fused kernel (ProcessGroupB200)."""
        return hasattr(self._pg, "allreduce_q8") and torch.cuda.is_available()

    @torch.profiler.record_function("torchft::manager::allreduce_delta")
    def allreduce_delta(self, out: torch.Tensor, a: torch.Tensor, b: torch.Tensor, should_quantize: bool = True) -> Work:
        """``out = AVG over replicas of (a - b)`` -- DiLoCo's pseudo-gradient reduction.

        On ProcessGroupB200 with ``should_quantize`` the subtraction, fp8 quantisation,
        exchange, fp32 reduction and dequantisation are one kernel; elsewhere this is
        ``torch.sub`` followed by :meth:`allreduce`. ``out`` may alias ``a``. Same
        error-latching contract as :meth:`allreduce`.
        """
        pg = self._pg
        if should_quantize and self.supports_fused_delta() and all(pg._native_ok(t) for t in (out, a, b)):  # type: ignore[attr-defined]
            return self.guarded(lambda: pg.allreduce_q8(out, a, b, scale=1.0 / max(self.num_participants(), 1),  # type: ignore[attr-defined]
                                                        contribute=self.is_participating()), out)
        torch.sub(a, b, out=out)
        return self.allreduce(out, should_quantize=should_quantize)

    def report_error(self, e: Exception) -> None:
        """Latch an error: the current step will not commit and the group reconfigures next step."""
        self._errored = ExceptionWithTraceback(e)

    def errored(self) -> Optional[ExceptionWithTraceback]:
        return self._errored

    def wrap_future(self, fut: Future, default: T, timeout: Optional[timedelta] = None) -> Future:
        """Future that never fails: errors/timeouts are reported to the manager and replaced by ``default``."""
        stream = torch.cuda.current_stream() if torch.cuda.is_available() else None

        def absorb(f: Future) -> T:
            with get_stream_context(stream):
                try:
                    return f.value()
                except Exception as e:  # noqa: BLE001
                    self._logger.exception(f"got exception in future -- skipping remaining: {e}")
                    self.report_error(e)
                    return default

        return future_timeout(fut, timeout or self._timeout).then(absorb)

    # ------------------------------------------------------------------ quorum
    def start_quorum(self, allow_heal: bool = True, shrink_only: bool = False, timeout: Optional[timedelta] = None) -> None:
        """Begin a new step: compute the quorum (async by default) and ready the group.

        Call before the forward pass (``OptimizerWrapper.zero_grad`` does). All
        replicas must pass the same ``allow_heal``.
        """
        if self._quorum_future is not None:
            self._quorum_future.result()
        self._errored = None
        self._healing = False
        device = torch.cuda.current_device() if torch.cuda.is_available() else -1
        self._quorum_future = self._executor.submit(self._quorum_task, allow_heal, shrink_only,
                                                    timeout or self._quorum_timeout, device)
        if not self._use_async_quorum:
            self.wait_quorum()
            if self._healing:
                # sync quorum: heal before the forward pass so this replica counts immediately
                self._install_pending_state()
                self._healing = False

    @torch.profiler.record_function("torchft::manager::wait_quorum")
    def wait_quorum(self) -> None:
        """Block until the quorum (and PG reconfiguration) for this step is done."""
        assert self._quorum_future is not None, "must call start_quorum before wait_quorum"
        self._quorum_future.result()

    @torch.profiler.record_function("torchft::manager::_async_quorum")
    def _quorum_task(self, allow_heal: bool, shrink_only: bool, quorum_timeout: timedelta, device: int) -> None:
        try:
            torch.multiprocessing._set_thread_name("torchft_quorum")
        except Exception:  # pragma: no cover
            pass
        if device >= 0 and torch.cuda.is_available():
            torch.cuda.set_device(device)

        # the previous step's device-side verdict decides which step number we report
        self._settle_deferred()

        with torch.profiler.record_function("torchft::manager::_client::_quorum"):
            with self._ledger_lock:
                step, failures = self._ledger.step, self._ledger.failures
            quorum = self._client._quorum(
                group_rank=self._group_rank,
                step=step,
                checkpoint_metadata=self._checkpoint_transport.metadata(),
                shrink_only=shrink_only,
                timeout=quorum_timeout,
                init_sync=self._init_sync,
                commit_failures=failures,
            )

        self._participation = _Participation.derive(
            quorum, everyone_counts=not (self._use_async_quorum or not allow_heal),
            mode=self._world_size_mode, cap=self._min_replica_size)
        self._quorum_members = list(quorum.replica_ids)
        self._serving_heal = bool(allow_heal and quorum.recover_dst_replica_ranks)

        if quorum.quorum_id != self._quorum_id and not self._reconfigure(quorum):
            return
        if allow_heal:
            self._recover(quorum)

    def _reconfigure(self, quorum: Any) -> bool:
        """The quorum id changed: point the process group at the new member set. False on failure (latched)."""
        gws = self._group_world_size
        global_ranks = [extract_trailing_digits(rid.split(":")[0]) * gws + self._group_rank for rid in quorum.replica_ids]
        self.quorum_logger.info("", extra={**self._log_tags(), "quorum_id": quorum.quorum_id, "step": quorum.max_step})
        prefix = f"{quorum.store_address}/torchft/{quorum.quorum_id}/{self._group_rank}"
        self._logger.info(f"reconfiguring for quorum_id={quorum.quorum_id} store_prefixed_addr={prefix!r}")
        try:
            self._quorum_id = quorum.quorum_id
            with torch.profiler.record_function("torchft::manager::_pg::configure"):
                self._pg.configure(prefix, self._replica_id if self._replica_id is not None else "0", quorum.replica_rank,
                                   quorum.replica_world_size, quorum.quorum_id, self._group_rank, gws, global_ranks)
            self._update_fr_path()
            reset = getattr(torch._C._distributed_c10d, "_reset_fr_recording_nccl", None)
            if reset is not None and "nccl" in self._pg.getBackendName():
                reset()
            return True
        except Exception as e:  # noqa: BLE001
            self._logger.exception(f"got exception in pg configure: {e}")
            self.report_error(e)
            return False

    def _recover(self, quorum: Any) -> None:
        """Serve our state to replicas that are behind and/or fetch it if we are (on the recovery stream)."""
        transport = self._checkpoint_transport
        with get_stream_context(self._recovery_stream):
            try:
                if quorum.recover_dst_replica_ranks:
                    self._logger.info(f"peers need recovery from us {quorum.recover_dst_replica_ranks}")
                    with torch.profiler.record_function("torchft::manager::_checkpoint_transport::send_checkpoint"):
                        transport.send_checkpoint(dst_ranks=quorum.recover_dst_replica_ranks, step=quorum.max_step,
                                                  state_dict=self._manager_state_dict(), timeout=self._timeout)
                if quorum.heal:
                    self._healing = True
                    src = quorum.recover_src_replica_rank
                    assert src is not None, "must have a recover rank when healing"
                    self._logger.info(f"healing required, fetching checkpoint metadata from "
                                      f"src_addr={quorum.recover_src_manager_address!r} max_step={quorum.max_step}")
                    peer = ManagerClient(quorum.recover_src_manager_address, connect_timeout=self._connect_timeout)
                    metadata = peer._checkpoint_metadata(self._group_rank, timeout=self._timeout)
                    with torch.profiler.record_function("torchft::manager::_checkpoint_transport::recv_checkpoint"):
                        # staged; the user part is installed on the main thread at commit time
                        self._pending_state_dict = transport.recv_checkpoint(
                            src_rank=src, metadata=metadata, step=quorum.max_step, timeout=self._timeout)
                    self.load_state_dict(cast(Dict[str, int], self._pending_state_dict["torchft"]))
                    with self._ledger_lock:
                        self._ledger.step = quorum.max_step
            except Exception as e:  # noqa: BLE001
                self._logger.exception(f"got exception in recovery: {e}")
                self.report_error(e)
            if self._recovery_stream is not None:
                self._recovery_event = torch.cuda.current_stream().record_event()

    def _update_fr_path(self) -> None:
        """Flight-recorder dumps go to ``<TORCH_FR_DUMP_TEMP_FILE>_quorum_<id>/<global_rank>``."""
        if self._original_fr_dump_temp_file is not None:
            folder = f"{self._original_fr_dump_temp_file}_quorum_{self._quorum_id}"
            os.makedirs(folder, exist_ok=True)
            os.environ[TORCH_FR_DUMP_TEMP_FILE_ENV] = f"{folder}/{self._global_rank}"

    def _install_pending_state(self) -> None:
        """Main thread: hand the staged checkpoint to the user's load functions."""
        assert self._healing, "must be in healing state"
        self.wait_quorum()
        staged, self._pending_state_dict = self._pending_state_dict, None
        if staged is None:
            assert self.errored(), "checkpoint was not staged and no error occured"
            return
        assert self._state_fns, "user load_state_dict is not initialized."
        self._logger.info("applying pending state dict")
        user = cast(Dict[str, object], staged["user"])
        for key, (load, _) in self._state_fns.items():
            load(user[key])
        self._logger.info("Loaded state dict.")

    # ------------------------------------------------------------------ liveness
    def _peers_in_quorum(self) -> List[str]:
        return [rid for rid in self._quorum_members if rid != self._full_replica_id]

    def _peer_died(self, replica_id: str) -> None:
        # NOT pg.errored(): on the native group that synchronises the comm stream -- i.e. it would wait for the very kernel
        # that is spinning on the dead peer (measured: the abort then only fired after the full collective timeout)
        if replica_id not in self._reported_dead:
            self._reported_dead.add(replica_id)
            self._logger.warn(f"lighthouse lost the heartbeat of {replica_id}: aborting in-flight collectives")
            self.errors_logger.info("", extra={**self._log_tags(), "quorum_id": self._quorum_id, "step": self._ledger.step,
                                               "error": f"peer {replica_id} stopped heart-beating"})
        self._pg.abort()

    # ------------------------------------------------------------------ commit
    def _log_tags(self) -> Dict[str, object]:
        return {"job_id": os.environ.get("JOB_ID", "unknown"), "replica_id": self._replica_id, "rank": self._group_rank}

    def _drain_and_collect_errors(self) -> None:
        """Host-synchronous prelude of a commit: recovery stream, current stream, latched PG error, staged heal."""
        with torch.profiler.record_function("torchft::manager::should_commit::recovery_stream::synchronize"):
            ev, self._recovery_event = self._recovery_event, None
            if ev is not None:
                ev.synchronize()
        with torch.profiler.record_function("torchft::manager::should_commit::current_stream::synchronize"):
            if torch.cuda.is_available():
                synchronize()
        err = self._pg.errored()
        if err:
            self.report_error(err)
        if self._healing:
            self._install_pending_state()

    def _local_verdict(self) -> bool:
        return self.num_participants() >= self._min_replica_size and self._errored is None

    @torch.profiler.record_function("torchft::manager::should_commit")
    def should_commit(self, timeout: Optional[timedelta] = None) -> bool:
        """Decide (identically on every rank of the group) whether to step the optimizer.

        Call once per step after backward and before ``optimizer.step()``; only step
        when this returns True. Raises ``RuntimeError`` after more than ``max_retries``
        consecutive failures.
        """
        self._settle_deferred()
        self._drain_and_collect_errors()
        mine = self._local_verdict()
        verdict = self._client.should_commit(self._group_rank, self._ledger.step, mine, timeout=timeout or self._timeout)
        self._logger.info(f"should_commit={verdict} enough_replicas={self.num_participants() >= self._min_replica_size}, "
                          f"errored={self._errored}")
        self._checkpoint_transport.disallow_checkpoint()
        if self._commit_gate is not None:
            self._commit_gate.fill_(1 if verdict else 0)
        with self._ledger_lock:
            self._ledger.record(verdict, self.num_participants(), {**self._log_tags(), "quorum_id": self._quorum_id})
        return verdict

    def commit_on_device(self, committer: Any) -> Optional[bool]:
        """Commit decision WITHOUT a host round trip (replica groups of one rank; see module docstring).

        ``committer`` enqueues the verdict kernel and later reports its result::

            seq = committer.enqueue(host_ok)      # kernel on the committer's stream; gate word on the device
            committer.wait(seq, timeout) -> bool  # block the CALLING thread until the verdict is on the host
            committer.resolved(verdict)           # bookkeeping hook once the manager has recorded it

        Returns ``None`` when the verdict was deferred (normal steps) and the verdict itself when this step
        had to be resolved synchronously (this replica is healing or is serving a checkpoint, where the
        reference's ordering -- install state / close the checkpoint window around the decision -- matters).
        """
        if self._group_world_size != 1:
            raise RuntimeError("commit_on_device needs a replica group of one rank; use should_commit()")
        self._settle_deferred()
        self.wait_quorum()
        synchronous = self._healing or self._serving_heal
        if synchronous:
            self._drain_and_collect_errors()
        seq = committer.enqueue(self._local_verdict())
        with self._ledger_lock:
            self._deferred = _DeferredCommit(committer, seq, self.num_participants(),
                                             {**self._log_tags(), "quorum_id": self._quorum_id})
        if not synchronous:
            return None
        verdict = self._settle_deferred()
        self._checkpoint_transport.disallow_checkpoint()
        return verdict

    def _settle_deferred(self) -> Optional[bool]:
        """Fetch the outstanding device-side verdict (if any) and book it. Safe from any thread."""
        with self._ledger_lock:
            d, self._deferred = self._deferred, None
            if d is None:
                return None
            try:
                verdict = bool(d.committer.wait(d.seq, self._timeout))
            except Exception as e:  # noqa: BLE001 - a verdict that never arrives is a failed step
                self._logger.exception(f"device commit verdict unavailable: {e}")
                verdict = False
            if not verdict:
                err = self._pg.errored()
                if err is not None:
                    self.errors_logger.info("", extra={**d.tags, "step": self._ledger.step, "error": str(err)})
            d.committer.resolved(verdict)
            self._ledger.record(verdict, d.participants, d.tags)
            return verdict

    def commit_gate(self) -> torch.Tensor:
        """Device int32 that ``should_commit`` sets to 1/0: lets a fused optimizer kernel be gated
        on the verdict (``FlatAdamW.step(gate=manager.commit_gate())``)."""
        if self._commit_gate is None:
            dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
            self._commit_gate = torch.zeros(1, dtype=torch.int32, device=dev)
        return self._commit_gate

    # ------------------------------------------------------------------ state / accessors
    def load_state_dict(self, state_dict: Dict[str, int]) -> None:
        with self._ledger_lock:
            self._ledger.step = state_dict["step"]
            self._ledger.batches = state_dict["batches_committed"]

    def state_dict(self) -> Dict[str, int]:
        """``{"step", "batches_committed"}`` -- persist with your periodic checkpoints."""
        self._settle_deferred()
        return {"step": self._ledger.step, "batches_committed": self._ledger.batches}

    def current_step(self) -> int:
        """Committed steps so far (resolves an outstanding device-side verdict first)."""
        self._settle_deferred()
        return self._ledger.step

    def batches_committed(self) -> int:
        """Total batches committed across all replicas and steps."""
        self._settle_deferred()
        return self._ledger.batches

    # kept as attributes of long standing (tests and user code read them)
    @property
    def _step(self) -> int:
        return self._ledger.step

    @_step.setter
    def _step(self, v: int) -> None:
        self._ledger.step = v

    @property
    def _batches_committed(self) -> int:
        return self._ledger.batches

    @property
    def _commit_failures(self) -> int:
        return self._ledger.failures

    def participating_rank(self) -> Optional[int]:
        """This replica's rank among the participants (None if not participating). Blocks on the quorum."""
        if self._quorum_future is None:
            return None
        self.wait_quorum()
        return self._participation.rank

    def num_participants(self) -> int:
        """Number of replicas contributing to this step. Blocks on the quorum."""
        if self._quorum_future is None:
            return 0
        self.wait_quorum()
        assert self._participation.world >= 0, "internal error"
        return self._participation.world

    def is_participating(self) -> bool:
        if self._participation.rank is None:
            return False
        if self._healing:
            assert self._use_async_quorum
            return False
        return True

    # reference attribute names, for code that pokes at them
    @property
    def _participating_replica_rank(self) -> Optional[int]:
        return self._participation.rank

    @property
    def _participating_replica_world_size(self) -> int:
        return self._participation.world


class _ManagerLogger:
    """``[replica/rank - step N]``-prefixed logging."""

    def __init__(self, manager: Manager, replica_id: str, group_rank: int) -> None:
        self._logger = logging.getLogger(__name__)
        self._who = f"{replica_id}/{group_rank}"
        self._manager = weakref.ref(manager)

    def _fmt(self, msg: str) -> str:
        m = self._manager()
        return f"[{self._who} - step {m._ledger.step if m is not None else '?'}] {msg}"

    def info(self, msg: str) -> None:
        self._logger.info(self._fmt(msg))

    def warn(self, msg: str) -> None:
        self._logger.warning(self._fmt(msg))

    def exception(self, msg: str) -> None:
        self._logger.exception(self._fmt(msg))


# ------------------------------------------------------------------ managed work
class _ValueFuture(Future):
    """Minimal future handed to chained callbacks: only ``value()`` is meaningful (never blocks)."""

    def __init__(self, value: object) -> None:
        super().__init__()
        self._v = value

    def value(self) -> object:
        return self._v

    def wait(self) -> object:
        return self._v


class _ManagedFuture(Future):
    """Handle into a :class:`_ManagedWork` callback pipeline.

    ``then(cb)`` only *records* ``cb`` (lazily, nothing runs and the host never
    blocks); the pipeline executes when the work is waited on. ``wait()`` resolves
    the pipeline and returns its final value.
    """

    def __init__(self, work: "weakref.ReferenceType[_ManagedWork]") -> None:
        super().__init__()
        self._work = work

    def _owner(self) -> "_ManagedWork":
        w = self._work()
        assert w is not None, "managed work was garbage collected"
        return w

    def then(self, callback: Callable[[Future], S]) -> Future:  # type: ignore[override]
        w = self._owner()
        w._callbacks.append(callback)
        return _ManagedFuture(self._work)

    def wait(self) -> object:  # type: ignore[override]
        w = self._owner()
        w._materialize()
        assert w._final is not None
        return w._final.wait()

    def value(self) -> object:  # type: ignore[override]
        raise NotImplementedError("use wait(); this future only builds the callback pipeline")

    def done(self) -> bool:  # type: ignore[override]
        raise NotImplementedError("use wait(); this future only builds the callback pipeline")

    def add_done_callback(self, callback: Callable[[Future], None]) -> None:  # type: ignore[override]
        raise NotImplementedError("use then(); this future only builds the callback pipeline")

    def set_result(self, result: object) -> None:  # type: ignore[override]
        raise NotImplementedError("managed futures are completed by their work")

    def set_exception(self, result: object) -> None:  # type: ignore[override]
        raise NotImplementedError("managed futures are completed by their work")


class _ManagedWork(Work):
    """``Work`` whose ``wait()`` never raises and whose continuation callbacks run on the
    launching stream AFTER a stream dependency on the collective has been established.

    Callbacks registered through ``get_future().then(...)`` are kept in a list and
    composed into one continuation the first time the work is waited on; that
    continuation is routed through ``Manager.wrap_future`` so a failure or timeout
    anywhere in the pipeline is reported to the manager and swallowed.
    """

    def __init__(self, manager: Manager, work: Work, value: object) -> None:
        super().__init__()
        self._manager = manager
        self._inner = work
        self._value = value
        self._callbacks: List[Callable[[Future], object]] = []
        self._final: Optional[Future] = None
        self._stream: Optional[torch.cuda.Stream] = torch.cuda.current_stream() if torch.cuda.is_available() else None

    def _materialize(self) -> None:
        if self._final is not None:
            return
        fut = self._inner.get_future()
        callbacks, value, stream = list(self._callbacks), self._value, self._stream

        def pipeline(f: Future) -> object:
            with get_stream_context(stream):
                f.wait()  # stream dependency on the collective, not a host block for CUDA futures
                v = value
                for cb in callbacks:
                    v = cb(_ValueFuture(v))
                return v

        self._final = self._manager.wrap_future(fut.then(pipeline), value)

    def _assert_same_stream(self) -> None:
        if self._stream is not None:
            assert self._stream == torch.cuda.current_stream(), "wait on the stream that launched the collective"

    def wait(self, timeout: Optional[timedelta] = None) -> bool:
        self._assert_same_stream()
        try:
            with get_stream_context(self._stream):
                self._inner.wait()
                self._materialize()
                assert self._final is not None
                self._final.wait()
            return True
        except Exception as e:  # noqa: BLE001
            self._manager._logger.exception(f"got exception waiting for work {e}")
            self._manager.report_error(e)
            return False

    def block_current_stream(self, timeout: Optional[timedelta] = None) -> None:
        self._assert_same_stream()
        with get_stream_context(self._stream):
            blk = getattr(self._inner, "block_current_stream", None)
            if blk is not None and self._stream is not None:
                blk()
            else:  # no accelerator stream to block: fall back to a host wait
                self._inner.wait()
        self._materialize()

    def synchronize(self) -> None:
        self._assert_same_stream()
        if torch.cuda.is_available():
            self.block_current_stream()
        else:
            self._materialize()

    def get_future(self) -> Future:
        return _ManagedFuture(weakref.ref(self))
