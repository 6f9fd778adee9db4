"""NVLink peer-memory manager + collectives for one replica-group rank.

This is the native replacement for "destroy and re-create the NCCL
communicator on every quorum change" (reference:
torchft/process_group.py:435-471,848-873). The CUDA context, streams, local
segments and the signal pad survive reconfiguration; ``configure()`` only

1. publishes this rank's segment descriptors (CUDA IPC handles) under the
   per-quorum store prefix,
2. maps segments of peers that are NEW to the quorum and unmaps those that left
   (handles of surviving peers are cached and reused), and
3. agrees on a flag floor so the epoch-tagged signal protocol restarts cleanly.

Failure containment: every in-kernel wait is a bounded, abortable spin on a
host-mapped status block (see ``csrc/kernels/common.cuh``), so a dead peer
produces a latched error (``errored()``) rather than a wedged stream --
the analogue of ``ncclCommAbort`` without tearing anything down.
"""

from __future__ import annotations

import json
import contextlib
import logging
import os
import socket
import threading
import time
from dataclasses import dataclass
from datetime import timedelta
from typing import Any, Dict, List, Optional, Tuple

import torch

from torchft_b200.ops import _native

logger = logging.getLogger(__name__)

_CH_ALLREDUCE = 0
_CH_Q8 = 1
_CH_HEAL = 2
_CH_USER = 3

_ALIGN = 2 << 20  # segment sizes rounded to 2 MiB (the VMM allocation granularity on H100)


class _CAI:
    """Minimal ``__cuda_array_interface__`` carrier to view raw device memory as a tensor."""

    def __init__(self, ptr: int, nbytes: int) -> None:
        self.__cuda_array_interface__ = {
            "shape": (nbytes,),
            "typestr": "|u1",
            "data": (ptr, False),
            "version": 3,
            "strides": None,
        }


def tensor_from_ptr(ptr: int, nbytes: int, device: torch.device) -> torch.Tensor:
    return torch.as_tensor(_CAI(ptr, nbytes), device=device)


@dataclass
class Segment:
    """A device region exported to peers: cudaMalloc + CUDA IPC ("ipc" mode) or a refcounted VMM
    allocation shared as a POSIX fd ("vmm" mode; required for NVLS multicast)."""

    name: str
    ptr: int
    nbytes: int
    handle: bytes
    tensor: torch.Tensor  # uint8 view keeping python-side references simple
    mem_handle: int = 0   # CUmemGenericAllocationHandle (vmm mode)
    fd: int = -1          # exported descriptor (vmm mode)

    def contains(self, p: int, n: int) -> bool:
        return self.ptr <= p and p + n <= self.ptr + self.nbytes


class SymmetricComm:
    """Peer-memory communicator over the current healthy replica set."""

    def __init__(
        self,
        device: Optional[torch.device] = None,
        staging_bytes: Optional[int] = None,
        timeout: timedelta = timedelta(seconds=60),
    ) -> None:
        self._K = _native.load()
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._lock = threading.RLock()
        self._status = None
        self._segments: Dict[str, Segment] = {}
        self._peer_ptrs: Dict[Tuple[str, int, bytes], int] = {}  # (host, pid, handle) -> mapped ptr
        self._tables: Dict[str, Any] = {}
        self._rank = 0
        self._world = 1
        self._epoch = 0
        self._flag = 0
        self._configured = False
        self._timeout = timeout
        if staging_bytes is None:
            staging_bytes = int(os.environ.get("TORCHFT_B200_STAGING_MB", "256")) << 20
        self._staging_bytes = (staging_bytes + _ALIGN - 1) // _ALIGN * _ALIGN
        # the tail of the staging buffer holds one send/recv mailbox per source rank; collectives use the head
        self._mailbox_bytes = min(4 << 20, (self._staging_bytes // 4 // 8) & ~15)
        self._mailbox_off = self._staging_bytes - 8 * self._mailbox_bytes
        self._staging_usable = self._mailbox_off
        self._send_seq: Dict[int, int] = {}
        self._recv_seq: Dict[int, int] = {}
        self._pad_bytes = (self._K.SIGNAL_PAD_BYTES + 65535) // 65536 * 65536
        self._max_blocks = max(1, min(int(os.environ.get("TORCHFT_B200_AR_BLOCKS", "64")), self._K.MAX_BLOCKS))
        self._q8_max_blocks = self._K.NUM_SMS  # phases A/C of the fp8 kernel are local HBM passes: use the whole chip
        self._threads = int(os.environ.get("TORCHFT_B200_AR_THREADS", "512"))
        self._oneshot_max = int(os.environ.get("TORCHFT_B200_ONESHOT_KB", "256")) << 10
        # "vmm": cuMemCreate-backed segments (survive exporter death, NVLS-capable); "ipc": cudaMalloc + cudaIpc
        self._mode = os.environ.get("TORCHFT_B200_SYMM", "ipc")
        self._nvls_enabled = os.environ.get("TORCHFT_B200_NVLS", "1") != "0"
        # NVLS threshold; None = pick by world size at configure() (see _default_nvls_min)
        env_nvls = os.environ.get("TORCHFT_B200_NVLS_MIN_KB")
        self._nvls_min_env: Optional[int] = (int(env_nvls) << 10) if env_nvls is not None else None
        self._nvls_min = self._nvls_min_env if self._nvls_min_env is not None else (1 << 62)
        self._fdserver: Any = None
        self._peer_vmm: Dict[Tuple[str, int, str], Tuple[int, int, int]] = {}  # (host, pid, seg) -> (va, handle, size)
        self._mc: Dict[str, Tuple[int, int, int]] = {}  # segment -> (mc handle, multicast va, size)
        self._mc_gen, self._mc_members = "", ""  # creation the objects in _mc belong to / the member list they span
        self._barrier_mode = int(os.environ.get("TORCHFT_B200_BARRIER_MODE", "2"))
        self._force_plan: Optional[Tuple[int, int]] = None  # (algo, blocks) override for tuning sweeps
        self.launches = 0  # native kernel launches issued (bench reports this)
        self._ptrs: Dict[str, List[int]] = {}  # segment -> mapped base pointer per quorum rank
        self._z1_ok_buf: Optional[torch.Tensor] = None
        self._commit_seq = 0
        self._hostname = socket.gethostname()

    # ------------------------------------------------------------------ memory
    def _ensure_core(self) -> None:
        if self._status is None:
            with torch.cuda.device(self.device):
                self._status = self._K.Status()
                self._status.set_timeout_ms(self._timeout.total_seconds() * 1e3)
                self._alloc_segment("core", self._pad_bytes + self._staging_bytes)

    def _alloc_segment(self, name: str, nbytes: int) -> Segment:
        nbytes = (nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        K = self._K
        with torch.cuda.device(self.device):
            if self._mode == "vmm":
                if self._fdserver is None:
                    self._fdserver = K.FdServer()
                gran = K.vmm_granularity()
                if self._nvls_enabled and K.multicast_supported():
                    gran = max(gran, K.mc_granularity(2, max(nbytes, gran)))
                nbytes = (nbytes + gran - 1) // gran * gran
                ptr, size, mem_handle, fd = K.vmm_alloc(nbytes)
                self._fdserver.publish(name, fd)
                seg = Segment(name, ptr, size, b"", tensor_from_ptr(ptr, size, self.device), mem_handle, fd)
            else:
                ptr = K.symm_alloc(nbytes)
                handle = K.ipc_get_handle(ptr)
                seg = Segment(name, ptr, nbytes, handle, tensor_from_ptr(ptr, nbytes, self.device))
        self._segments[name] = seg
        return seg

    def alloc(self, name: str, nbytes: int) -> torch.Tensor:
        """Allocate a symmetric (peer-visible) segment; returns a uint8 tensor.

        Call with the same ``name``/``nbytes`` on every replica. Peers learn about segments at ``configure()``: a
        segment becomes symmetric (zero-copy collectives, peer pointers) at the first quorum in which EVERY rank has it.
        Allocating after the group was configured is allowed; until the next quorum change tensors carved from the new
        segment are ordinary device memory to the collectives (they go through the staging buffer) and
        :meth:`is_symmetric` says so. Code that NEEDS peer pointers (FT-ZeRO-1) allocates before the first quorum.
        """
        with self._lock:
            self._ensure_core()
            if name in self._segments:
                raise ValueError(f"symmetric segment {name!r} already exists")
            seg = self._alloc_segment(name, nbytes)
            return seg.tensor[:nbytes]

    def is_symmetric(self, name: str) -> bool:
        """True once segment ``name`` is mapped by (and from) every rank of the current quorum."""
        return name in self._tables

    def set_timeout(self, timeout: timedelta) -> None:
        self._timeout = timeout
        if self._status is not None:
            self._status.set_timeout_ms(timeout.total_seconds() * 1e3)
        for t in self._tables.values():
            t.set_timeout_ms(timeout.total_seconds() * 1e3)

    # --------------------------------------------------------------- configure
    def configure(self, store: Any, rank: int, world: int, epoch: int) -> None:
        """(Re)map peer memory for a new quorum. ``store`` is any c10d Store scoped to the quorum."""
        K = self._K
        with self._lock:
            self._ensure_core()
            with torch.cuda.device(self.device):
                # Drain in-flight collectives of the old quorum (they either
                # finished or bailed out through the abort flag).
                torch.cuda.synchronize(self.device)
                self._status.clear()
                desc = {
                    "host": self._hostname,
                    "pid": os.getpid(),
                    "device": self.device.index,
                    "floor": self._flag,
                    "mode": self._mode,
                    "fd_server": self._fdserver.name() if self._fdserver is not None else "",
                    "mc_gen": self._mc_gen,
                    "segments": {n: {"handle": s.handle.hex(), "nbytes": s.nbytes} for n, s in self._segments.items()},
                }
                store.set(f"symm/{rank}", json.dumps(desc))
                descs: List[Dict[str, Any]] = []
                for r in range(world):
                    descs.append(desc if r == rank else json.loads(bytes(store.get(f"symm/{r}")).decode()))
                # symmetric = registered by EVERY rank of this quorum (a replica may have allocated a segment after its
                # peers' last configure, or not yet): the rest stays local-only until a later quorum
                names = sorted(n for n in self._segments if all(n in d["segments"] for d in descs))
                if "core" not in names:
                    raise RuntimeError("a quorum member has no core segment")
                for r, d in enumerate(descs):
                    for n in names:
                        if d["segments"][n]["nbytes"] != self._segments[n].nbytes:
                            raise RuntimeError(f"segment {n!r} size mismatch on rank {r}")
                late = sorted(set(self._segments) - set(names))
                if late:
                    logger.warning("symmetric segments %s are not registered on every replica yet: staged path until "
                                   "the next quorum change", late)
                needed: Dict[Tuple[str, int, bytes], int] = {}
                needed_vmm: Dict[Tuple[str, int, str], Tuple[int, int, int]] = {}
                ptrs: Dict[str, List[int]] = {n: [] for n in names}
                for r, d in enumerate(descs):
                    if d.get("mode", "ipc") != self._mode:
                        raise RuntimeError(f"rank {r} uses symmetric-memory mode {d.get('mode')!r}, we use {self._mode!r}")
                    for n in names:
                        if r == rank:
                            ptrs[n].append(self._segments[n].ptr)
                            continue
                        if d["host"] != self._hostname:
                            raise RuntimeError("peer-memory transport requires all replicas on one NVSwitch domain (same host)")
                        if self._mode == "vmm":
                            vkey = (d["host"], int(d["pid"]), n)
                            ent = self._peer_vmm.get(vkey)
                            if ent is None:
                                fd = K.fetch_fd(d["fd_server"], n)
                                va, h = K.vmm_import(fd, self._segments[n].nbytes)
                                ent = (va, h, self._segments[n].nbytes)
                            needed_vmm[vkey] = ent
                            ptrs[n].append(ent[0])
                            continue
                        h = bytes.fromhex(d["segments"][n]["handle"])
                        key = (d["host"], int(d["pid"]), h)
                        if d["host"] != self._hostname:
                            raise RuntimeError("peer-memory transport requires all replicas on one NVSwitch domain (same host)")
                        p = self._peer_ptrs.get(key)
                        if p is None:
                            p = K.ipc_open_handle(h)
                        needed[key] = p
                        ptrs[n].append(p)
                # unmap peers that left the quorum
                for key, p in list(self._peer_ptrs.items()):
                    if key not in needed:
                        try:
                            K.ipc_close_handle(p)
                        except RuntimeError:
                            pass  # exporter already gone
                self._peer_ptrs = needed
                for vkey, (va, h, size) in list(self._peer_vmm.items()):
                    if vkey not in needed_vmm:
                        K.vmm_unmap(va, size, h)  # our reference kept the memory alive even if the peer died
                self._peer_vmm = needed_vmm
                self._install(ptrs, rank, world, int(epoch), max(int(d["floor"]) for d in descs))
                if self._mode == "vmm" and self._nvls_enabled and world > 1 and K.multicast_supported():
                    self._setup_multicast(store, descs, [n for n in names if n != "core"], rank, world)
                else:
                    self._release_multicast()
                self._configured = True

    def _install(self, ptrs: Dict[str, List[int]], rank: int, world: int, epoch: int, floor: int,
                 pads: Optional[List[int]] = None) -> None:
        """Build the per-segment peer tables from mapped base pointers and restart the flag sequence."""
        K = self._K
        self._ptrs = ptrs
        core_ptrs = ptrs["core"]
        if pads is None:
            pads = core_ptrs  # signal pad sits at offset 0 of the core segment
        self._tables = {}
        base = K.PeerTable([p + self._pad_bytes for p in core_ptrs], pads, rank, world)
        base.set_timeout_ms(self._timeout.total_seconds() * 1e3)
        self._tables["core"] = base
        for n in ptrs:
            if n != "core":
                self._tables[n] = base.with_data(ptrs[n])
        self._flag = max(floor, int(epoch) << 32) + 16
        self._rank, self._world, self._epoch = rank, world, int(epoch)
        self._send_seq, self._recv_seq = {}, {}
        self._nvls_min = self._nvls_min_env if self._nvls_min_env is not None else self._default_nvls_min(world)

    @staticmethod
    def virtual_world(world: int, segments: Dict[str, int], device: Optional[torch.device] = None,
                      presignal: bool = True, timeout: timedelta = timedelta(seconds=10),
                      staging_bytes: int = 8 << 20) -> "List[SymmetricComm]":
        """``world`` ranks of ONE quorum inside this process, all on ``device`` (testing / self-check harness).

        Every rank gets its own segments and signal pad; the peer tables point at each other directly (no IPC).
        With ``presignal`` every flag slot is pre-set to "arrived", so a rank's kernel never waits: because each
        collective only ever reads slice r of all buffers and writes slice r back (or, one-shot, writes nothing
        shared), running rank 0's kernel, then rank 1's, ... reproduces the W-rank result exactly -- in one
        process, one kernel at a time, which is what profilers (ncu serialises launches), compute-sanitizer and
        the one-GPU test tier need. With ``presignal=False`` the ranks synchronise for real and must be launched
        concurrently on different streams.
        """
        comms = [SymmetricComm(device, staging_bytes=staging_bytes, timeout=timeout) for _ in range(world)]
        for c in comms:
            c._mode = "ipc"
            # all ranks share ONE GPU: with real signalling every CTA of every rank must be resident at once
            c._max_blocks = c._q8_max_blocks = max(2, 112 // world)
            c._ensure_core()
            for name, nbytes in segments.items():
                c._alloc_segment(name, nbytes)
        names = list(comms[0]._segments)
        ptrs = {n: [c._segments[n].ptr for c in comms] for n in names}
        for r, c in enumerate(comms):
            pads = None
            if presignal:
                # own pad: every slot reads "arrived" (>= any flag) and "verdict ok" (odd) forever; the flags this rank
                # publishes go to a private sink instead of the peers' pads, so nothing ever un-signals a slot
                pad = c._segments["core"].tensor[: c._K.SIGNAL_PAD_BYTES].view(torch.int64)
                pad.fill_((1 << 62) | 1)
                c._sink = torch.zeros(c._K.SIGNAL_PAD_BYTES, dtype=torch.uint8, device=c.device)
                pads = [c._segments["core"].ptr if t == r else c._sink.data_ptr() for t in range(world)]
            c._install({n: list(v) for n, v in ptrs.items()}, r, world, epoch=1, floor=0, pads=pads)
            c._configured = True
        torch.cuda.synchronize(comms[0].device)
        return comms

    def segment(self, name: str) -> torch.Tensor:
        """uint8 view of this rank's segment ``name``."""
        return self._segments[name].tensor

    # --------------------------------------------------------------- multicast
    def _store_barrier(self, store: Any, key: str, world: int) -> None:
        n = store.add(key, 1)
        deadline = time.monotonic() + self._timeout.total_seconds()
        while n < world:
            if time.monotonic() > deadline:
                raise TimeoutError(f"store barrier {key} timed out ({n}/{world})")
            time.sleep(0.0005)
            n = store.add(key, 0)

    def _setup_multicast(self, store: Any, descs: List[Dict[str, Any]], names: List[str], rank: int, world: int) -> None:
        """One NVLS multicast object per user segment over the CURRENT quorum. Objects are bound to a fixed device set,
        so a membership change re-creates them -- all segments in one round (two store barriers in total, not two per
        segment) -- and a quorum whose members all still hold the objects of the same earlier creation keeps them."""
        K = self._K
        members = json.dumps([[d["host"], int(d["pid"])] for d in descs])
        gens = {d.get("mc_gen", "") for d in descs}
        if self._mc and len(gens) == 1 and self._mc_gen in gens and self._mc_gen and self._mc_members == members:
            return  # every rank reports the same live creation over the same members: nothing to rebuild
        self._release_multicast()
        gen = f"mc:{self._epoch}:{self._flag}"
        keys = {n: f"{gen}:{n}" for n in names}
        mcs: Dict[str, int] = {}
        if rank == 0:
            for n in names:
                mc, fd = K.mc_create(world, self._segments[n].nbytes)
                self._fdserver.publish(keys[n], fd)
                mcs[n] = mc
            store.set("mcready", gen)
        else:
            gen = bytes(store.get("mcready")).decode()
            keys = {n: f"{gen}:{n}" for n in names}
            for n in names:
                mcs[n] = K.mc_import(K.fetch_fd(descs[0]["fd_server"], keys[n]))
        for n in names:
            K.mc_add_device(mcs[n])
        self._store_barrier(store, "mcadd", world)
        for n in names:
            seg = self._segments[n]
            self._mc[n] = (mcs[n], K.mc_bind_and_map(mcs[n], seg.mem_handle, seg.nbytes), seg.nbytes)
        self._store_barrier(store, "mcbind", world)
        if rank == 0:
            for n in names:
                self._fdserver.unpublish(keys[n])
        self._mc_gen, self._mc_members = gen, members

    def _release_multicast(self) -> None:
        for n, (mc, va, size) in list(self._mc.items()):
            try:
                self._K.mc_release(mc, va, size)
            except Exception:  # noqa: BLE001
                pass
        self._mc = {}
        self._mc_gen, self._mc_members = "", ""

    # ------------------------------------------------------------- collectives
    def _plan(self, nbytes: int) -> Tuple[int, int]:
        """(algo, blocks): identical on every rank for a given message size.

        Thresholds from a ``bench/comm_tune.py`` sweep on an earlier NVLink generation; not re-measured on H100. One-shot (each
        rank reads the whole message from every peer; two flag exchanges, no write-back hop)
        wins while (world-1) x bytes still fits the latency budget; it likes MANY small CTAs
        (16 KB each, <= 64 KB because results stay in registers across the closing barrier).
        Two-shot moves 2(N-1)/N of the bytes using both link directions; one CTA per 64 KB up
        to ``max_blocks`` (a comm kernel that overlaps backward should not take every SM).
        """
        if self._force_plan is not None:
            return self._force_plan
        w = max(self._world, 2)
        oneshot_max = self._oneshot_max * (8 if w == 2 else (4 if w <= 4 else 1))  # W=8: two-shot wins from 256 KB
        if nbytes <= oneshot_max:
            blocks = max(1, min(128, (nbytes + (16 << 10) - 1) // (16 << 10)))
            if (nbytes + blocks - 1) // blocks <= (64 << 10):
                return 0, blocks
        blocks = max(8, min(self._max_blocks, nbytes // (64 << 10)))
        return 1, blocks

    @staticmethod
    def _default_nvls_min(world: int) -> int:
        """In-switch reduction moves ~(1 + 1/N)·S per link direction, the P2P two-shot 2(N-1)/N·S: equal at
        N=4, 1.5x worse at N=2, 1.3x better at N=8, so NVLS is used from 5 ranks (and from 256 KB) up."""
        return (256 << 10) if world >= 5 else (1 << 62)

    def _next_flag(self) -> int:
        f = self._flag
        self._flag += 2
        return f

    def _segment_of(self, t: torch.Tensor) -> Optional[Tuple[Segment, int]]:
        """(segment, byte offset) if ``t`` lives in a segment that is mapped on every rank of the current quorum."""
        p, n = t.data_ptr(), t.numel() * t.element_size()
        for s in self._segments.values():
            if s.contains(p, n):
                return (s, p - s.ptr) if s.name in self._tables else None
        return None

    def allreduce_(self, t: torch.Tensor, op: int = _native.OP_SUM, scale: float = 1.0,
                   contribute: bool = True, stream: Optional[torch.cuda.Stream] = None) -> None:
        """In-place all-reduce of ``t`` over the current quorum on ``stream``.

        ``scale`` is fused (1/num_participants for AVG); ``contribute=False`` makes
        this rank add zeros (healing / spare replica) without touching ``t`` first.
        """
        K = self._K
        if not t.is_cuda or not t.is_contiguous():
            raise ValueError("allreduce_ needs a contiguous CUDA tensor")
        dt = _native.dtype_code(t)
        sp = _native.stream_ptr(stream)
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            if self._world == 1 and scale == 1.0 and contribute:
                return
            es = t.element_size()
            hit = self._segment_of(t)
            if hit is not None and hit[0].name != "core" and hit[1] % 16 == 0:
                seg, off = hit
                n = t.numel()
                mc = self._mc.get(seg.name)
                if (mc is not None and op == _native.OP_SUM and n * es >= self._nvls_min and self._world > 1
                        and self._force_plan is None):
                    blocks = max(8, min(self._max_blocks, (n * es) // (64 << 10)))
                    K.allreduce_nvls(self._tables[seg.name], self._status, mc[1], off, n, dt, scale, self._next_flag(),
                                     _CH_ALLREDUCE, contribute, blocks, self._threads, self._barrier_mode, sp)
                    self.launches += 1
                    return
                algo, blocks = self._plan(n * es)
                K.allreduce(self._tables[seg.name], self._status, off, 0, 0, n, dt, op, scale, self._next_flag(),
                            _CH_ALLREDUCE, contribute, algo, blocks, self._threads, self._barrier_mode, sp)
                self.launches += 1
                return
            if t.data_ptr() % 16:
                raise ValueError("allreduce_ needs a 16-byte aligned tensor")
            max_elems = self._staging_usable // es
            flat = t.view(-1)
            for lo in range(0, flat.numel(), max_elems):
                n = min(max_elems, flat.numel() - lo)
                algo, blocks = self._plan(n * es)
                ptr = flat.data_ptr() + lo * es
                K.allreduce(self._tables["core"], self._status, 0, ptr, ptr, n, dt, op, scale, self._next_flag(),
                            _CH_ALLREDUCE, contribute, algo, blocks, self._threads, self._barrier_mode, sp)
                self.launches += 1

    def q8_bytes(self, numel: int) -> int:
        return self._K.q8_buffer_bytes(numel, max(self._world, 1))

    def q8_allreduce_(self, out: torch.Tensor, a: torch.Tensor, b: Optional[torch.Tensor] = None,
                      scale: float = 1.0, contribute: bool = True,
                      stream: Optional[torch.cuda.Stream] = None) -> None:
        """out = dequant(allreduce_fp8(quant(a - b))) * scale, one launch per staging chunk.

        ``b`` (optional) fuses DiLoCo's pseudo-gradient ``original - local``
        (reference: torchft/local_sgd.py:324-337); ``out`` may alias ``a``.
        """
        K = self._K
        for x in (out, a) + ((b,) if b is not None else ()):
            if not x.is_cuda or not x.is_contiguous() or x.data_ptr() % 16:
                raise ValueError("q8_allreduce_ needs contiguous 16-byte aligned CUDA tensors")
        dt = _native.dtype_code(a)
        sp = _native.stream_ptr(stream)
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            if self._world == 1:
                # degenerate quorum: exact arithmetic, no quantisation noise
                res = a if b is None else a - b
                if not contribute:
                    out.zero_()
                elif scale != 1.0:
                    torch.mul(res, scale, out=out)
                elif out.data_ptr() != res.data_ptr():
                    out.copy_(res)
                return
            es = a.element_size()
            # a dedicated scratch segment ("<name>_q8", allocated by the caller before the first quorum) that holds the whole
            # message in wire format (+ this rank's reduced slice): three bandwidth-bound launches of any grid size
            # separated by one-CTA handshakes instead of one barrier-laden launch per 256 MB staging chunk
            n = a.numel()
            q_bytes = (self._K.q8_buffer_bytes(n, self._world) + 255) // 256 * 256
            need = q_bytes + self._K.q8_slice_buffer_bytes(n, self._world)
            for name, seg in self._segments.items():
                if name.endswith("_q8") and seg.nbytes >= need and name in self._tables:
                    table = self._tables[name]
                    ngroups = self._K.q8_ngroups(n, self._world)
                    big = max(1, min(self._K.NUM_SMS * 16, ngroups // 16 + 1))
                    if contribute:
                        K.q8_quantize_raw(a.data_ptr(), b.data_ptr() if b is not None else 0, n, ngroups, dt, seg.ptr, sp)
                    else:
                        K.memset_async(seg.ptr, 0, q_bytes, sp)  # zero scales: this replica adds nothing
                    self._handshake(2, True, _CH_Q8, sp)
                    K.q8_slice_reduce(table, self._z1_ok(2), 0, q_bytes, n, scale, max(1, min(self._K.NUM_SMS * 8, ngroups // self._world // 16 + 1)), sp)
                    self._handshake(2, True, _CH_Q8, sp)
                    K.q8_gather_dequant(table, self._z1_ok(2), q_bytes, n, dt, out.data_ptr(), big, sp)
                    self.launches += 3
                    return
            # elements per launch such that the Q8G buffer fits in staging
            per = (self._staging_usable * 512 // 516) // (512 * self._world) * (512 * self._world) - 512 * self._world
            fo, fa = out.view(-1), a.view(-1)
            fb = b.view(-1) if b is not None else None
            for lo in range(0, fa.numel(), per):
                n = min(per, fa.numel() - lo)
                blocks = max(4, min(self._q8_max_blocks, (n // 512) // 32 + 1))
                K.q8_allreduce(self._tables["core"], self._status, 0, fa.data_ptr() + lo * es,
                               (fb.data_ptr() + lo * es) if fb is not None else 0, fo.data_ptr() + lo * es, n, dt,
                               scale, self._next_flag(), _CH_Q8, contribute, blocks, self._barrier_mode, sp)
                self.launches += 1

    def q8_reduce_scatter_(self, out: torch.Tensor, inp: torch.Tensor, slice_elems: int, scale: float = 1.0,
                           contribute: bool = True, stream: Optional[torch.cuda.Stream] = None) -> None:
        """fp8 reduce-scatter in ONE launch: rank-slice s of ``inp`` is ``[s*slice_elems, (s+1)*slice_elems)``; ``out``
        (``slice_elems`` elements) receives this rank's slice, fp32-reduced over the quorum and scaled. Quantise, exchange
        and reduce happen inside the kernel (reference: collectives.py:159-294 = 2 kernels + alltoall + 2 allocations)."""
        self._check_raw(out, inp)
        dt = _native.dtype_code(inp)
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            W = self._world
            if W < 2:
                raise ValueError("q8_reduce_scatter_ needs a quorum of at least 2")
            assert inp.numel() <= W * slice_elems and out.numel() >= min(slice_elems, max(0, inp.numel() - self._rank * slice_elems))
            if self._K.q8_rs_buffer_bytes(slice_elems, W) > self._staging_usable:
                raise ValueError("q8_reduce_scatter_: message larger than the staging segment")
            groups = W * ((slice_elems + 511) // 512)
            blocks = max(4, min(self._q8_max_blocks, groups // 32 + 1))
            self._K.q8_reduce_scatter(self._tables["core"], self._status, 0, inp.data_ptr(), out.data_ptr(), inp.numel(), slice_elems,
                                      dt, scale, self._next_flag(), _CH_Q8, contribute, blocks, self._barrier_mode,
                                      _native.stream_ptr(stream))
            self.launches += 1

    # ------------------------------------------------------------------ the rest of the collective surface
    def _xblocks(self, nbytes: int) -> int:
        return max(1, min(self._max_blocks, self._K.MAX_BLOCKS, nbytes // (64 << 10)))

    def _exchange(self, inp: int, out: int, send: List[Tuple[int, int]], recv: List[Tuple[int, int]], stream: Any,
                  rounds: Optional[int] = None) -> None:
        """One push-exchange launch per staging round. ``send[p] = (offset, bytes)`` into ``inp`` owed to rank p,
        ``recv[p] = (offset, bytes)`` into ``out`` expected from rank p. Every rank must run the same number of
        rounds: either the message lengths are known quorum-wide (default: derived from them) or the caller agreed on
        ``rounds`` beforehand (:meth:`alltoallv_`)."""
        W = self._world
        stride = (self._staging_usable // W) & ~15
        longest = max([n for _, n in send] + [n for _, n in recv] + [0])
        if rounds is not None:
            longest = rounds * stride
        if longest == 0:
            return
        sp = _native.stream_ptr(stream)
        for lo in range(0, longest, stride):
            s_off = [o + min(lo, n) for o, n in send]
            s_len = [max(0, min(stride, n - lo)) for _, n in send]
            r_off = [o + min(lo, n) for o, n in recv]
            r_len = [max(0, min(stride, n - lo)) for _, n in recv]
            self._K.push_exchange(self._tables["core"], self._status, inp, out, s_off, s_len, r_len, r_off, stride,
                                  self._next_flag(), _CH_ALLREDUCE, self._xblocks(max(s_len + r_len)), self._barrier_mode, sp)
            self.launches += 1

    @staticmethod
    def _check_raw(*ts: torch.Tensor) -> None:
        for t in ts:
            if not t.is_cuda or not t.is_contiguous():
                raise ValueError("native collectives need contiguous CUDA tensors")

    def allgather_(self, out: torch.Tensor, inp: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """``out[r*n:(r+1)*n] = inp of rank r`` (any dtype; moves (W-1)*n bytes out of every rank)."""
        self._check_raw(out, inp)
        n = inp.numel() * inp.element_size()
        assert out.numel() * out.element_size() == n * max(self._world, 1)
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            if self._world == 1:
                if out.data_ptr() != inp.data_ptr():
                    out.view(-1).view(torch.uint8)[:n].copy_(inp.view(-1).view(torch.uint8))
                return
            W = self._world
            self._exchange(inp.data_ptr(), out.data_ptr(), [(0, n)] * W, [(p * n, n) for p in range(W)], stream)

    def broadcast_(self, t: torch.Tensor, root: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Root's ``t`` lands in everybody's ``t`` (root stores into the peers' staging slots; n bytes per peer link)."""
        self._check_raw(t)
        n = t.numel() * t.element_size()
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            if self._world == 1:
                return
            W, me = self._world, self._rank
            send = [(0, n if (me == root and p != me) else 0) for p in range(W)]
            recv = [(0, n if (p == root and me != root) else 0) for p in range(W)]
            self._exchange(t.data_ptr(), t.data_ptr(), send, recv, stream)

    def alltoall_(self, out: torch.Tensor, inp: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Equal-split all-to-all: chunk p of ``inp`` goes to rank p, where it becomes chunk ``rank`` of ``out``."""
        self._check_raw(out, inp)
        nb = inp.numel() * inp.element_size()
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            W = max(self._world, 1)
            if nb % W or out.numel() * out.element_size() != nb:
                raise ValueError("alltoall_: buffers must have equal size divisible by the world size")
            if W == 1:
                if out.data_ptr() != inp.data_ptr():
                    out.view(-1).view(torch.uint8).copy_(inp.view(-1).view(torch.uint8))
                return
            c = nb // W
            self._exchange(inp.data_ptr(), out.data_ptr(), [(p * c, c) for p in range(W)], [(p * c, c) for p in range(W)], stream)

    def alltoallv_(self, out: torch.Tensor, inp: torch.Tensor, out_bytes: List[int], in_bytes: List[int],
                   stream: Optional[torch.cuda.Stream] = None) -> None:
        """All-to-all with per-peer lengths: the first ``in_bytes[p]`` ... bytes of ``inp`` (consecutive chunks) go to rank
        p, which stores what it gets from rank q as its q-th consecutive chunk of ``out_bytes[q]`` bytes. A rank only
        knows its own row and column of the split matrix, so the ranks first agree on the number of staging rounds with
        one 16-byte MAX all-reduce that is read back on the host (a synchronisation: this is not a hot-path collective)."""
        self._check_raw(out, inp)
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            W = max(self._world, 1)
            if len(out_bytes) != W or len(in_bytes) != W:
                raise ValueError("alltoallv_: one length per rank")
            if sum(in_bytes) > inp.numel() * inp.element_size() or sum(out_bytes) > out.numel() * out.element_size():
                raise ValueError("alltoallv_: splits exceed the buffers")
            if W == 1:
                out.view(-1).view(torch.uint8)[: in_bytes[0]].copy_(inp.view(-1).view(torch.uint8)[: in_bytes[0]])
                return
            stride = (self._staging_usable // W) & ~15
            mine = (max(list(in_bytes) + list(out_bytes)) + stride - 1) // stride
            with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
                agree = torch.tensor([float(mine), 0.0, 0.0, 0.0], dtype=torch.float32, device=self.device)
            self.allreduce_(agree, op=_native.OP_MAX, stream=stream)
            rounds = int(agree[0].item())  # exact: a round count is far below 2^24
            send, recv, so, ro = [], [], 0, 0
            for p in range(W):
                send.append((so, int(in_bytes[p])))
                recv.append((ro, int(out_bytes[p])))
                so += int(in_bytes[p])
                ro += int(out_bytes[p])
            self._exchange(inp.data_ptr(), out.data_ptr(), send, recv, stream, rounds=rounds)

    def reduce_scatter_(self, out: torch.Tensor, inp: torch.Tensor, op: int = _native.OP_SUM, scale: float = 1.0,
                        stream: Optional[torch.cuda.Stream] = None) -> None:
        """``out = scale * reduce over ranks of inp[rank*n:(rank+1)*n]`` (fp32 accumulate, fixed rank order)."""
        self._check_raw(out, inp)
        dt = _native.dtype_code(inp)
        n, es = out.numel(), inp.element_size()
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            W = max(self._world, 1)
            assert inp.numel() == n * W and out.dtype == inp.dtype
            if W == 1:
                torch.mul(inp.view(-1), scale, out=out.view(-1)) if scale != 1.0 else out.view(-1).copy_(inp.view(-1))
                return
            sp = _native.stream_ptr(stream)
            hit = self._segment_of(inp)
            if hit is not None and hit[0].name != "core" and hit[1] % 16 == 0:
                seg, off = hit  # zero-copy: peers read the input where it lives
                self._K.reduce_scatter(self._tables[seg.name], self._status, off, 0, out.data_ptr(), n, dt, op, scale,
                                       self._next_flag(), _CH_ALLREDUCE, self._xblocks(n * es), self._barrier_mode, sp)
                self.launches += 1
                return
            per = (self._staging_usable // (W * es)) // 8 * 8  # elements of every slot per round (16 B aligned slots)
            if n <= per:
                self._K.reduce_scatter(self._tables["core"], self._status, 0, inp.data_ptr(), out.data_ptr(), n, dt, op, scale,
                                       self._next_flag(), _CH_ALLREDUCE, self._xblocks(n * es), self._barrier_mode, sp)
                self.launches += 1
                return
            rows, flat_out = inp.view(W, n), out.view(-1)
            for lo in range(0, n, per):  # larger than staging: one strided gather per round
                hi = min(n, lo + per)
                piece = rows[:, lo:hi].contiguous()
                self._K.reduce_scatter(self._tables["core"], self._status, 0, piece.data_ptr(), flat_out[lo:hi].data_ptr(), hi - lo, dt,
                                       op, scale, self._next_flag(), _CH_ALLREDUCE, self._xblocks((hi - lo) * es), self._barrier_mode, sp)
                piece.record_stream(stream if stream is not None else torch.cuda.current_stream())
                self.launches += 1

    def _p2p(self, is_send: bool, t: torch.Tensor, peer: int, stream: Optional[torch.cuda.Stream]) -> None:
        self._check_raw(t)
        nbytes = t.numel() * t.element_size()
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            if nbytes == 0:
                return
            book = self._send_seq if is_send else self._recv_seq
            seq = book.get(peer, 0) + 1
            pieces = (nbytes + self._mailbox_bytes - 1) // self._mailbox_bytes
            book[peer] = seq + pieces - 1
            self._K.p2p(self._tables["core"], self._status, is_send, t.data_ptr(), nbytes, peer, self._mailbox_off,
                        self._mailbox_bytes, (self._epoch << 32) + seq, _CH_USER, _native.stream_ptr(stream))
            self.launches += 1

    def send_(self, t: torch.Tensor, dst: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Stream ``t`` into rank ``dst``'s mailbox (pieces of <= 4 MiB, flow-controlled by its acks)."""
        self._p2p(True, t, dst, stream)

    def recv_(self, t: torch.Tensor, src: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Receive the next message of rank ``src`` (FIFO per ordered pair; tags are not matched) into ``t``."""
        self._p2p(False, t, src, stream)

    # ------------------------------------------------------------------ FT-ZeRO-1 (csrc/kernels/zero1.cu)
    def peer_pointers(self, name: str) -> List[int]:
        """Mapped base address of segment ``name`` on every quorum rank (index = rank)."""
        return list(self._ptrs[name])

    def _mc_base(self, name: str, nbytes: int) -> int:
        mc = self._mc.get(name)
        return mc[1] if (mc is not None and self._world > 1 and nbytes >= self._nvls_min) else 0

    def _z1_ok(self, slot: int) -> int:
        """Device word the handshake kernels write their outcome to (slot 0: comm stream, slot 1: optimizer stream)."""
        if self._z1_ok_buf is None:
            self._z1_ok_buf = torch.ones(4, dtype=torch.int32, device=self.device)
        return self._z1_ok_buf.data_ptr() + 4 * slot

    def _handshake(self, slot: int, release: bool, channel: int, sp: int) -> None:
        self._K.zero1_handshake(self._tables["core"], self._status, self._z1_ok(slot), self._next_flag(), channel, release,
                                self._barrier_mode, sp)
        self.launches += 1

    def zero1_reduce_scatter_(self, segment: str, off: int, nelem: int, scale: float, contribute: bool,
                              replication: int, blocks: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Reduce-scatter ``nelem`` bf16 elements at byte offset ``off`` of ``segment`` in place: afterwards rank r
        (and its ``replication - 1`` successors) hold the scaled sum of slice r. Three launches on ``stream``:
        handshake ("my unit is ready") -> sync-free reduce kernel (any grid) -> handshake ("my pushes landed")."""
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            sp = _native.stream_ptr(stream)
            if not contribute:
                # healing / spare replica: its gradients count as zeros (reference manager.py:441-442)
                self._K.memset_async(self._segments[segment].ptr + off, 0, nelem * 2, sp)
            self._handshake(0, not contribute, _CH_ALLREDUCE, sp)
            blocks = max(1, min(blocks, self._K.NUM_SMS * 32, (nelem // 8 + 511) // 512))
            self._K.zero1_reduce(self._tables[segment], self._z1_ok(0), self._mc_base(segment, nelem * 2), off, nelem, scale,
                                 replication, blocks, self._threads, sp)
            self.launches += 1
            self._handshake(0, True, _CH_ALLREDUCE, sp)

    def zero1_commit_(self, gate: torch.Tensor, host_ok: bool, exchange: bool,
                      stream: Optional[torch.cuda.Stream] = None) -> int:
        """Device-side commit verdict (AND over the quorum when ``exchange``): writes ``gate[0]`` (verdict),
        increments ``gate[1]`` on success and posts the verdict to the host-mapped ring. Returns the sequence
        number to pass to :meth:`verdict`."""
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            self._commit_seq = (self._commit_seq + 1) & 0x3fffffff
            seq = self._commit_seq
            self._K.zero1_commit(self._tables["core"], self._status, gate.data_ptr(), self._next_flag(), seq, _CH_USER,
                                 bool(host_ok), bool(exchange), _native.stream_ptr(stream))
            self.launches += 1
            return seq

    def verdict(self, seq: int) -> Optional[bool]:
        """Verdict of commit ``seq`` if the kernel has run, else ``None`` (never blocks)."""
        v = self._status.verdict(seq)
        return None if v < 0 else bool(v)

    def zero1_update_(self, segment: str, poff: int, grad: int, master: int, m: int, v: int, nelem: int,
                      hyper: Tuple[float, float, float, float, float], gate: torch.Tensor, replication: int, mode: int,
                      blocks: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Gated AdamW on the held slices of one unit + all-gather of the primary slice's new bf16 weights into
        ``segment`` on the ranks that do not hold it (``mode`` 1: ungated re-broadcast of bf16(master) to everybody, no
        state change). A sync-free kernel (any grid) followed by one handshake when anything was pushed."""
        with self._lock:
            if not self._configured:
                raise RuntimeError("SymmetricComm is not configured")
            lr, b1, b2, eps, wd = hyper
            sp = _native.stream_ptr(stream)
            blocks = max(1, min(blocks, self._K.NUM_SMS * 32, (nelem // 8 + 511) // 512))
            self._K.zero1_update(self._tables[segment], self._mc_base(segment, nelem * 2), gate.data_ptr(), poff, grad, master,
                                 m, v, nelem, lr, b1, b2, eps, wd, replication, mode, blocks, self._threads, sp)
            self.launches += 1
            pushes = self._world > 1 and (mode == 1 or self._world > replication)
            if pushes:
                self._handshake(1, True, _CH_HEAL, sp)

    # ------------------------------------------------------------------ status
    def abort(self) -> None:
        """Make every in-flight / future kernel wait bail out immediately."""
        if self._status is not None:
            self._status.set_abort(True)

    def errored(self) -> Optional[Exception]:
        if self._status is None:
            return None
        code, peer, seq = self._status.error()
        if code == 0:
            return None
        what = {1: "timeout", 2: "aborted"}.get(code, f"error {code}")
        return RuntimeError(f"peer-memory collective {what} waiting for replica rank {peer} (seq {seq})")

    @property
    def rank(self) -> int:
        return self._rank

    @property
    def world(self) -> int:
        return self._world

    @property
    def configured(self) -> bool:
        return self._configured

    def shutdown(self) -> None:
        K = self._K
        with self._lock:
            if self._status is not None:
                self._status.set_abort(True)
            try:
                torch.cuda.synchronize(self.device)
            except RuntimeError:
                pass
            self._release_multicast()
            for p in self._peer_ptrs.values():
                try:
                    K.ipc_close_handle(p)
                except RuntimeError:
                    pass
            self._peer_ptrs = {}
            for va, h, size in self._peer_vmm.values():
                try:
                    K.vmm_unmap(va, size, h)
                except Exception:  # noqa: BLE001
                    pass
            self._peer_vmm = {}
            self._tables = {}
            self._configured = False
            # local segments are intentionally leaked until process exit if a
            # peer may still have them mapped; free only the python views

    def free_segments(self) -> None:
        """Return this rank's segments to the driver. Only after :meth:`shutdown` AND once every peer has shut down
        too (they unmap on shutdown): a benchmark that builds a second trainer in the same process needs the memory."""
        with self._lock:
            assert not self._configured, "shutdown() first"
            torch.cuda.synchronize(self.device)
            for seg in self._segments.values():
                seg.tensor = torch.empty(0, dtype=torch.uint8)
                try:
                    if self._mode == "vmm":
                        self._K.vmm_unmap(seg.ptr, seg.nbytes, seg.mem_handle)
                    else:
                        self._K.symm_free(seg.ptr)
                except Exception:  # noqa: BLE001
                    logger.warning("could not free symmetric segment %s", seg.name)
            self._segments = {}
            self._status = None
