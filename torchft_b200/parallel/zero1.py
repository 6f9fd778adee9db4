"""FT-ZeRO-1: optimizer state partitioned across REPLICA GROUPS, without giving up fault tolerance.

The reference keeps the full optimizer on every replica and all-reduces every gradient
(upstream torchft/manager.py:466-478, upstream torchft/optim.py:52-55). Here the
cross-replica collective and the optimizer are one pipeline of three hand-written sm_90a kernels
(``csrc/kernels/zero1.cu``):

* backward:  ``reduce_scatter`` per unit (one transformer block = one unit), overlapped with backward;
  rank ``r`` reduces slice ``r`` of the unit out of every peer's HBM and also pushes the result to its
  ``k-1`` buddies (ranks ``r+1 .. r+k-1``) -- every slice of optimizer state lives on ``k`` replicas;
* commit:    ONE kernel ANDs "my step was clean" over the quorum through the signal pads and writes a
  device gate word -- no host synchronisation, no RPC; the Manager reads the verdict lazily;
* update:    gated AdamW on the held slices; the primary holder stores the new bf16 weights straight
  into every replica's parameter buffer (the all-gather is the update's epilogue) while the next
  forward already runs, unit by unit.

Fault tolerance. Ownership is a pure function of (unit, quorum rank, world, k) -- see
:class:`ShardLayout` -- so every replica derives it from the quorum alone. On every quorum change
each rank publishes which element ranges of (master, m, v) it holds and at which update count; a
rank whose new slices it does not hold yet pulls them over NVLink (``heal_copy`` kernel, peer
memory) from any replica that does. A slice is lost only if all ``k`` holders disappear within one
quorum transition; it is then re-seeded from the (fully replicated) bf16 weights with zero moments
and reported. The first commit phase after a quorum change re-broadcasts the weights from the
master copies, so a failure in the middle of an all-gather can never leave replicas with
different weights for more than one (discarded or slightly stale) step.
"""

from __future__ import annotations

import json
import logging
import os
import threading
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

logger = logging.getLogger(__name__)

Range = Tuple[int, int]

__all__ = ["ShardLayout", "Zero1Optimizer", "merge_ranges", "subtract_ranges", "intersect_ranges", "plan_pulls"]


# --------------------------------------------------------------------------- interval arithmetic
def merge_ranges(rs: Sequence[Range]) -> List[Range]:
    """Sorted, coalesced, non-empty half-open ranges."""
    out: List[Range] = []
    for lo, hi in sorted((int(a), int(b)) for a, b in rs if b > a):
        if out and lo <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], hi))
        else:
            out.append((lo, hi))
    return out


def intersect_ranges(a: Sequence[Range], b: Sequence[Range]) -> List[Range]:
    a, b = merge_ranges(a), merge_ranges(b)
    out: List[Range] = []
    i = j = 0
    while i < len(a) and j < len(b):
        lo, hi = max(a[i][0], b[j][0]), min(a[i][1], b[j][1])
        if lo < hi:
            out.append((lo, hi))
        if a[i][1] < b[j][1]:
            i += 1
        else:
            j += 1
    return out


def subtract_ranges(a: Sequence[Range], b: Sequence[Range]) -> List[Range]:
    """``a`` minus ``b``."""
    out: List[Range] = []
    b = merge_ranges(b)
    for lo, hi in merge_ranges(a):
        cur = lo
        for blo, bhi in b:
            if bhi <= cur or blo >= hi:
                continue
            if blo > cur:
                out.append((cur, blo))
            cur = max(cur, bhi)
            if cur >= hi:
                break
        if cur < hi:
            out.append((cur, hi))
    return out


def total(rs: Sequence[Range]) -> int:
    return sum(hi - lo for lo, hi in rs)


# --------------------------------------------------------------------------- ownership
@dataclass(frozen=True)
class ShardLayout:
    """Which element ranges of the flat parameter vector a quorum rank holds optimizer state for.

    ``units`` are contiguous element ranges (multiples of 8 elements) tiling the flat buffer. Unit
    ``u`` is cut into ``world`` slices of ``ceil(nvec / world)`` 16-byte vectors (the arithmetic of
    ``Geo`` in ``zero1.cu``); slice ``s`` has primary holder ``s`` and buddies ``s+1 .. s+k-1``.
    """

    units: Tuple[Range, ...]
    replication: int = 2

    def slice_bounds(self, unit: int, world: int, s: int) -> Range:
        lo, hi = self.units[unit]
        nvec = (hi - lo) // 8
        per = (nvec + world - 1) // world
        a, b = min(s * per, nvec), min((s + 1) * per, nvec)
        return lo + a * 8, lo + b * 8

    def k(self, world: int) -> int:
        return max(1, min(self.replication, world))

    def primary(self, rank: int, world: int) -> List[Range]:
        return merge_ranges([self.slice_bounds(u, world, rank) for u in range(len(self.units))])

    def held(self, rank: int, world: int) -> List[Range]:
        """Ranges whose (master, m, v) this rank keeps up to date: its primary slices and the slices it backs up."""
        out: List[Range] = []
        for u in range(len(self.units)):
            for j in range(self.k(world)):
                out.append(self.slice_bounds(u, world, (rank - j) % world))
        return merge_ranges(out)

    def holders(self, unit: int, world: int, s: int) -> List[int]:
        return [(s + j) % world for j in range(self.k(world))]


def plan_pulls(need: Sequence[Range], holdings: Dict[int, Sequence[Range]], me: int) -> Tuple[List[Tuple[int, int, int]], List[Range]]:
    """Cover ``need`` from peers' ``holdings``: ``[(src_rank, lo, hi), ...]`` plus the ranges nobody holds.

    Sources are tried in the order ``me+1, me+2, ...`` so concurrent pullers spread over different peers.
    """
    pulls: List[Tuple[int, int, int]] = []
    left = merge_ranges(need)
    ranks = sorted(r for r in holdings if r != me)
    if ranks:
        start = next((i for i, r in enumerate(ranks) if r > me), 0)
        ranks = ranks[start:] + ranks[:start]
    for r in ranks:
        if not left:
            break
        got = intersect_ranges(left, holdings[r])
        for lo, hi in got:
            pulls.append((r, lo, hi))
        left = subtract_ranges(left, got)
    return pulls, left


# --------------------------------------------------------------------------- the optimizer
class Zero1Optimizer:
    """AdamW with fp32 master/m/v partitioned over the replicas of the current quorum (see module doc).

    All five flat buffers live in NVLink-symmetric segments of the process group: ``param`` and ``grad``
    (bf16; written/read by peers every step) and ``master``/``m``/``v`` (fp32; read by peers only when
    ownership moves). The state arrays are full-size and addressed by GLOBAL element index -- only the
    held ranges are kept up to date -- which makes re-sharding a plain ranged copy.

    Args:
        pg: a ``ProcessGroupB200`` (symmetric segments must be allocated before its first ``configure``)
        numel: elements of the flat parameter vector (multiple of 8)
        units: element ranges in FORWARD order that tile ``[0, numel)`` (one per transformer block)
        replication: holders per slice (``k``); ``min(k, world)`` is used
    """

    def __init__(self, pg: Any, numel: int, units: Optional[Sequence[Range]] = None, lr: float = 3e-4,
                 betas: Tuple[float, float] = (0.9, 0.95), eps: float = 1e-8, weight_decay: float = 0.1,
                 replication: int = 2, blocks: Optional[int] = None) -> None:
        from torchft_b200.ops import _native

        assert numel % 8 == 0
        self._K = _native.load()
        self.pg = pg
        self.comm = pg.comm
        self.device = pg.comm.device
        self.numel = numel
        self._replication = int(os.environ.get("TORCHFT_B200_Z1_REPLICATION", replication))
        self.layout: ShardLayout = ShardLayout(((0, numel),), self._replication)
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]
        # the big kernels are sync-free, so their grids are free parameters: the reduce-scatter is NVLink-latency bound
        # and shares the SMs with backward; the update is HBM-bound and likes many short CTAs (cf. the AdamW cap sweep)
        self._rs_blocks = int(os.environ.get("TORCHFT_B200_Z1_RS_BLOCKS", 128))
        self._upd_blocks = int(os.environ.get("TORCHFT_B200_Z1_UPD_BLOCKS", blocks or self._K.NUM_SMS * 16))
        self.param = pg.alloc_symmetric("z1_param", numel * 2).view(torch.bfloat16)
        self.grad = pg.alloc_symmetric("z1_grad", numel * 2).view(torch.bfloat16)
        self.master = pg.alloc_symmetric("z1_master", numel * 4).view(torch.float32)
        self.m = pg.alloc_symmetric("z1_m", numel * 4).view(torch.float32)
        self.v = pg.alloc_symmetric("z1_v", numel * 4).view(torch.float32)
        # gate[0]: verdict of the last commit, gate[1]: applied updates (AdamW's t), both written on the device
        self.gate = torch.zeros(2, dtype=torch.int32, device=self.device)
        self.t = 0                       # host mirror of gate[1] (advanced when a verdict is resolved)
        self._holdings: List[Range] = [(0, numel)]  # identical seed on every replica => everything valid at t = 0
        self._lock = threading.Lock()
        self._reshard_stream = torch.cuda.Stream(device=self.device)
        self._reshard_event: Optional[torch.cuda.Event] = None
        self._refresh_pending = False
        self._commit_layout: Optional[Tuple[int, int]] = None
        self._commit_stream: torch.cuda.Stream = torch.cuda.current_stream(self.device)
        self._commit_event: Optional[torch.cuda.Event] = None
        self.lost_elements = 0           # state elements that had to be re-seeded because no holder survived
        self.pulled_bytes = 0
        if units is not None:
            self.set_units(units)
        pg.add_configure_hook(self._on_configured)

    def set_units(self, units: Sequence[Range]) -> None:
        """Fix the unit ranges (forward order, tiling ``[0, numel)``); call before the first quorum."""
        assert all(lo % 8 == 0 and hi % 8 == 0 for lo, hi in units)
        assert merge_ranges(units) == [(0, self.numel)] and total(units) == self.numel, "units must tile the flat buffer exactly"
        self.layout = ShardLayout(tuple((int(a), int(b)) for a, b in units), self._replication)

    # ------------------------------------------------------------------ init / heal
    @torch.no_grad()
    def seed_master(self) -> None:
        """Call once after the bf16 weights were initialised (same seed on every replica)."""
        self.master.copy_(self.param)
        self.m.zero_()
        self.v.zero_()

    def state_dict(self) -> Dict[str, Any]:
        """What a healing replica needs from ANY peer: the replicated bf16 weights and the update count.
        Its slices of (master, m, v) arrive through the re-shard pull from their holders."""
        return {"param": self.param, "t": self.t}

    def load_state_dict(self, sd: Dict[str, Any]) -> None:
        with torch.no_grad():
            if sd["param"].data_ptr() != self.param.data_ptr():
                self.param.copy_(sd["param"])
        self._set_t(int(sd["t"]))

    def _set_t(self, t: int) -> None:
        self.t = t
        with torch.cuda.stream(self._reshard_stream):
            self.gate[1:2].fill_(t)

    # ------------------------------------------------------------------ re-shard on quorum change
    def _on_configured(self, store: Any, rank: int, world: int, epoch: int) -> None:
        """Runs inside ``ProcessGroupB200.configure`` (quorum thread) with the quorum-scoped store."""
        with self._lock:
            missing = [n for n in ("z1_param", "z1_grad", "z1_master", "z1_m", "z1_v") if not self.comm.is_symmetric(n)]
            if missing:
                # the kernels dereference peer pointers: every replica must construct its Zero1Optimizer before its first
                # quorum (segments allocated later only become symmetric at the NEXT quorum change)
                raise RuntimeError(f"FT-ZeRO-1 segments {missing} are not mapped on every replica of this quorum")
            me = {"t": self.t, "hold": self._holdings}
            store.set(f"z1/{rank}", json.dumps(me))
            peers: Dict[int, Dict[str, Any]] = {rank: me}
            for r in range(world):
                if r != rank:
                    peers[r] = json.loads(bytes(store.get(f"z1/{r}")).decode())
            tmax = max(int(p["t"]) for p in peers.values())
            if self.t < tmax:
                self._holdings = []  # we missed an update: nothing we hold is current
            valid = {r: [tuple(x) for x in p["hold"]] for r, p in peers.items() if int(p["t"]) == tmax and r != rank}
            need = subtract_ranges(self.layout.held(rank, world), self._holdings)
            pulls, lost = plan_pulls(need, valid, rank)
            with torch.cuda.stream(self._reshard_stream):
                if pulls:
                    self._pull(pulls)
                for lo, hi in lost:
                    # every holder vanished in one transition: re-seed from the replicated bf16 weights
                    self.master[lo:hi].copy_(self.param[lo:hi])
                    self.m[lo:hi].zero_()
                    self.v[lo:hi].zero_()
                if self.t != tmax:
                    self.gate[1:2].fill_(tmax)
                self._reshard_event = self._reshard_stream.record_event()
            if lost:
                self.lost_elements += total(lost)
                logger.warning("zero1: %d state elements had no surviving holder and were re-seeded from the weights "
                               "(moments reset)", total(lost))
            self.pulled_bytes += 12 * total([(lo, hi) for _, lo, hi in pulls])
            self.t = tmax
            self._holdings = merge_ranges(list(self._holdings) + list(need))
            self._refresh_pending = world > 1

    def _pull(self, pulls: List[Tuple[int, int, int]]) -> None:
        """One heal_copy launch that gathers (master, m, v)[lo:hi] from the source ranks' segments."""
        from torchft_b200.checkpointing.p2p_transport import device_copy

        entries: List[Tuple[int, int, int]] = []
        for name, local in (("z1_master", self.master), ("z1_m", self.m), ("z1_v", self.v)):
            ptrs = self.comm.peer_pointers(name)
            for src, lo, hi in pulls:
                entries.append((ptrs[src] + lo * 4, local.data_ptr() + lo * 4, (hi - lo) * 4))
        device_copy(entries, torch.cuda.current_stream(), chunk_bytes=1 << 20)

    # ------------------------------------------------------------------ per-step pipeline
    def unit_of(self, lo: int, hi: int) -> int:
        return self.layout.units.index((lo, hi))

    def reduce_scatter(self, unit: int, scale: float, contribute: bool) -> Any:
        """Reduce unit ``unit`` of the gradient buffer across the quorum (comm stream, overlaps backward)."""
        lo, hi = self.layout.units[unit]
        if self.comm.world == 1:
            if scale != 1.0 or not contribute:
                self.grad[lo:hi].mul_(scale if contribute else 0.0)
            return None
        k = self.layout.replication
        return self.pg._launch(
            lambda s: self.comm.zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, scale, contribute, k, self._rs_blocks, s),
            None)

    # -- committer protocol of Manager.commit_on_device ---------------------------------------------------------
    def bind_stream(self, stream: torch.cuda.Stream) -> None:
        """The stream the verdict and update kernels run on (the trainer's optimizer stream)."""
        self._commit_stream = stream

    def enqueue(self, host_ok: bool) -> int:
        """Enqueue the verdict kernel behind this step's reduce-scatters (comm stream) and backward (current stream)."""
        stream = self._commit_stream
        stream.wait_stream(self.pg.comm_stream)
        stream.wait_stream(torch.cuda.current_stream(self.device))
        if self._reshard_event is not None:
            stream.wait_event(self._reshard_event)  # a verdict also tells peers "my pulls are done"
            self._reshard_event = None
        self._commit_layout = (self.comm.rank, self.comm.world)
        seq = self.comm.zero1_commit_(self.gate, host_ok, True, stream)
        self._commit_event = stream.record_event()
        return seq

    def wait(self, seq: int, timeout: Any = None) -> bool:
        """Block the calling thread until the verdict of ``seq`` is on the host."""
        self._commit_event.synchronize()
        v = self.comm.verdict(seq)
        if v is None:
            raise RuntimeError(f"commit {seq}: the verdict kernel finished without posting a verdict")
        return v

    def update(self, events: Optional[Sequence[torch.cuda.Event]] = None) -> None:
        """Gated AdamW + weight all-gather for every unit, in forward order, on the commit stream; ``events[i]``
        fires when unit ``i``'s weights are current on THIS replica (all peers' pushes have landed)."""
        stream = self._commit_stream
        k = self.layout.replication
        lr = self.param_groups[0]["lr"]
        hp = (lr, self.betas[0], self.betas[1], self.eps, self.weight_decay)
        modes = (1, 0) if self._refresh_pending else (0,)
        self._refresh_pending = False
        for i, (lo, hi) in enumerate(self.layout.units):
            for mode in modes:
                self.comm.zero1_update_("z1_param", lo * 2, self.grad.data_ptr() + lo * 2, self.master.data_ptr() + lo * 4,
                                        self.m.data_ptr() + lo * 4, self.v.data_ptr() + lo * 4, hi - lo, hp,
                                        self.gate, k, mode, self._upd_blocks, stream)
            if events is not None:
                events[i].record(stream)

    def resolved(self, verdict: bool) -> None:
        """The Manager learned the verdict of the last :meth:`commit` (lazily, on the quorum thread)."""
        with self._lock:
            if verdict and self._commit_layout is not None:
                rank, world = self._commit_layout
                self.t += 1
                self._holdings = self.layout.held(rank, world)
            self._commit_layout = None

    # ------------------------------------------------------------------ introspection
    def state_bytes_held(self) -> int:
        return 12 * total(self.layout.held(self.comm.rank, max(self.comm.world, 1)))

    def zero_grad(self, set_to_none: bool = False) -> None:  # gradients are overwritten by the wgrad GEMMs
        pass
