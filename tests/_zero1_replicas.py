"""What the FT-ZeRO-1 GPU tests share: the three-unit geometry and its data, the fp32 AdamW reference, virtual worlds
for direct kernel launches, FT-ZeRO-1 replicas in one process on one GPU, and a trainer on a local lighthouse.

Replicas are ranks of ``SymmetricComm.virtual_world`` (pre-signalled), each with a ``Zero1Optimizer`` over the slice of
``ProcessGroupB200`` it uses, configured on one thread per rank and stepped in the Manager's order (enqueue / update /
wait / resolved)."""

from __future__ import annotations

import contextlib
import math
import threading
from datetime import timedelta

import numpy as np
import torch

HP = (1e-2, 0.9, 0.95, 1e-8, 0.1)  # lr, b1, b2, eps, wd
SHIFT = 8  # paged state: 256-element pages, so unit and slice bounds fall inside pages
UNITS = [(0, 8 * 4096), (8 * 4096, 8 * 4096 + 8 * 1001), (8 * 4096 + 8 * 1001, 8 * 4096 + 8 * 1001 + 8 * 7)]
NUMEL = UNITS[-1][1]
STEPS = 4  # entries of the warmup_cosine schedule


def warmup_cosine(i):
    """Two warmup steps, then a cosine to 0.1 over the rest of the table."""
    if i < 2:
        return (i + 1) / 2
    return 0.1 + 0.9 * 0.5 * (1 + math.cos(math.pi * (i - 2) / (STEPS - 2)))


def raws(world, seed, scales=(1.0,), numel=NUMEL):
    """``raws[i][r]``: rank r's bf16 gradient ``randn * (r + 1) * scales[i]``, from one generator seeded with ``seed``.
    One entry per micro-batch of a step, or per step."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [[(torch.randn(numel, device="cuda", generator=g) * (r + 1) * s).bfloat16() for r in range(world)]
            for s in scales]


def reduced(micro, quiet=None):
    """The reduced gradient of one step of micro-batches ``micro[m][r]``: per micro-batch the fp32 sum of the ranks' bf16
    gradients in rank order, the micro-batches summed in order, scaled by ``1 / (contributors * M)`` in fp32 and rounded
    once to bf16. A quiet (healing or spare) rank contributes nothing and is not counted."""
    world, M = len(micro[0]), len(micro)
    total = None
    for raw in micro:
        s = None
        for r in range(world):
            if r != quiet:
                s = raw[r].float() if s is None else s + raw[r].float()
        total = s if total is None else total + s
    contributors = world - (1 if quiet is not None else 0)
    return (total * (1.0 / (contributors * M))).bfloat16()


def ref_adamw(master, m, v, g, t):
    """Step ``t`` of fp32 AdamW with ``HP`` on gradient ``g``, in place: the reference of the update kernel."""
    lr, b1, b2, eps, wd = HP
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    denom = v.sqrt() / (bc2 ** 0.5) + eps
    master.mul_(1 - lr * wd).addcdiv_(m, denom, value=-lr / bc1)


def bits(x):
    """bf16 tensor -> numpy uint16 bit patterns."""
    assert x.dtype == torch.bfloat16
    return x.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def widen(b):
    """bf16 bit patterns -> the fp32 values they stand for."""
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)


def seeded_weights(numel, seed=2):
    dev = torch.device("cuda", 0)
    return (torch.randn(numel, device=dev, generator=torch.Generator(device=dev).manual_seed(seed)) * 0.05).bfloat16()


def kernel_world(n, presignal=True):
    """``n`` virtual ranks with the gradient, weight and norm segments of ``UNITS``, for direct kernel launches."""
    from torchft_b200.parallel.symm_mem import SymmetricComm

    seg = {"z1_grad": NUMEL * 2, "z1_param": NUMEL * 2, "z1_gnorm": 8 * len(UNITS)}
    return SymmetricComm.virtual_world(n, seg, presignal=presignal, timeout=timedelta(seconds=20))


@contextlib.contextmanager
def trainer(model, tag, **kw):
    """A ``FaultTolerantTrainer`` of ``model``, replica ``{tag}_0`` alone on a local lighthouse; both shut down on exit."""
    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    lh = local_lighthouse()
    try:
        tr = FaultTolerantTrainer(model, loopback(lh.address()), replica_id=f"{tag}_0", timeout=timedelta(seconds=30),
                                  **kw)
        try:
            yield tr
        finally:
            tr.shutdown()
    finally:
        lh.shutdown()


class PG:
    """The slice of ``ProcessGroupB200`` that ``Zero1Optimizer`` uses, over one virtual-world rank whose segments exist;
    collectives run on the current stream."""

    def __init__(self, comm):
        self.comm = comm
        self.comm_stream = torch.cuda.current_stream()

    def alloc_symmetric(self, name, nbytes):
        seg = self.comm.segment(name)
        assert seg.numel() >= nbytes
        return seg[:nbytes]

    def add_configure_hook(self, fn):
        pass

    def _launch(self, fn, result):
        fn(self.comm_stream)
        return None


class Replicas:
    """``n`` virtual ranks, each with a ``Zero1Optimizer`` over ``units`` (``k`` holders per slice, updates of at most
    ``blocks`` CTAs), seeded from the same weights (``init``, default :func:`seeded_weights`).

    ``options`` go to ``Zero1Optimizer`` under its own names (``compact``, ``min_world``, ``max_grad_norm``,
    ``grad_accum_steps``, ``lr_lambda``, ``lr_steps``, ``no_decay``, ``moment_dtype``, ``ema_decay``, ...); the
    hyper-parameters default to ``HP``, the page shift to ``SHIFT`` and ``compact`` to False. A list gives one value per
    member, to build replicas that disagree; ``no_decay`` ranges are therefore given as a tuple."""

    def __init__(self, n, units=UNITS, k=2, blocks=4, init=None, **options):
        from torch.distributed import HashStore

        from torchft_b200.parallel.symm_mem import SymmetricComm
        from torchft_b200.parallel.zero1 import GNORM_UNITS, ShardLayout, pool_pages

        self.units, self.numel, self.k, self.blocks = list(units), units[-1][1], k, blocks
        self.options = {"lr": HP[0], "betas": HP[1:3], "eps": HP[3], "weight_decay": HP[4], "page_shift": SHIFT,
                        "compact": False, **options}
        per = [self.options_of(i) for i in range(n)]
        n_state = max((pool_pages(ShardLayout(tuple(units), k), o.get("min_world", 1), 1 << o["page_shift"])
                       << o["page_shift"]) if o["compact"] else self.numel for o in per)
        state = ("z1_master", "z1_m", "z1_v") + (("z1_ema",) if any(o.get("ema_decay") for o in per) else ())
        seg = {"z1_grad": self.numel * 2, "z1_param": self.numel * 2, "z1_gnorm": GNORM_UNITS * 8,
               **{x: n_state * 4 for x in state}}
        self.comms = SymmetricComm.virtual_world(n, seg, presignal=True, timeout=timedelta(seconds=20))
        self.init = seeded_weights(self.numel) if init is None else init
        self.opts = [self.make(c) for c in self.comms]
        for o in self.opts:
            o.param.copy_(self.init)
            o.seed_master()
        self.store = HashStore()
        self.members = list(range(n))
        self.pending = None

    def options_of(self, i):
        return {name: x[i] if isinstance(x, list) else x for name, x in self.options.items()}

    def make(self, comm):
        """A fresh optimizer on rank ``comm`` (a restarted process), configured like the others."""
        from torchft_b200.parallel.zero1 import Zero1Optimizer

        return Zero1Optimizer(PG(comm), self.numel, units=self.units, replication=self.k, blocks=self.blocks,
                              **self.options_of(self.comms.index(comm)))

    def layout(self):
        from torchft_b200.parallel.zero1 import ShardLayout

        return ShardLayout(tuple(self.units), self.k)

    def configure_errors(self, members, epoch):
        """The re-shard of every member for quorum ``members`` (quorum rank = position), one thread per member; returns
        the exception each member raised."""
        from torch.distributed import PrefixStore

        from torchft_b200.parallel.symm_mem import SymmetricComm

        SymmetricComm.virtual_quorum(self.comms, members, epoch)
        errs = {}

        def run(rank, m):
            try:
                self.opts[m]._on_configured(PrefixStore(f"q/{epoch}", self.store), rank, len(members), epoch)
            except Exception as e:  # noqa: BLE001
                errs[m] = e

        ts = [threading.Thread(target=run, args=(rank, m)) for rank, m in enumerate(members)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        torch.cuda.synchronize()
        return errs

    def configure(self, members, epoch):
        """The re-shard of every member for quorum ``members``, after the verdicts of the last step are settled."""
        self.settle()
        errs = self.configure_errors(members, epoch)
        assert not errs, errs
        self.members = list(members)

    def settle(self):
        """Resolve the verdicts of the last step, as the Manager does when the next one starts."""
        if self.pending is not None:
            for m, s in self.pending.items():
                self.opts[m].resolved(self.opts[m].wait(s))
            self.pending = None

    def step(self, raws, skip=None, veto=(), reduce=True, sync=True):
        """One step: micro-batch ``m`` writes ``raws[m][rank]`` into quorum rank ``rank``'s gradient and (``reduce``)
        every member reduces every unit, except ``skip = (unit, micro)`` on every member. Then every member enqueues
        its verdict (the members in ``veto`` vote no) and its update; ``sync`` waits for the device at the end."""
        self.settle()
        scale = 1.0 / (len(self.members) * self.opts[self.members[0]].grad_accum_steps)
        for micro, raw in enumerate(raws):
            for rank, i in enumerate(self.members):
                self.opts[i].grad.copy_(raw[rank])
            if reduce:
                for i in self.members:
                    for u in range(len(self.units)):
                        if skip != (u, micro):
                            self.opts[i].reduce_scatter(u, scale, True, micro)
        self.pending = {i: self.opts[i].enqueue(i not in veto) for i in self.members}
        for i in self.members:
            self.opts[i].update()
        if sync:
            torch.cuda.synchronize()

    def step_vetoed_by_all(self, raws):
        """:meth:`step` in which every member votes no: the verdict one rank's veto gives every rank once the commit
        kernel has exchanged it (the pre-signalled virtual world does not exchange verdicts)."""
        self.step(raws, veto=self.members)

    def verdicts(self):
        return {i: self.opts[i].comm.verdict(s) for i, s in self.pending.items()}

    def save(self, directory, keep=2):
        """Every member saves a checkpoint; returns the step they saved."""
        self.settle()
        t = {self.opts[i].save(directory, {"step": self.opts[i].t, "batches_committed": 0}, keep=keep) for i in self.members}
        assert len(t) == 1
        return t.pop()

    def held(self):
        """``(member, lo, hi)`` over every range a member of the current quorum holds."""
        L, world = self.layout(), len(self.members)
        return [(i, lo, hi) for rank, i in enumerate(self.members) for lo, hi in L.held(rank, world)]

    def _at(self, i, x, lo, hi):
        o = self.opts[i]
        return [(x[at:at + b - a], a, b) for a, b, at in o._pieces(o._table_host, lo, hi)]

    def get(self, i, lo, hi):
        """(master, m, v) of member ``i`` over ``[lo, hi)``, through its page table."""
        torch.cuda.synchronize()
        o = self.opts[i]
        return tuple(torch.cat([p for p, _, _ in self._at(i, x, lo, hi)]) for x in (o.master, o.m, o.v))

    def get_ema(self, i, lo, hi):
        """The EMA of member ``i`` over ``[lo, hi)``, through its page table."""
        torch.cuda.synchronize()
        return torch.cat([p for p, _, _ in self._at(i, self.opts[i].ema, lo, hi)])

    def put(self, m, v):
        """Write the flat vectors ``m`` and ``v`` into every holder's moments."""
        for i, lo, hi in self.held():
            o = self.opts[i]
            for x, y in ((o.m, m), (o.v, v)):
                for p, a, b in self._at(i, x, lo, hi):
                    p.copy_(y[a:b])
        torch.cuda.synchronize()

    def _assemble(self, get, names, dtypes):
        """Whole-vector tensors from ``get(member, lo, hi)`` over every held range; the holders must agree bit for bit."""
        self.settle()
        out = [torch.zeros(self.numel, dtype=d, device="cuda") for d in dtypes]
        seen = torch.zeros(self.numel, dtype=torch.bool, device="cuda")
        for i, lo, hi in self.held():
            for name, x, y in zip(names, out, get(i, lo, hi)):
                had = seen[lo:hi]
                assert torch.equal(x[lo:hi][had].view(torch.uint8), y[had].view(torch.uint8)), \
                    f"holders disagree on {name} over {(lo, hi)} (member {i})"
                x[lo:hi] = y
            seen[lo:hi] = True
        assert bool(seen.all())
        return out

    def full_state(self):
        """(master, m, v) over the whole vector assembled from the holders, which must agree bit for bit."""
        o = self.opts[self.members[0]]
        return self._assemble(self.get, ("master", "m", "v"), (o.master.dtype, o.m.dtype, o.v.dtype))

    def full_ema(self):
        """The EMA over the whole vector assembled from the holders, which must agree bit for bit."""
        return self._assemble(lambda i, lo, hi: [self.get_ema(i, lo, hi)], ("the EMA",),
                              (self.opts[self.members[0]].ema.dtype,))[0]
