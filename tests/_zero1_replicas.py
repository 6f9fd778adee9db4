"""FT-ZeRO-1 replicas in one process on one GPU, for the GPU tests: ranks of ``SymmetricComm.virtual_world``
(pre-signalled), each with a ``Zero1Optimizer`` over the slice of ``ProcessGroupB200`` it uses, configured on one thread
per rank and stepped in the Manager's order (enqueue / update / wait / resolved)."""

from __future__ import annotations

import threading
from datetime import timedelta

import torch

HP = (1e-2, 0.9, 0.95, 1e-8, 0.1)  # lr, b1, b2, eps, wd
SHIFT = 8  # paged state: 256-element pages, so unit and slice bounds fall inside pages


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


def ref_adamw(master, m, v, g, t):
    """Step ``t`` of fp32 AdamW with ``HP`` on gradient ``g``, in place: the reference of the update kernel."""
    lr, b1, b2, eps, wd = HP
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    denom = v.sqrt() / (bc2 ** 0.5) + eps
    master.mul_(1 - lr * wd).addcdiv_(m, denom, value=-lr / bc1)


def seeded_weights(numel, seed=2):
    dev = torch.device("cuda", 0)
    return (torch.randn(numel, device=dev, generator=torch.Generator(device=dev).manual_seed(seed)) * 0.05).bfloat16()


class Replicas:
    """``n`` virtual ranks, each with a ``Zero1Optimizer`` over ``units`` (``k`` holders per slice, ``compact`` state
    pooled for ``min_world``, clipping at ``max_norm``, ``M`` micro-batches per step), seeded from the same weights
    (``init``, default :func:`seeded_weights`)."""

    def __init__(self, n, units, k=2, compact=False, min_world=1, max_norm=None, M=1, init=None):
        from torch.distributed import HashStore

        from torchft_b200.parallel.symm_mem import SymmetricComm
        from torchft_b200.parallel.zero1 import GNORM_UNITS, ShardLayout, pool_pages

        self.units, self.numel = list(units), units[-1][1]
        self.k, self.compact, self.min_world, self.max_norm, self.M = k, compact, min_world, max_norm, M
        n_state = (pool_pages(ShardLayout(tuple(units), k), min_world, 1 << SHIFT) << SHIFT) if compact else self.numel
        seg = {"z1_grad": self.numel * 2, "z1_param": self.numel * 2, "z1_gnorm": GNORM_UNITS * 8,
               **{x: n_state * 4 for x in ("z1_master", "z1_m", "z1_v")}}
        self.comms = SymmetricComm.virtual_world(n, seg, presignal=True, timeout=timedelta(seconds=20))
        self.init = seeded_weights(self.numel) if init is None else init
        self.opts = [self.make(c) for c in self.comms]
        for o in self.opts:
            o.param.copy_(self.init)
            o.seed_master()
        self.store = HashStore()
        self.members = list(range(n))
        self.pending = None

    def make(self, comm):
        """A fresh optimizer on rank ``comm`` (a restarted process), configured like the others."""
        from torchft_b200.parallel.zero1 import Zero1Optimizer

        return Zero1Optimizer(PG(comm), self.numel, units=self.units, lr=HP[0], betas=HP[1:3], eps=HP[3],
                              weight_decay=HP[4], replication=self.k, blocks=4, compact=self.compact,
                              min_world=self.min_world, page_shift=SHIFT, max_grad_norm=self.max_norm,
                              grad_accum_steps=self.M)

    def configure(self, members, epoch):
        """The re-shard of every member for quorum ``members`` (quorum rank = position), one thread per member."""
        from torch.distributed import PrefixStore

        from torchft_b200.parallel.symm_mem import SymmetricComm

        self.settle()
        SymmetricComm.virtual_quorum(self.comms, members, epoch)
        errs = []

        def run(rank, m):
            try:
                self.opts[m]._on_configured(PrefixStore(f"q/{epoch}", self.store), rank, len(members), epoch)
            except Exception as e:  # noqa: BLE001
                errs.append(e)

        ts = [threading.Thread(target=run, args=(rank, m)) for rank, m in enumerate(members)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert not errs, errs
        torch.cuda.synchronize()
        self.members = list(members)

    def settle(self):
        """Resolve the verdicts of the last step, as the Manager does when the next one starts."""
        if self.pending is not None:
            for m, s in self.pending.items():
                self.opts[m].resolved(self.opts[m].wait(s))
            self.pending = None

    def step(self, raws, skip=None, veto=None, reduce=True, sync=True):
        """One step: micro-batch ``m`` writes ``raws[m][rank]`` into quorum rank ``rank``'s gradient and (``reduce``)
        every member reduces every unit, except ``skip = (unit, micro)`` on every member. Then every member enqueues
        its verdict (member ``veto`` votes no) and its update; ``sync`` waits for the device at the end."""
        self.settle()
        scale = 1.0 / (len(self.members) * self.M)
        for micro, raw in enumerate(raws):
            for rank, i in enumerate(self.members):
                self.opts[i].grad.copy_(raw[rank])
            if reduce:
                for i in self.members:
                    for u in range(len(self.units)):
                        if skip != (u, micro):
                            self.opts[i].reduce_scatter(u, scale, True, micro)
        self.pending = {i: self.opts[i].enqueue(i != veto) for i in self.members}
        for i in self.members:
            self.opts[i].update()
        if sync:
            torch.cuda.synchronize()

    def verdicts(self):
        return {i: self.opts[i].comm.verdict(s) for i, s in self.pending.items()}
