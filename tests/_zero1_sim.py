"""The geometry and the numpy emulation of the FT-ZeRO-1 state protocol that the CPU tests share."""

from __future__ import annotations

import numpy as np

from torchft_b200.parallel.zero1 import ShardLayout, plan_quorum

UNITS = ((0, 4096), (4096, 4096 + 8 * 1001), (4096 + 8 * 1001, 4096 + 8 * 1001 + 64))
NUMEL = UNITS[-1][1]


def _mask(rs, n):
    m = np.zeros(n, bool)
    for lo, hi in rs:
        m[lo:hi] = True
    return m


class _Sim:
    """Numpy emulation of N replicas running the FT-ZeRO-1 state protocol (update = +1 on held ranges), re-sharded by
    the optimizer's own planner (``plan_quorum``); only the state arrays and the counters are the emulation's."""

    def __init__(self, n, k):
        self.L = ShardLayout(UNITS, k)
        self.state = {r: np.zeros(NUMEL) for r in range(n)}      # every replica seeds identically
        self.hold = {r: [(0, NUMEL)] for r in range(n)}
        self.t = {r: 0 for r in range(n)}
        self.members = list(range(n))
        self.lost = 0
        self.read = 0

    def configure(self, members, ckpt=None):
        """``ckpt``: checkpoint files for ``plan_quorum``, whose file objects are the arrays of values they store."""
        self.members = list(members)
        published = {i: {"t": self.t[m], "hold": self.hold[m]} for i, m in enumerate(members)}
        plans = plan_quorum(self.L, len(members), published, ckpt=ckpt)
        for i, m in enumerate(members):  # a source never writes the ranges it is read from: they are current there
            p = plans[i]
            for src, lo, hi in p.pulls:
                self.state[m][lo:hi] = self.state[members[src]][lo:hi]
            for vals, off, lo, hi in p.reads:
                self.state[m][lo:hi] = vals[off:off + hi - lo]
                self.read += hi - lo
            for lo, hi in p.lost:
                self.state[m][lo:hi] = -1000.0 if p.counted else 0.0
                self.lost += (hi - lo) if p.counted else 0
            self.hold[m], self.t[m] = p.hold, p.tmax

    def step(self, commit_on=None):
        world = len(self.members)
        for i, m in enumerate(self.members):
            if commit_on is not None and m not in commit_on:
                continue
            for lo, hi in self.L.held(i, world):
                self.state[m][lo:hi] += 1
            self.hold[m] = self.L.held(i, world)
            self.t[m] += 1

    def check(self):
        world = len(self.members)
        tmax = max(self.t[m] for m in self.members)
        for i, m in enumerate(self.members):
            for lo, hi in self.L.held(i, world):
                assert (self.state[m][lo:hi] == tmax).all(), (m, lo, hi)
