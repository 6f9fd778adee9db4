"""FT-ZeRO-1 compact (paged) optimizer state, host logic (no GPU): pool sizing, page lifetimes during a re-shard, and
agreement with the full-size state under random walks of kills, rejoins and split commits."""

from __future__ import annotations

import numpy as np
import pytest

from _zero1_sim import NUMEL, UNITS, _mask, _Sim
from torchft_b200.models.llama import CONFIGS
from torchft_b200.parallel.zero1 import (ShardLayout, intersect_ranges, merge_ranges, page_ranges, plan_quorum,
                                         pool_pages, total)

SHIFT = 8  # 256-element pages: the 12 168-element test vector spans 48 of them
PAGE = 1 << SHIFT


class _CompactSim:
    """The state protocol of ``_Sim`` with every replica's state in a page pool behind a page table, re-sharded the way
    ``Zero1Optimizer`` does it in compact mode, by the same planner (``plan_quorum``) and its page steps. Ranks run
    each phase one after the other, every rank's frees and allocations before anybody pulls, so a page freed too early
    is reused and poisoned before a peer reads it."""

    POISON = -7.0

    def __init__(self, n, k, min_world, cap=None):
        self.L = ShardLayout(UNITS, k)
        self.min_world = min_world
        self.cap = cap or pool_pages(self.L, min_world, PAGE)
        self.pool = {r: np.full(self.cap * PAGE, np.nan) for r in range(n)}
        self.table = {r: {} for r in range(n)}
        self.free = {r: list(range(self.cap)) for r in range(n)}
        self.hold = {r: [] for r in range(n)}
        self.t = {r: 0 for r in range(n)}
        self.members = list(range(n))
        self.lost = 0
        self.peak = 0

    def restart(self, m):
        self.pool[m][:] = np.nan
        self.table[m], self.free[m], self.hold[m], self.t[m] = {}, list(range(self.cap)), [], 0

    def _idx(self, m, lo, hi):
        e = np.arange(lo, hi)
        slots = np.array([self.table[m][p] for p in (e >> SHIFT)])
        return slots * PAGE + (e & (PAGE - 1))

    def read(self, m, lo, hi):
        return self.pool[m][self._idx(m, lo, hi)]

    def _pages(self, m):
        return merge_ranges([(p, p + 1) for p in self.table[m]])

    def _free_pages(self, m, pages):
        for lo, hi in pages:
            for p in range(lo, hi):
                if p in self.table[m]:
                    self.free[m].append(self.table[m].pop(p))

    def configure(self, members, abort_after_alloc=False):
        """``abort_after_alloc``: the re-shard fails after every rank freed and allocated (a peer died before the barrier)."""
        world = len(members)
        if world < self.min_world:
            raise RuntimeError(f"quorum of {world} is below min_world")
        published = {i: {"t": self.t[m], "hold": self.hold[m], "pages": [(p, s, 1) for p, s in sorted(self.table[m].items())]}
                     for i, m in enumerate(members)}
        plans = plan_quorum(self.L, world, published, SHIFT)
        worst = max(p.peak for p in plans.values())
        if worst > self.cap:
            raise RuntimeError(f"needs {worst} pages")
        sources = {i: merge_ranges([(lo, hi) for p in plans.values() for s, lo, hi in p.pulls if s == i]) for i in range(world)}
        for i, m in enumerate(members):  # 1. free what is neither kept nor a source, 2. allocate the new pages
            p = plans[i]
            assert not intersect_ranges(p.free_first, page_ranges(sources[i], SHIFT)), "a page freed while a peer sources from it"
            self._free_pages(m, p.free_first)
            self.hold[m] = p.hold_mid
            self.free[m].sort(reverse=True)
            for lo, hi in p.allocate:
                for pg in range(lo, hi):
                    self.table[m][pg] = slot = self.free[m].pop()
                    self.pool[m][slot * PAGE:(slot + 1) * PAGE] = self.POISON
            self.peak = max(self.peak, len(self.table[m]))
        if abort_after_alloc:
            return
        for i, m in enumerate(members):  # 3. pull through both page tables, seed what nobody holds
            p = plans[i]
            for src, lo, hi in p.pulls:
                self.pool[m][self._idx(m, lo, hi)] = self.read(members[src], lo, hi)
            for lo, hi in p.lost:
                self.pool[m][self._idx(m, lo, hi)] = -1000.0 if p.counted else 0.0
                self.lost += (hi - lo) if p.counted else 0
        for i, m in enumerate(members):  # 6. after the barrier: drop the pages kept only for peers
            self._free_pages(m, plans[i].free_last)
            self.hold[m], self.t[m] = plans[i].hold, plans[i].tmax
            assert self._pages(m) == page_ranges(self.hold[m], SHIFT)
        self.members = list(members)

    def step(self, commit_on=None):
        world = len(self.members)
        for i, m in enumerate(self.members):
            if commit_on is not None and m not in commit_on:
                continue
            for lo, hi in self.L.held(i, world):
                self.pool[m][self._idx(m, lo, hi)] += 1
            self.hold[m] = self.L.held(i, world)
            self.t[m] += 1


@pytest.mark.parametrize("seed", range(6))
def test_random_walk_compact_reads_back_the_full_size_state(seed):
    """The walk of ``test_random_walk_of_kills_rejoins_and_split_commits_keeps_holders_consistent``, driven through the
    full-size emulation and the paged one in lockstep. Compact state drops the ranges a rank held before a re-shard but
    no longer holds, so it can lose an element the full-size state still had; everywhere else it reads back the same
    values. A quorum below ``min_world`` is refused. Several members may leave or join at once here, which
    ``pool_pages`` does not size for, so the pools get one slot per page of the vector (``state_pages=``)."""
    rng = np.random.default_rng(2000 + seed)
    n, k = 8, int(rng.integers(1, 4))
    min_world = int(rng.integers(1, 5))
    flat, comp = _Sim(n, k), _CompactSim(n, k, min_world, cap=(NUMEL + PAGE - 1) // PAGE)
    flat.configure(range(n))
    comp.configure(range(n))
    assert comp.lost == 0
    comp_lost = np.zeros(NUMEL, bool)
    alive = set(range(n))

    def reconfigure(members):
        members = sorted(members)
        if len(members) < min_world:
            with pytest.raises(RuntimeError):
                comp.configure(members)
            return False
        tmax = max(comp.t[m] for m in members)
        before = (flat.lost, comp.lost)
        avail = np.zeros(NUMEL, bool)
        for m in members:
            if comp.t[m] == tmax:
                avail |= _mask(comp.hold[m], NUMEL)
        flat.configure(members)
        comp.configure(members)
        for i, m in enumerate(members):
            if tmax > 0:
                comp_lost[_mask(comp.L.held(i, len(members)), NUMEL) & ~avail] = True
        assert comp.lost - before[1] >= flat.lost - before[0]
        return True

    for _ in range(120):
        ev = rng.random()
        if ev < 0.45:
            flat.step(), comp.step()
        elif ev < 0.55 and len(flat.members) > 1:
            sub = [m for m in flat.members if rng.random() < 0.6] or [flat.members[0]]
            flat.step(commit_on=sub), comp.step(commit_on=sub)
            reconfigure(flat.members)
        elif ev < 0.8 and len(alive) > 1:
            gone = [int(m) for m in rng.choice(sorted(alive), size=int(rng.integers(1, min(3, len(alive)))), replace=False)]
            if reconfigure(alive - set(gone)):
                alive -= set(gone)
        else:
            dead = sorted(set(range(n)) - alive)
            back = dead[: int(rng.integers(1, 3))]
            for m in back:
                flat.state[m], flat.hold[m], flat.t[m] = np.zeros(NUMEL), [(0, NUMEL)], 0
                comp.restart(m)
            alive |= set(back)
            if dead:
                assert reconfigure(alive)
        assert comp.peak <= comp.cap
        world = len(comp.members)
        tmax = max(comp.t[m] for m in comp.members)
        for i, m in enumerate(comp.members):
            if comp.t[m] != tmax:
                continue
            for lo, hi in comp.L.held(i, world):
                ok = ~comp_lost[lo:hi]
                got = comp.read(m, lo, hi)
                assert not np.isnan(got).any() and not (got == _CompactSim.POISON).any()
                assert (got[ok] == flat.state[m][lo:hi][ok]).all(), (seed, m, lo, hi)


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("min_world", [2, 4, 7])
def test_every_single_loss_and_join_fits_the_pool(k, min_world):
    """Walk every single-member loss and join inside ``[min_world, 8]`` after a committed step: the peak pages of every
    rank stay within ``pool_pages``, no state is lost when ``k >= 2``, and one member fewer than ``min_world`` raises."""
    for w in range(min_world, 9):
        for d in range(w):  # member d is lost
            sim = _CompactSim(w, k, min_world)
            sim.configure(range(w))
            sim.step()
            if w - 1 < min_world:
                with pytest.raises(RuntimeError):
                    sim.configure([m for m in range(w) if m != d])
                continue
            sim.configure([m for m in range(w) if m != d])
            assert k == 1 or sim.lost == 0
            assert sim.peak <= sim.cap
        for j in range(w + 1 if w < 8 else 0):  # a member without state joins at quorum rank j
            sim = _CompactSim(w + 1, k, min_world)
            sim.configure(range(w))
            sim.step()
            sim.configure(list(range(j)) + [w] + list(range(j, w)))
            assert sim.lost == 0 and sim.peak <= sim.cap


def test_layout_change_at_t0_counts_nothing_lost():
    """Before the first committed update every replica holds the same seed, so slices nobody holds yet are seeded, not lost."""
    sim = _CompactSim(4, 1, 2)
    sim.configure(range(4))
    sim.configure([0, 2, 3])  # k = 1: rank 1's slices had no other holder
    assert sim.lost == 0
    sim.step()
    sim.configure([0, 2])
    assert sim.lost > 0


def _llama_units(cfg, align=128):
    """Stage ranges of ``FaultTolerantTrainer`` (forward order; the flat buffer stores the stages in reverse)."""
    d, f, v = cfg.dim, cfg.ffn_dim, cfg.vocab_size
    pad = lambda n: (n + align - 1) // align * align  # noqa: E731
    block = [d, (cfg.n_heads + 2 * cfg.n_kv_heads) * cfg.head_dim * d, d * d, d, 2 * f * d, d * f]
    sizes = [pad(v * d)] + [sum(map(pad, block))] * cfg.n_layers + [pad(d) + pad(v * d)]
    out, hi = [], sum(sizes)
    for n in sizes:
        out.append((hi - n, hi))
        hi -= n
    return out


def test_llama3_8b_page_counts():
    """Per GPU, llama3_8b, k = 2, 64 Ki-element pages: fp32 master/m/v take 22.5 GiB at W = 8 and 25.7 GiB at W = 7
    (89.7 GiB full-size), and a pool for min_world = 7 rides through 8 -> 7 and 7 -> 8 in at most 35.3 GiB."""
    units = _llama_units(CONFIGS["llama3_8b"])
    assert len(units) == 34 and total(units) == 8_030_261_248
    L = ShardLayout(tuple(units), 2)
    gib = lambda pages: round(pages * (1 << 16) * 12 / 2**30, 1)  # noqa: E731
    steady = {w: max(total(page_ranges(L.held(r, w), 16)) for r in range(w)) for w in (7, 8)}
    assert gib(steady[8]) == 22.5 and gib(steady[7]) == 25.7
    cap = pool_pages(L, 7, 1 << 16)
    assert gib(cap) == 35.3 and cap >= steady[7]
    assert pool_pages(L, 8, 1 << 16) == steady[8]


def test_page_ranges_and_pool_pages_arguments():
    assert page_ranges([(0, 1), (255, 257), (1024, 1024)], 8) == [(0, 2)]
    assert page_ranges([(512, 768)], 8) == [(2, 3)]
    L = ShardLayout(UNITS, 2)
    assert pool_pages(L, 1, PAGE) == (NUMEL + PAGE - 1) // PAGE  # a quorum of one holds everything
    with pytest.raises(ValueError):
        pool_pages(L, 0, PAGE)
    with pytest.raises(AssertionError):
        pool_pages(L, 2, 100)


@pytest.mark.parametrize("k", [1, 2])
def test_reshard_that_fails_before_the_barrier_claims_only_pages_it_kept(k):
    """A peer dies after every rank freed and allocated for the next quorum but before anybody pulled. The ranks keep
    their old update count; what they claim afterwards must still be backed by pages with the old data, so the next
    re-shard pulls or re-seeds (and counts) everything else and never reads a freed or freshly allocated page."""
    flat, comp = _Sim(6, k), _CompactSim(6, k, 2)
    for sim in (flat, comp):
        sim.configure(range(6))
        sim.step(), sim.step()
    comp.configure([0, 1, 2, 4, 5], abort_after_alloc=True)  # member 3 dies in the middle of this re-shard
    for m in range(6):
        assert all(comp.table[m].get(p, -1) >= 0 for lo, hi in page_ranges(comp.hold[m], SHIFT) for p in range(lo, hi))
        for lo, hi in comp.hold[m]:
            assert (comp.read(m, lo, hi) == 2).all()
    members = [0, 1, 2, 4, 5]  # the retry of the same quorum
    flat.configure(members)
    comp.configure(members)
    assert comp.lost >= flat.lost and (k == 1 or flat.lost == 0)
    for i, m in enumerate(members):
        for lo, hi in comp.L.held(i, len(members)):
            got = comp.read(m, lo, hi)
            assert not np.isnan(got).any() and not (got == _CompactSim.POISON).any()
            assert ((got == 2) | (got == -1000.0)).all()
    assert comp.lost == int(sum((comp.read(m, lo, hi) == -1000.0).sum()
                                for i, m in enumerate(members) for lo, hi in comp.L.held(i, len(members))))
