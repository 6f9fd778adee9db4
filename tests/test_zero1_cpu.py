"""FT-ZeRO-1 host logic (no GPU): interval arithmetic, ownership layout, re-shard planning, device-commit bookkeeping."""

from __future__ import annotations

import random
from datetime import timedelta
from unittest.mock import MagicMock, create_autospec, patch

import numpy as np
import pytest
from torch.distributed import TCPStore

from _zero1_sim import NUMEL, UNITS, _mask, _Sim
from torchft_b200.parallel.zero1 import (ShardLayout, intersect_ranges, merge_ranges, page_ranges, plan_quorum,
                                         subtract_ranges, total)


def test_interval_arithmetic_matches_bitmaps():
    rnd = random.Random(3)
    n = 200
    for _ in range(200):
        a = [tuple(sorted((rnd.randrange(n), rnd.randrange(n)))) for _ in range(rnd.randrange(6))]
        b = [tuple(sorted((rnd.randrange(n), rnd.randrange(n)))) for _ in range(rnd.randrange(6))]
        ma, mb = _mask(a, n), _mask(b, n)
        assert (_mask(merge_ranges(a), n) == ma).all()
        assert (_mask(intersect_ranges(a, b), n) == (ma & mb)).all()
        assert (_mask(subtract_ranges(a, b), n) == (ma & ~mb)).all()
        m = merge_ranges(a)
        assert all(x[1] < y[0] for x, y in zip(m, m[1:])) and all(lo < hi for lo, hi in m)


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_layout_every_element_has_exactly_k_holders_and_one_primary(world, k):
    L = ShardLayout(UNITS, k)
    holders = np.zeros(NUMEL, int)
    prim = np.zeros(NUMEL, int)
    for r in range(world):
        holders += _mask(L.held(r, world), NUMEL)
        prim += _mask(L.primary(r, world), NUMEL)
        assert (_mask(L.primary(r, world), NUMEL) <= _mask(L.held(r, world), NUMEL)).all()
    assert (prim == 1).all()
    assert (holders == min(k, world)).all()
    # slice bounds are 8-element (16-byte) aligned, as the kernels require
    for u in range(len(UNITS)):
        for s in range(world):
            lo, hi = L.slice_bounds(u, world, s)
            assert lo % 8 == 0 and hi % 8 == 0 and UNITS[u][0] <= lo <= hi <= UNITS[u][1]


def test_reshard_survives_any_single_loss_join_and_split_commit():
    sim = _Sim(8, 2)
    sim.configure(range(8))
    sim.step(), sim.step()
    sim.check()
    for dead in (0, 3, 7):
        s = _Sim(8, 2)
        s.configure(range(8)); s.step(); s.step()
        s.configure([m for m in range(8) if m != dead])
        assert s.lost == 0
        s.check(); s.step(); s.check()
        # the dead replica restarts with seed state (t = 0) and rejoins
        s.state[dead] = np.zeros(NUMEL); s.hold[dead] = [(0, NUMEL)]; s.t[dead] = 0
        s.configure(range(8))
        assert s.lost == 0
        s.check(); s.step(); s.check()
    # split commit: replica 5 missed update 3 that the others applied -> it re-pulls everything it holds
    sim.step(commit_on=[m for m in range(8) if m != 5])
    sim.configure(range(8))
    assert sim.lost == 0
    sim.check()


def test_k1_loses_state_and_k2_loses_only_on_adjacent_double_failure():
    s = _Sim(4, 1)
    s.configure(range(4)); s.step()
    s.configure([0, 1, 2])
    assert s.lost > 0
    s = _Sim(8, 2)
    s.configure(range(8)); s.step()
    s.configure([m for m in range(8) if m not in (2, 5)])  # non-adjacent: every slice keeps a holder
    assert s.lost == 0
    s = _Sim(8, 2)
    s.configure(range(8)); s.step()
    s.configure([m for m in range(8) if m not in (2, 3)])  # slice 2 lived on exactly {2, 3}
    # both new holders of the orphaned ranges re-seed them
    assert s.lost == 2 * total([ShardLayout(UNITS, 2).slice_bounds(u, 8, 2) for u in range(len(UNITS))])


@pytest.mark.parametrize("paged", [False, True])
def test_plan_quorum_holdings_after_and_losses_at_t0(paged):
    """What a rank claims after a re-shard is what its state really keeps. Full-size state keeps every range it held at
    ``tmax``, also those outside the new layout, and peers may pull them at a later quorum; paged state keeps exactly its
    new slices, not the whole pages they touch. A slice nobody holds at t = 0 is seeded, and not counted as lost."""
    shift = 8
    L = ShardLayout(UNITS, 2)

    def pub(t, holds):
        pages = lambda h: [(lo, 0, hi - lo) for lo, hi in page_ranges(h, shift)]  # noqa: E731
        return {r: {"t": t, "hold": h, **({"pages": pages(h)} if paged else {})} for r, h in enumerate(holds)}

    old = [L.held(r, 4) for r in range(4)]
    plans = plan_quorum(L, 3, pub(5, old[:3]), shift if paged else None)  # member 3 is gone after update 5
    for r, p in plans.items():
        new = L.held(r, 3)
        assert p.tmax == 5 and p.counted
        assert p.need == subtract_ranges(new, old[r]) and not p.lost
        assert p.hold == (new if paged else merge_ranges(old[r] + new))
    assert any(subtract_ranges(old[r], L.held(r, 3)) for r in range(3)), "the test needs ranges the new layout drops"
    if paged:
        assert any(page_ranges(L.held(r, 3), shift) != [(lo >> shift, hi >> shift) for lo, hi in L.held(r, 3)]
                   for r in range(3)), "the test needs slices that end inside a page"
    # the first quorum of paged state, or a quorum of restarted replicas: nobody holds anything at t = 0
    for p in plan_quorum(L, 3, pub(0, [[]] * 3), shift if paged else None).values():
        assert p.lost == p.need and not p.pulls and not p.counted
    # a split commit: rank 1 missed update 6, so what it held is not current
    plans = plan_quorum(L, 3, pub(6, [L.held(r, 3) for r in range(3)]) | {1: pub(5, [L.held(1, 3)] * 2)[1]},
                        shift if paged else None)
    assert plans[1].need == L.held(1, 3) and plans[1].hold == L.held(1, 3) and not plans[1].lost


# ----------------------------------------------------------------------------- Manager.commit_on_device
class _FakeCommitter:
    def __init__(self, verdicts):
        self.verdicts = list(verdicts)
        self.enqueued, self.resolved_with = [], []

    def enqueue(self, host_ok):
        self.enqueued.append(host_ok)
        return len(self.enqueued)

    def wait(self, seq, timeout=None):
        return self.verdicts[seq - 1] and self.enqueued[seq - 1]

    def resolved(self, verdict):
        self.resolved_with.append(verdict)


def _manager(client_mock, **kw):
    from torchft_b200._C import QuorumResult
    from torchft_b200.manager import Manager
    from torchft_b200.process_group import ProcessGroup

    store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
    store.set("manager_addr", "dummy")
    store.set("replica_id", "dummy_id")
    pg = create_autospec(ProcessGroup)
    pg.errored.return_value = None
    m = Manager(pg=pg, min_replica_size=2, load_state_dict=MagicMock(), state_dict=lambda: {}, rank=1, world_size=1,
                store_addr="127.0.0.1", store_port=store.port, timeout=timedelta(seconds=10),
                checkpoint_transport=MagicMock(), **kw)
    q = QuorumResult()
    q.quorum_id, q.replica_rank, q.replica_world_size = 7, 0, 2
    q.max_step, q.max_replica_rank, q.max_world_size, q.heal = 0, 0, 2, False
    q.store_address = f"127.0.0.1:{store.port}"
    q.replica_ids = ["a", "b"]
    client_mock()._quorum.return_value = q
    return m, store, q


def test_commit_on_device_defers_and_books_at_next_quorum():
    with patch("torchft_b200.manager.ManagerClient", autospec=True) as client:
        m, store, q = _manager(client)
        try:
            c = _FakeCommitter([True, False, True])
            m.start_quorum()
            assert m.commit_on_device(c) is None          # deferred: no RPC, no sync
            assert client().should_commit.call_count == 0
            assert c.resolved_with == []
            m.start_quorum()                               # the quorum thread books step 0's verdict first
            m.wait_quorum()
            assert c.resolved_with == [True]
            assert client()._quorum.call_args.kwargs["step"] == 1
            assert m.commit_on_device(c) is None
            assert m.current_step() == 1 and c.resolved_with == [True, False]   # asking resolves; failed commit
            assert m._commit_failures == 1
            m.start_quorum(); m.wait_quorum()
            assert client()._quorum.call_args.kwargs["commit_failures"] == 1
            m.commit_on_device(c)
            assert m.batches_committed() == 4 and m.current_step() == 2
        finally:
            m.shutdown(wait=False)


def test_commit_on_device_vetoes_when_errored_or_too_few_replicas_and_syncs_when_serving_a_heal():
    with patch("torchft_b200.manager.ManagerClient", autospec=True) as client:
        m, store, q = _manager(client)
        try:
            c = _FakeCommitter([True] * 4)
            m.start_quorum(); m.wait_quorum()
            m.report_error(RuntimeError("boom"))
            m.commit_on_device(c)
            assert c.enqueued == [False] and m.current_step() == 0
            q.max_world_size = 1                           # not enough participants
            m.start_quorum()
            m.commit_on_device(c)
            assert c.enqueued == [False, False] and m.current_step() == 0
            q.max_world_size = 2
            q.recover_dst_replica_ranks = [1]              # we serve a checkpoint this step -> synchronous verdict
            m.start_quorum()
            assert m.commit_on_device(c) is True
            assert m._checkpoint_transport.disallow_checkpoint.call_count == 1
            assert m._step == 1
        finally:
            m.shutdown(wait=False)


# ----------------------------------------------------------------------------- liveness-driven abort
def test_liveness_watch_aborts_the_group_when_a_quorum_member_stops_heartbeating(monkeypatch):
    """Reference analogue: user-space op timeout -> ncclCommAbort (process_group.py:738-763), which costs the full
    collective timeout. Here the Manager asks the Lighthouse who is still heart-beating and releases the spinning
    kernels (pg.abort()) about one heartbeat timeout after a peer went silent."""
    import threading
    import time

    from torchft_b200.bench_utils import loopback
    from torchft_b200.coordination import LighthouseServer
    from torchft_b200.manager import Manager
    from torchft_b200.process_group import ProcessGroupDummy

    monkeypatch.setenv("TORCHFT_B200_LIVENESS_ABORT", "1")
    aborts = []

    class PG(ProcessGroupDummy):
        def abort(self, *a, **k):
            aborts.append(time.monotonic())

        def errored(self):
            return None

    transport = MagicMock()
    transport.metadata.return_value = "none"
    lh = LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=1000, heartbeat_timeout_ms=600)
    addr = loopback(lh.address())
    stores, managers = [], []
    for name in ("live_0", "live_1"):
        st = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
        stores.append(st)
        managers.append(Manager(pg=PG(0, 1), load_state_dict=lambda s: None, state_dict=lambda: {}, min_replica_size=1, rank=0,
                                world_size=1, store_addr="127.0.0.1", store_port=st.port, lighthouse_addr=addr, replica_id=name,
                                timeout=timedelta(seconds=5), init_sync=False, checkpoint_transport=transport))
    try:
        ts = [threading.Thread(target=lambda m=m: (m.start_quorum(), m.wait_quorum())) for m in managers]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert len(managers[0]._quorum_members) == 2
        time.sleep(0.8)
        assert aborts == []                      # everybody alive: nothing is aborted
        t0 = time.monotonic()
        managers[1]._manager.shutdown()          # the peer's heartbeats stop (process death)
        while not aborts and time.monotonic() - t0 < 5:
            time.sleep(0.05)
        assert aborts and aborts[0] - t0 < 2.5   # ~ heartbeat timeout + one poll period, not the 5 s op timeout
    finally:
        for m in managers:
            m.shutdown(wait=False)
        lh.shutdown()


# ----------------------------------------------------------------------------- randomized protocol walk
@pytest.mark.parametrize("seed", range(6))
def test_random_walk_of_kills_rejoins_and_split_commits_keeps_holders_consistent(seed):
    """Long random sequences of membership changes (several replicas may die or rejoin in one transition), committed
    steps and split commits, for k in {1, 2, 3}. Checked after every event against an independent bitmap oracle:
    (1) every holder of an element carries the same value (holders are bit-identical replicas of a slice);
    (2) an element is counted lost exactly when no surviving up-to-date replica held it -- never otherwise; in particular
        never while every replica is alive and none missed a commit (after a split commit the slices whose holders all
        missed the update ARE re-seeded: stale state is never mixed with current state);
    (3) elements that were never lost equal the number of committed updates."""
    rng = np.random.default_rng(1000 + seed)
    n, k = 8, int(rng.integers(1, 4))
    sim = _Sim(n, k)
    sim.configure(range(n))
    ever_lost = np.zeros(NUMEL, dtype=bool)
    alive = set(range(n))

    def reconfigure(members):
        members = sorted(members)
        tmax = max(sim.t[m] for m in members)
        available = np.zeros(NUMEL, dtype=bool)  # oracle: somebody up to date in the new quorum holds it
        for m in members:
            if sim.t[m] == tmax:
                available |= _mask(sim.hold[m], NUMEL)
        before = sim.lost
        stale = any(sim.t[m] != tmax for m in members)
        sim.configure(members)
        world = len(members)
        expect_lost = 0
        for i, m in enumerate(members):
            need = _mask(sim.L.held(i, world), NUMEL)
            gone = need & ~available
            expect_lost += int(gone.sum())
            ever_lost[gone] = True
        assert sim.lost - before == expect_lost
        if len(alive) == n and not stale and expect_lost:
            raise AssertionError("state lost although every replica is alive and up to date")

    def check():
        members, world = sim.members, len(sim.members)
        tmax = max(sim.t[m] for m in members)
        value = np.full(NUMEL, np.nan)
        for i, m in enumerate(members):
            if sim.t[m] != tmax:
                continue
            for lo, hi in sim.L.held(i, world):
                seg, cur = sim.state[m][lo:hi], value[lo:hi]
                fresh = np.isnan(cur)
                assert (seg[~fresh] == cur[~fresh]).all(), "holders of one slice disagree"
                cur[fresh] = seg[fresh]
        ok = ~ever_lost & ~np.isnan(value)
        assert (value[ok] == tmax).all()
        assert not np.isnan(value).any(), "an element has no up-to-date holder inside the quorum"

    for _ in range(120):
        ev = rng.random()
        if ev < 0.45:
            sim.step()
        elif ev < 0.55 and len(sim.members) > 1:
            # split commit: a random non-empty strict subset applies the update, then everybody meets in a new quorum
            sub = [m for m in sim.members if rng.random() < 0.6] or [sim.members[0]]
            sim.step(commit_on=sub)
            reconfigure(sim.members)
        elif ev < 0.8 and len(alive) > 1:
            for m in rng.choice(sorted(alive), size=int(rng.integers(1, min(3, len(alive)))), replace=False):
                alive.discard(int(m))
            reconfigure(alive)
        else:
            dead = sorted(set(range(n)) - alive)
            for m in dead[: int(rng.integers(1, 3))]:
                sim.state[m] = np.zeros(NUMEL)  # restarted process: seed state, step 0
                sim.hold[m] = [(0, NUMEL)]
                sim.t[m] = 0
                alive.add(m)
            if dead:
                reconfigure(alive)
        check()
