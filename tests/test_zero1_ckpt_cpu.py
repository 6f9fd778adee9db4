"""FT-ZeRO-1 durable checkpoints, host logic (no GPU): the files of one quorum tile the flat vector, the read plan of a
restore at any world, newest-complete selection, the disk as holder of last resort in the random kill/rejoin walk, and
the file format's refusals."""

from __future__ import annotations

import json
import os

import numpy as np
import pytest

from _zero1_sim import NUMEL, UNITS, _mask, _Sim
from torchft_b200.checkpointing.sharded import (check_compatible, encode_header, file_name, read_header, scan,
                                                sections)
from torchft_b200.parallel.zero1 import (ShardLayout, ckpt_read_plan, intersect_ranges, merge_ranges,
                                         newest_complete_step, plan_quorum, total)


def _files(L, world, t=1):
    """What every rank of a quorum of ``world`` writes after a committed step: ``primary ∩ held``, packed."""
    out = []
    for r in range(world):
        ranges, off = [], 0
        for lo, hi in intersect_ranges(L.primary(r, world), L.held(r, world)):
            ranges.append((lo, hi, off))
            off += hi - lo
        out.append(({"T": t, "world": world, "rank": r, "ranges": ranges}, ranges))
    return out


@pytest.mark.parametrize("k", [1, 2, 3])
def test_files_tile_and_every_restore_reads_exactly_what_it_holds(k):
    L = ShardLayout(UNITS, k)
    for save_world in range(1, 9):
        files = _files(L, save_world)
        cover = np.zeros(NUMEL, int)
        contents = {}  # per file: the flat index stored at each element offset
        for h, ranges in files:
            buf = np.full(sum(hi - lo for lo, hi, _ in ranges), -1)
            for lo, hi, off in ranges:
                cover[lo:hi] += 1
                buf[off:off + hi - lo] = np.arange(lo, hi)
            contents[h["rank"]] = buf
        assert (cover == 1).all(), f"files of a quorum of {save_world} do not tile the vector"
        assert newest_complete_step([h for h, _ in files], NUMEL) == 1
        for world in range(1, 9):
            for r in range(world):
                need = L.held(r, world)
                reads = ckpt_read_plan(need, files)
                assert merge_ranges([(lo, hi) for _, _, lo, hi in reads]) == need
                assert total([(lo, hi) for _, _, lo, hi in reads]) == total(need), "an element is read twice"
                for h, off, lo, hi in reads:
                    assert any(a <= lo and hi <= b for a, b, _ in files[h["rank"]][1]), "read outside a written range"
                    assert (contents[h["rank"]][off:off + hi - lo] == np.arange(lo, hi)).all()


def test_newest_complete_step_falls_back_and_accepts_mixed_worlds():
    L = ShardLayout(UNITS, 2)
    h = lambda t, w: [f for f, _ in _files(L, w, t)]  # noqa: E731
    newest = h(5, 4)
    assert newest_complete_step(h(3, 4) + newest, NUMEL) == 5
    assert newest_complete_step(h(3, 4) + newest[:2] + newest[3:], NUMEL) == 3  # rank 2's file of step 5 is missing
    assert newest_complete_step(newest[:3], NUMEL) is None
    # step 7 from a quorum of 3 (ranks 0, 1) and a quorum of 2 (rank 1): complete because the union is
    w3, w2 = h(7, 3), h(7, 2)
    assert merge_ranges(sum(([(lo, hi) for lo, hi, _ in f["ranges"]] for f in w3[:2] + w2[1:]), [])) == [(0, NUMEL)]
    assert newest_complete_step(newest + w3[:2], NUMEL) == 5
    assert newest_complete_step(newest + w3[:2] + w2[1:], NUMEL) == 7
    with pytest.raises(ValueError):
        ckpt_read_plan([(0, NUMEL)], [(f, f["ranges"]) for f in w3[:2]])


def test_plan_quorum_reads_its_own_restore_else_the_first_checkpoint_that_covers():
    L = ShardLayout(UNITS, 1)

    def tagged(tag, files):
        return [(dict(h, tag=tag), r) for h, r in files]

    part, full = tagged("part", _files(L, 2)[:1]), tagged("full", _files(L, 2))  # part: rank 0's file of a quorum of 2
    fresh = lambda world: {r: {"t": 1, "hold": []} for r in range(world)}  # noqa: E731  (restored: t = T, holds nothing)
    sources = lambda p: {h["tag"] for h, _, _, _ in p.reads}  # noqa: E731
    plans = plan_quorum(L, 2, fresh(2), ckpt={0: part, 1: full})
    assert sources(plans[0]) == {"part"} and sources(plans[1]) == {"full"}
    assert all(not p.lost and merge_ranges([(lo, hi) for _, _, lo, hi in p.reads]) == L.held(r, 2) for r, p in plans.items())
    plans = plan_quorum(L, 3, fresh(3), ckpt={0: part, 1: full})
    assert sources(plans[2]) == {"full"} and not plans[2].lost  # rank 0's restore does not cover its slices
    plans = plan_quorum(L, 2, fresh(2), ckpt={0: part})
    assert not plans[1].reads and plans[1].lost == L.held(1, 2) and plans[1].counted


# ----------------------------------------------------------------------------- the disk in the random walk
class _DiskSim(_Sim):
    """``_Sim`` with durable checkpoints: ``save`` writes every member's ``primary ∩ hold`` at its own ``t``; a restarted
    member restores the newest complete step (``t = T``, holds nothing) and is armed; at the next quorum, ranges that
    no live holder at ``tmax`` has are read from the files when a member is armed at ``T == tmax`` (any rank may read
    them), and re-seeded otherwise. The optimizer's planner decides, as in ``Zero1Optimizer._on_configured``."""

    def __init__(self, n, k):
        super().__init__(n, k)
        self.files = []   # (header, ranges, values)
        self.armed = {}   # member -> T

    def save(self):
        world = len(self.members)
        for i, m in enumerate(self.members):
            ranges, vals, off = [], [], 0
            for lo, hi in intersect_ranges(self.L.primary(i, world), self.hold[m]):
                ranges.append((lo, hi, off))
                vals.append(self.state[m][lo:hi].copy())
                off += hi - lo
            self.files.append(({"T": self.t[m], "ranges": ranges}, ranges, np.concatenate(vals) if vals else np.zeros(0)))

    def restore(self, m):
        T = newest_complete_step([h for h, _, _ in self.files], NUMEL)
        assert T is not None
        self.state[m] = np.full(NUMEL, np.nan)  # the state arrives at the re-shard, from live holders or the files
        self.hold[m], self.t[m] = [], T
        self.armed[m] = T

    def configure(self, members):
        tmax = max(self.t[m] for m in members)
        files = [(vals, r) for h, r, vals in self.files if h["T"] == tmax]
        super().configure(members, ckpt={i: files for i, m in enumerate(members) if self.armed.get(m) == tmax})
        for m in members:
            self.armed.pop(m, None)


@pytest.mark.parametrize("seed", range(6))
def test_random_walk_with_restores_from_disk(seed):
    """The random kill/rejoin/split-commit walk of ``test_zero1_cpu`` plus saves, whole-job restarts from disk and
    partial restarts from disk next to live replicas, checked after every event against the bitmap oracle: holders
    agree, an element is lost exactly when neither an up-to-date holder nor a checkpoint at ``tmax`` has it, and every
    element never lost equals the number of committed updates."""
    rng = np.random.default_rng(3000 + seed)
    n, k = 8, int(rng.integers(1, 4))
    sim = _DiskSim(n, k)
    sim.configure(range(n))
    ever_lost = np.zeros(NUMEL, dtype=bool)
    alive = set(range(n))
    restores = 0

    def reconfigure(members):
        members = sorted(members)
        tmax = max(sim.t[m] for m in members)
        available = np.zeros(NUMEL, dtype=bool)
        for m in members:
            if sim.t[m] == tmax:
                available |= _mask(sim.hold[m], NUMEL)
        if any(sim.armed.get(m) == tmax for m in members):
            available[:] = True  # a complete checkpoint at tmax covers everything
        before = sim.lost
        sim.configure(members)
        world = len(members)
        expect = 0
        for i, m in enumerate(members):
            gone = _mask(sim.L.held(i, world), NUMEL) & ~available
            expect += int(gone.sum())
            ever_lost[gone] = True
        assert sim.lost - before == expect

    def check():
        members, world = sim.members, len(sim.members)
        tmax = max(sim.t[m] for m in members)
        value = np.full(NUMEL, np.nan)
        for i, m in enumerate(members):
            if sim.t[m] != tmax:
                continue
            for lo, hi in sim.L.held(i, world):
                seg, cur = sim.state[m][lo:hi], value[lo:hi]
                assert not np.isnan(seg).any(), "a held element was never filled"
                fresh = np.isnan(cur)
                assert (seg[~fresh] == cur[~fresh]).all(), "holders of one slice disagree"
                cur[fresh] = seg[fresh]
        ok = ~ever_lost & ~np.isnan(value)
        assert (value[ok] == tmax).all()
        assert not np.isnan(value).any()

    for _ in range(150):
        ev = rng.random()
        if ev < 0.4:
            sim.step()
        elif ev < 0.5:
            sim.save()
        elif ev < 0.58 and len(sim.members) > 1:
            sub = [m for m in sim.members if rng.random() < 0.6] or [sim.members[0]]
            sim.step(commit_on=sub)
            reconfigure(sim.members)
        elif ev < 0.75 and len(alive) > 1:
            for m in rng.choice(sorted(alive), size=int(rng.integers(1, min(3, len(alive)))), replace=False):
                alive.discard(int(m))
            reconfigure(alive)
        elif ev < 0.88:
            dead = sorted(set(range(n)) - alive)
            for m in dead[: int(rng.integers(1, 3))]:
                sim.state[m], sim.hold[m], sim.t[m] = np.zeros(NUMEL), [(0, NUMEL)], 0
                alive.add(m)
            if dead:
                reconfigure(alive)
        elif newest_complete_step([h for h, _, _ in sim.files], NUMEL) is not None:
            # restart from disk: everybody (a whole-job restart, at a new size) or a few next to live replicas
            everyone = rng.random() < 0.5
            back = sorted(range(n)) if everyone else sorted({int(m) for m in rng.choice(n, size=int(rng.integers(1, 4)))})
            if everyone:
                alive = set(int(m) for m in rng.choice(n, size=int(rng.integers(1, n + 1)), replace=False))
                back = sorted(alive)
            for m in back:
                sim.restore(m)
                alive.add(m)
            restores += 1
            lost_before = sim.lost
            reconfigure(alive)
            if everyone:
                assert sim.lost == lost_before, "a whole-job restore lost state"
        check()
    assert restores > 0 and sim.read > 0


# ----------------------------------------------------------------------------- file format
def _write(path, header, elements, tail=0):
    with open(path, "wb") as f:
        f.write(encode_header(header))
        f.write(b"\0" * (14 * elements - tail))


def _header(t, world, rank, ranges, numel=NUMEL, units=UNITS):
    e = sum(hi - lo for lo, hi, _ in ranges)
    return {"version": 1, "numel": numel, "units": [list(u) for u in units], "T": t, "step": t, "batches": t,
            "world": world, "rank": rank, "k": 1, "ranges": [list(r) for r in ranges], "elements": e,
            "sections": sections(e)}


def test_truncated_and_bad_files_are_skipped_and_a_mismatch_raises(tmp_path):
    L = ShardLayout(UNITS, 1)
    for t in (1, 2):
        for h, ranges in _files(L, 2, t):
            _write(tmp_path / file_name(t, 2, h["rank"]), _header(t, 2, h["rank"], ranges), total([(a, b) for a, b, _ in ranges]))
    hs = scan(str(tmp_path))
    assert newest_complete_step(hs, NUMEL) == 2
    h = hs[-1]
    assert h["data"] % 16 == 0 and all(v % 16 == 0 for v in h["sections"].values())
    assert os.path.getsize(h["path"]) == h["data"] + 14 * h["elements"]
    # a torn newest file: step 2 is incomplete, step 1 is restored
    with open(tmp_path / file_name(2, 2, 1), "r+b") as f:
        f.truncate(os.path.getsize(tmp_path / file_name(2, 2, 1)) - 16)
    assert read_header(str(tmp_path / file_name(2, 2, 1))) is None
    assert newest_complete_step(scan(str(tmp_path)), NUMEL) == 1
    # a bad header on a step-1 file: nothing is complete
    raw = bytearray((tmp_path / file_name(1, 2, 0)).read_bytes())
    raw[20] ^= 0xFF
    (tmp_path / file_name(1, 2, 0)).write_bytes(bytes(raw))
    assert newest_complete_step(scan(str(tmp_path)), NUMEL) is None
    (tmp_path / file_name(1, 2, 0)).write_bytes(b"TFTZ1CKP" + b"\xff" * 8)
    assert read_header(str(tmp_path / file_name(1, 2, 0))) is None
    # another format version is skipped
    hv = _header(3, 1, 0, [(0, NUMEL, 0)])
    hv["version"] = 99
    _write(tmp_path / file_name(3, 1, 0), hv, NUMEL)
    assert read_header(str(tmp_path / file_name(3, 1, 0))) is None
    # another model or unit split refuses
    hs = scan(str(tmp_path))
    check_compatible(hs, NUMEL, UNITS)
    with pytest.raises(ValueError, match="numel"):
        check_compatible(hs, NUMEL + 8, UNITS)
    with pytest.raises(ValueError, match="units"):
        check_compatible(hs, NUMEL, ((0, NUMEL),))
    assert json.loads(encode_header({"a": 1})[16:].rstrip(b"\0")) == {"a": 1}
