"""FT-ZeRO-1 replica audit on the CPU: the numpy digest (the device's specification) and the host policy that turns a
report into the ranges each rank stops claiming, checked against independent oracles."""

from __future__ import annotations

import random

import numpy as np
import pytest

from torchft_b200.parallel.zero1 import (AUDIT_ARRAYS, AUDIT_SEEDS, ShardLayout, audit_every_value, audit_findings,
                                         audit_stride, decode_audit_report, merge_ranges, plan_quorum, subtract_ranges,
                                         z1_digest)

M64 = (1 << 64) - 1


def fmix64_py(x):
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    return x ^ (x >> 33)


def digest_py(data, word0, seed):
    """The digest in Python integers, word by word."""
    b = np.ascontiguousarray(data).view(np.uint8).tobytes()
    s = 0
    for n in range(len(b) // 8):
        w = int.from_bytes(b[8 * n:8 * n + 8], "little")
        s = (s + fmix64_py(w ^ (((word0 + n) * 0x9E3779B97F4A7C15 + seed) & M64))) & M64
    return s


@pytest.mark.parametrize("dtype", [np.float32, np.uint16])
def test_digest_matches_integer_definition(dtype):
    rng = np.random.default_rng(0)
    x = rng.integers(0, 1 << 16, size=200).astype(dtype) if dtype == np.uint16 else rng.standard_normal(100).astype(dtype)
    for word0, seed in ((0, 0), (12345, AUDIT_SEEDS["master"]), ((1 << 40) + 2, AUDIT_SEEDS["weights"])):
        assert z1_digest(x, word0, seed) == digest_py(x, word0, seed)


def test_digest_independent_of_order_and_chunking():
    rng = np.random.default_rng(1)
    x = rng.standard_normal(4096).astype(np.float32)
    words = x.view(np.uint64)
    seed, word0 = AUDIT_SEEDS["v"], 777 * 2
    whole = z1_digest(x, word0, seed)
    for _ in range(20):
        cuts = sorted(rng.choice(np.arange(1, words.size), size=rng.integers(1, 30), replace=False).tolist())
        pieces = list(zip([0] + cuts, cuts + [words.size]))
        rng.shuffle(pieces)
        assert sum(z1_digest(words[a:b], word0 + a, seed) for a, b in pieces) & M64 == whole


def test_every_single_word_change_is_detected():
    rng = np.random.default_rng(2)
    x = rng.integers(0, 1 << 63, size=512, dtype=np.uint64)
    seed = AUDIT_SEEDS["m"]
    base = z1_digest(x, 64, seed)
    for i in range(x.size):
        for bit in (0, int(rng.integers(1, 63)), 63):
            y = x.copy()
            y[i] ^= np.uint64(1 << bit)
            assert z1_digest(y, 64, seed) != base, (i, bit)
        y = x.copy()
        y[i] = rng.integers(0, 1 << 63, dtype=np.uint64)
        assert y[i] == x[i] or z1_digest(y, 64, seed) != base


def test_position_and_seed_matter():
    x = np.arange(16, dtype=np.uint64)
    assert z1_digest(x, 0, 1) != z1_digest(x, 2, 1)
    assert z1_digest(x, 0, AUDIT_SEEDS["m"]) != z1_digest(x, 0, AUDIT_SEEDS["v"])
    assert len(set(AUDIT_SEEDS.values())) == len(AUDIT_SEEDS)
    assert z1_digest(np.zeros(0, np.uint64), 5, 1) == 0


@pytest.mark.parametrize("es,shift", [(4, 3), (2, 3), (4, 6), (2, 8)])
def test_flat_equals_paged(es, shift):
    """A range read page by page out of a pool in random slot order, each page digested at its global word index."""
    rng = np.random.default_rng(3)
    page = 1 << shift
    npages = 24
    flat = rng.integers(0, 256, size=npages * page * es, dtype=np.uint8)
    slots = rng.permutation(npages)
    pool = np.zeros_like(flat)
    pb = page * es
    for p, s in enumerate(slots):
        pool[s * pb:(s + 1) * pb] = flat[p * pb:(p + 1) * pb]
    lo, hi = 3 * page + 8, 19 * page - 16  # element range, multiples of 8
    want = z1_digest(flat[lo * es:hi * es], lo * es // 8, AUDIT_SEEDS["ema"])
    got = 0
    e = lo
    while e < hi:
        end = min(hi, (e // page + 1) * page)
        s = slots[e // page]
        at = (s * page + e % page) * es
        got += z1_digest(pool[at:at + (end - e) * es], e * es // 8, AUDIT_SEEDS["ema"])
        e = end
    assert got & M64 == want


def test_audit_every_value(monkeypatch):
    monkeypatch.delenv("TORCHFT_B200_Z1_AUDIT_EVERY", raising=False)
    assert audit_every_value(None) == 0
    assert audit_every_value(5) == 5
    monkeypatch.setenv("TORCHFT_B200_Z1_AUDIT_EVERY", "100")
    assert audit_every_value(None) == 100
    assert audit_every_value(0) == 0
    with pytest.raises(ValueError):
        audit_every_value(-1)
    assert audit_stride(2) == 1 + 2 * len(AUDIT_ARRAYS)


# --------------------------------------------------------------------------- reports and findings
UNITS = ((0, 8 * 100), (8 * 100, 8 * 100 + 8 * 37))


def clean_report(world, k, narrays=3, t=7, units=UNITS):
    """A report in which every rank at ``t`` agrees: weights digest ``1000 + u``, state digest of slice ``s``'s array
    ``a`` ``hash((u, s, a))``."""
    L = ShardLayout(units, k)
    kk = L.k(world)
    rep = {"seq": 1, "mismatches": 0, "world": world, "t": [t] * world,
           "weights": [[1000 + u for u in range(len(units))] for _ in range(world)], "state": []}
    for r in range(world):
        rep["state"].append([[[(u * 131 + ((r - j) % world) * 17 + a) * 7919 + 1 for a in range(narrays)]
                              for j in range(kk)] for u in range(len(units))])
    return L, rep


def corrupt(rep, r, u, j, a):
    rep["state"][r][u][j][a] ^= 0xBAD


def test_clean_report_finds_nothing():
    for world in range(1, 9):
        for k in (1, 2, 3):
            L, rep = clean_report(world, k)
            findings, drops = audit_findings(rep, L, world)
            assert findings == [] and all(not d for d in drops.values())


def test_weights_mismatch_drops_nothing():
    L, rep = clean_report(4, 2)
    rep["weights"][2][1] += 1
    findings, drops = audit_findings(rep, L, 4)
    assert findings == [{"unit": 1, "array": "weights", "slice": None, "ranks": [2], "t": 7}]
    assert all(not d for d in drops.values())


def test_k3_one_odd_holder_drops_alone():
    world = 5
    L, rep = clean_report(world, 3)
    s, u, a = 1, 0, 2
    h = (s + 2) % world  # the second buddy of slice 1 holds it as its j = 2 slice
    corrupt(rep, h, u, 2, a)
    findings, drops = audit_findings(rep, L, world)
    assert findings == [{"unit": u, "array": AUDIT_ARRAYS[a], "slice": s, "ranks": [h], "t": 7}]
    assert drops[h] == [L.slice_bounds(u, world, s)]
    assert all(not drops[r] for r in range(world) if r != h)


def test_k2_disagreement_drops_both_and_plan_reseeds():
    world = 4
    L, rep = clean_report(world, 2)
    s, u = 3, 1
    corrupt(rep, (s + 1) % world, u, 1, 0)  # the buddy's master differs from the primary's
    findings, drops = audit_findings(rep, L, world)
    assert len(findings) == 1 and findings[0]["ranks"] == sorted([s, (s + 1) % world])
    bounds = L.slice_bounds(u, world, s)
    published = {}
    for r in range(world):
        assert drops[r] == ([bounds] if r in (s, (s + 1) % world) else [])
        published[r] = {"t": 7, "hold": subtract_ranges(L.held(r, world), drops[r])}
    plans = plan_quorum(L, world, published)
    for r in range(world):
        assert plans[r].pulls == [] or all(not (lo < bounds[1] and bounds[0] < hi) for _, lo, hi in plans[r].pulls)
        assert plans[r].lost == drops[r] and plans[r].counted
    assert sum(hi - lo for r in range(world) for lo, hi in plans[r].lost) == 2 * (bounds[1] - bounds[0])


def test_ranks_behind_are_ignored():
    world = 4
    L, rep = clean_report(world, 3)
    rep["t"][2] = 6  # a split commit left rank 2 one update behind
    rep["weights"][2][0] += 5
    corrupt(rep, 2, 0, 0, 1)
    findings, drops = audit_findings(rep, L, world)
    assert findings == [] and all(not d for d in drops.values())


def test_compact_plan_takes_the_slice_from_the_majority():
    """Paged state: a holder whose ``hold`` claims less than its pages back re-pulls the dropped slice into its own page."""
    world, shift = 3, 4
    units = ((0, 8 * 64),)
    L, rep = clean_report(world, 3, units=units)
    corrupt(rep, 1, 0, 0, 1)  # rank 1's own primary slice of m differs from its two buddies'
    _, drops = audit_findings(rep, L, world)
    assert drops[1] == [L.slice_bounds(0, world, 1)] and not drops[0] and not drops[2]
    from torchft_b200.parallel.zero1 import page_ranges

    published = {}
    for r in range(world):
        pages = page_ranges(L.held(r, world), shift)
        published[r] = {"t": 7, "hold": subtract_ranges(L.held(r, world), drops[r]),
                        "pages": [(lo, lo, hi - lo) for lo, hi in pages]}
    plans = plan_quorum(L, world, published, shift)
    p = plans[1]
    assert p.need == drops[1] and p.lost == [] and p.allocate == [] and p.free_first == []
    assert merge_ranges([(lo, hi) for _, lo, hi in p.pulls]) == drops[1]
    assert all(src != 1 for src, _, _ in p.pulls)
    assert p.hold == L.held(1, world)
    assert all(plans[r].need == [] for r in (0, 2))


def test_decode_report_roundtrip():
    world, k, narrays, nunits = 3, 2, 4, 2
    stride = audit_stride(k)
    n = nunits * stride + 1
    slots = np.zeros((world, n), dtype=np.uint64)
    for r in range(world):
        for u in range(nunits):
            slots[r, u * stride] = 10 * r + u
            for j in range(k):
                for a in range(narrays):
                    slots[r, u * stride + 1 + j * narrays + a] = 1000 * r + 100 * u + 10 * j + a
        slots[r, -1] = 40 + r
    raw = np.concatenate([np.array([9, 2, world, n], dtype=np.uint64), slots.ravel()]).tobytes()
    rep = decode_audit_report(raw, nunits, stride, narrays, k)
    assert rep["seq"] == 9 and rep["mismatches"] == 2 and rep["t"] == [40, 41, 42]
    assert rep["weights"][2][1] == 21 and rep["state"][1][0][1][3] == 1013
    assert decode_audit_report(bytes(8 * (4 + world * n)), nunits, stride, narrays, k)["t"] == []


def bitmap_oracle(rep, L, world, numel):
    """Per element and rank: does the rank stop claiming it? Decided element by element from the holders' digests of
    the slice the element is in."""
    t = rep["t"]
    tmax = max(t)
    drop = np.zeros((world, numel), dtype=bool)
    k = L.k(world)
    if k < 2:
        return drop
    for u in range(len(L.units)):
        for s in range(world):
            lo, hi = L.slice_bounds(u, world, s)
            holders = [(s + j) % world for j in range(k) if t[(s + j) % world] == tmax]
            for a in range(len(rep["state"][0][0][0])):
                vals = [rep["state"][h][u][(h - s) % world][a] for h in holders]
                for h, val in zip(holders, vals):
                    agree = sum(v == val for v in vals)
                    best = max(sum(v == w for v in vals) for w in vals)
                    no_majority = 2 * best <= len(vals)
                    if len(set(vals)) > 1 and (no_majority or 2 * agree <= len(vals)):
                        drop[h, lo:hi] = True
    return drop


def test_random_walk_against_bitmap_oracle():
    """Quorums that lose and gain members, split commits that leave ranks behind, and divergences in random holders
    and arrays: the ranges each rank drops are exactly the oracle's, and the next re-shard never takes a dropped range
    from a rank that dropped it, and re-seeds exactly what every current holder dropped."""
    rng = random.Random(4)
    units = ((0, 8 * 40), (8 * 40, 8 * 40 + 8 * 23), (8 * 63, 8 * 64))
    numel = units[-1][1]
    for step in range(300):
        world = rng.randint(1, 8)
        k = rng.randint(1, 4)
        narrays = rng.choice((3, 4))
        L, rep = clean_report(world, k, narrays, t=rng.randint(1, 9), units=units)
        for r in range(world):
            if rng.random() < 0.2:
                rep["t"][r] -= 1  # behind: left out, and holds nothing at tmax
        if max(rep["t"]) != rep["t"][0] and all(x != max(rep["t"]) for x in rep["t"]):
            continue
        for _ in range(rng.randint(0, 4)):
            r, u = rng.randrange(world), rng.randrange(len(units))
            if L.k(world) > 1:
                corrupt(rep, r, u, rng.randrange(L.k(world)), rng.randrange(narrays))
            if rng.random() < 0.3:
                rep["weights"][r][u] ^= 1
        findings, drops = audit_findings(rep, L, world)
        oracle = bitmap_oracle(rep, L, world, numel)
        for r in range(world):
            got = np.zeros(numel, dtype=bool)
            for lo, hi in drops[r]:
                got[lo:hi] = True
            assert np.array_equal(got, oracle[r]), (step, r)
        # the same members form the next quorum
        tmax = max(rep["t"])
        published = {r: {"t": rep["t"][r], "hold": subtract_ranges(L.held(r, world), drops[r])} for r in range(world)}
        plans = plan_quorum(L, world, published)
        claimed = np.zeros((world, numel), dtype=bool)
        for r in range(world):
            if rep["t"][r] == tmax:
                for lo, hi in published[r]["hold"]:
                    claimed[r, lo:hi] = True
        for r, p in plans.items():
            for src, lo, hi in p.pulls:
                assert claimed[src, lo:hi].all() and not oracle[src, lo:hi].any()
            for lo, hi in p.lost:
                assert not claimed[:, lo:hi].any()


def test_zeroed_rows_only_add_drops():
    """A report in which some ranks' rows were zeroed (their next audit's memset ran before this rank's compare): every
    rank whose row is intact drops at least the ranges the complete report makes it drop."""
    rng = random.Random(5)
    units = ((0, 8 * 40), (8 * 40, 8 * 40 + 8 * 23))
    tied = 0
    for _ in range(400):
        world = rng.randint(2, 8)
        k = rng.randint(2, 4)
        L, rep = clean_report(world, k, 3, units=units)
        for _ in range(rng.randint(1, 4)):
            corrupt(rep, rng.randrange(world), rng.randrange(len(units)), rng.randrange(L.k(world)), rng.randrange(3))
        _, want = audit_findings(rep, L, world)
        zeroed = rng.sample(range(world), rng.randint(1, world - 1))
        for r in zeroed:
            rep["t"][r] = 0
            rep["weights"][r] = [0] * len(units)
            rep["state"][r] = [[[0] * 3 for _ in range(L.k(world))] for _ in units]
        _, got = audit_findings(rep, L, world)
        for r in range(world):
            if r not in zeroed:
                assert subtract_ranges(want[r], got[r]) == [], (world, k, r, want[r], got[r])
        tied += any(got[r] != want[r] for r in range(world) if r not in zeroed)
    assert tied  # the zeroed rows did make some ranks drop more


def test_a_zeroed_row_does_not_turn_a_tie_into_a_majority():
    world = 4
    L, rep = clean_report(world, 4)
    s, u = 0, 0
    corrupt(rep, 2, u, 2, 0)  # holders 0..3 of slice 0 hold x, x, y, y for the master
    corrupt(rep, 3, u, 3, 0)
    rep["state"][3][u][3][0] = rep["state"][2][u][2][0]
    _, want = audit_findings(rep, L, world)
    assert all(want[r] == [L.slice_bounds(u, world, s)] for r in range(world))
    rep["t"][3] = 0
    rep["weights"][3] = [0, 0]
    _, got = audit_findings(rep, L, world)
    assert all(got[r] == want[r] for r in range(3))


def test_seed_source_is_the_lowest_rank_at_tmax():
    from torchft_b200.parallel.zero1 import audit_seed_source

    assert audit_seed_source({0: {"t": 3}, 1: {"t": 5}, 2: {"t": 5}}) == 1  # rank 0 is a joiner being healed
    assert audit_seed_source({0: {"t": 5}, 1: {"t": 5}}) == 0
