"""The heal copy's table (``p2p_transport.copy_table``) and the CPU model of ``heal_copy_kernel`` (``tests/_heal_ref.py``)
on hand-computed cases: every destination byte of every entry is stored exactly once, and no other byte is stored."""

from collections import Counter

import numpy as np
import pytest

from _heal_ref import THREADS, UNROLL, VEC, chunk_paths, chunks, find_entry, path_report, replay, vector_split
from torchft_b200.checkpointing.p2p_transport import copy_table

SRC, DST = 0x10000, 0x800000  # 16-byte aligned bases of two fake regions


def _memory(src_bytes, dst_bytes, seed=0):
    rng = np.random.default_rng(seed)
    return {SRC: rng.integers(0, 256, src_bytes, dtype=np.uint8), DST: rng.integers(0, 256, dst_bytes, dtype=np.uint8)}


def _check(entries, chunk_bytes, mem):
    """Replay ``entries`` and check the result byte for byte against plain slicing; returns the path report."""
    rows, total = copy_table(entries, chunk_bytes)
    want = {b: m.copy() for b, m in mem.items()}
    for s, d, n in entries:
        if n > 0:
            want[DST][d - DST:d - DST + n] = mem[SRC][s - SRC:s - SRC + n]
    inside = np.zeros(mem[DST].size, dtype=bool)
    for _, d, n in entries:
        inside[d - DST:d - DST + max(n, 0)] = True
    stores, report = replay(rows, total, chunk_bytes, mem)
    assert (stores[SRC] == 0).all(), "a source byte was stored"
    assert (stores[DST][inside] == 1).all(), "a destination byte was stored never or twice"
    assert (stores[DST][~inside] == 0).all(), "a byte outside the entries was stored"
    for b in mem:
        assert np.array_equal(mem[b], want[b])
    assert sum(report.values()) == sum(max(n, 0) for _, _, n in entries)
    return rows, total, report


def test_copy_table_hand_computed():
    rows, total = copy_table([(1, 2, 10), (3, 4, 0), (5, 6, 4096), (7, 8, 4097), (9, 10, -3), (11, 12, 1)], 4096)
    assert rows == [(1, 2, 10, 0), (5, 6, 4096, 1), (7, 8, 4097, 2), (11, 12, 1, 4)]
    assert total == 5
    assert copy_table([(1, 2, 0)], 16) == ([], 0)
    assert copy_table([], 16) == ([], 0)
    assert [find_entry(rows, c) for c in range(total)] == [0, 1, 2, 2, 3]
    assert [(c.entry, c.start, c.end) for c in chunks(rows, total, 4096)] == \
        [(0, 0, 10), (1, 0, 4096), (2, 0, 4096), (2, 4096, 4097), (3, 0, 1)]


def test_one_byte_entries():
    mem = _memory(8192, 4096)
    entries = [(SRC + 17 * i, DST + 3 * i, 1) for i in range(300)]
    rows, total, report = _check(entries, 16, mem)
    aligned = sum((17 * i) % 16 == 0 and (3 * i) % 16 == 0 for i in range(300))  # i = 0, 16, ..., 288: the byte tail
    assert aligned == 19 and total == 300 and report == Counter(bytes=300 - aligned, tail=aligned)


@pytest.mark.parametrize("chunk", [16, 4096, 1 << 16, (1 << 16) + 8])
def test_one_chunk_and_one_chunk_plus_a_byte(chunk):
    mem = _memory(4 * chunk + 64, 4 * chunk + 64)
    entries = [(SRC, DST, chunk), (SRC + chunk + 16 + (chunk % 16), DST + chunk + 48 + (chunk % 16), chunk + 1)]
    rows, total, report = _check(entries, chunk, mem)
    assert [r[3] for r in rows] == [0, 1] and total == 3
    spans = [(c.entry, c.start, c.end) for c in chunks(rows, total, chunk)]
    assert spans == [(0, 0, chunk), (1, 0, chunk), (1, chunk, chunk + 1)]
    if chunk == 1 << 16:  # 4096 vectors: one unrolled pass of 512 threads x 8, then one tail byte
        assert report == Counter(unrolled=2 * chunk, tail=1)


def test_only_the_last_entry_is_not_empty():
    mem = _memory(8192, 8192)
    entries = [(SRC + i, DST + i, 0) for i in range(50)] + [(SRC + 32, DST + 64, 5000)]
    rows, total, report = _check(entries, 1024, mem)
    assert rows == [(SRC + 32, DST + 64, 5000, 0)] and total == 5
    assert report == Counter(vec16=4992, tail=8)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_tables_of_thousands_of_entries(seed):
    rng = np.random.default_rng(100 + seed)
    n = 3000
    lens = rng.integers(0, 200, n)
    lens[rng.random(n) < 0.1] = 0
    lens[rng.random(n) < 0.02] = rng.integers(1000, 5000)
    soffs = rng.integers(0, 1 << 20, n)
    # destinations packed back to back, so neighbours share 16-byte vectors
    doffs = np.concatenate([[0], np.cumsum(lens)[:-1]]) + rng.integers(0, 16)
    mem = _memory(int(soffs.max() + lens.max()) + 16, int(doffs[-1] + lens[-1]) + 32, seed)
    entries = [(SRC + int(s), DST + int(d), int(k)) for s, d, k in zip(soffs, doffs, lens)]
    chunk = int(rng.choice([16, 48, 4096]))
    rows, total, _ = _check(entries, chunk, mem)
    assert len(rows) == int((lens > 0).sum()) and total == int(((lens + chunk - 1) // chunk).sum())


@pytest.mark.parametrize("nv", [0, 1, 511, 3584, 3585, 4095, 4096, 4097, 8191, 8192, 65536, 65537, 100_003])
def test_vector_split_partitions_the_vectors(nv):
    un, rem = vector_split(nv)
    assert np.array_equal(np.sort(np.concatenate([un, rem])), np.arange(nv))
    # a thread's unrolled iteration stores vectors t + 512 u, u < 8, and only runs while all 8 are below nv
    assert (un.size == 0) == (nv <= (UNROLL - 1) * THREADS)
    assert un.size % UNROLL == 0
    assert chunk_paths(0, 0, nv * VEC + 3) == +Counter(unrolled=un.size * VEC, vec16=rem.size * VEC, tail=3)


def test_chunk_paths():
    assert chunk_paths(16, 32, 17) == Counter(vec16=16, tail=1)
    assert chunk_paths(16, 33, 17) == Counter(bytes=17)
    assert chunk_paths(8, 8, 64) == Counter(bytes=64)
    assert chunk_paths(0, 0, 65536) == Counter(unrolled=65536)
    assert chunk_paths(0, 0, 65537) == Counter(unrolled=65536, tail=1)
    assert chunk_paths(0, 0, 65536 + 16) == Counter(unrolled=65536, vec16=16)


def test_a_chunk_size_off_the_vector_grid_alternates_paths():
    # chunks of 1 MiB + 8: chunk 1 starts 8 bytes off alignment and is copied byte by byte, chunk 2 is aligned again
    chunk = (1 << 20) + 8
    rows, total = copy_table([(0, 1 << 30, 3 * chunk)], chunk)
    paths = [set(chunk_paths(c.src, c.dst, c.end - c.start)) for c in chunks(rows, total, chunk)]
    assert paths == [{"unrolled", "tail"}, {"bytes"}, {"unrolled", "tail"}]
    assert sum(path_report(rows, total, chunk).values()) == 3 * chunk


def test_raw_table_contract_an_empty_row_hides_the_row_before_it():
    """What ``copy_table`` protects against: handed to the kernel directly, an empty row with the ``chunk0`` of the
    non-empty row before it takes that row's first chunk, which is then never copied."""
    mem = _memory(256, 256)
    want = mem[DST].copy()
    rows = [(SRC, DST, 100, 0), (SRC + 128, DST + 128, 0, 0)]
    assert [c.entry for c in chunks(rows, 1, 4096)] == [1]
    stores, report = replay(rows, 1, 4096, mem)
    assert (stores[DST] == 0).all() and np.array_equal(mem[DST], want) and not report
    rows, total = copy_table([(SRC, DST, 100), (SRC + 128, DST + 128, 0)], 4096)
    assert rows == [(SRC, DST, 100, 0)] and total == 1

