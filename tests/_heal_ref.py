"""A CPU model of ``heal_copy_kernel`` (``model_ops.cu``): which entry each chunk belongs to, the byte range it covers,
and which of the kernel's four copy paths moves each of its bytes.

The kernel runs ``THREADS`` threads per CTA over the chunks of a table built by ``p2p_transport.copy_table``. A chunk whose
source and destination are both 16-byte aligned is moved by an ``UNROLL``-way unrolled loop of 16-byte vectors, then a
16-byte remainder loop, then a byte tail; any other chunk is moved byte by byte. :func:`replay` performs the copy the
same way on host memory and counts every byte it stores."""

from __future__ import annotations

from collections import Counter
from typing import Dict, Iterator, List, NamedTuple, Sequence, Tuple

import numpy as np

THREADS = 512
UNROLL = 8
VEC = 16
PATHS = ("unrolled", "vec16", "tail", "bytes")  # 8 x 16 B loop, 16 B remainder loop, byte tail, byte-only path


class Chunk(NamedTuple):
    c: int       # chunk index
    entry: int   # table row it belongs to
    start: int   # byte range [start, end) of that row
    end: int
    src: int     # addresses of byte `start`
    dst: int


def find_entry(rows: Sequence[Tuple[int, int, int, int]], c: int) -> int:
    """The kernel's binary search: the last row whose ``chunk0`` is not above ``c``."""
    lo, hi = 0, len(rows) - 1
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if rows[mid][3] <= c:
            lo = mid
        else:
            hi = mid - 1
    return lo


def chunks(rows: Sequence[Tuple[int, int, int, int]], total_chunks: int, chunk_bytes: int) -> Iterator[Chunk]:
    """Every chunk the kernel copies, in index order (the grid-stride loop visits each exactly once)."""
    for c in range(total_chunks):
        i = find_entry(rows, c)
        src, dst, n, chunk0 = rows[i]
        start = (c - chunk0) * chunk_bytes
        end = min(start + chunk_bytes, n)
        yield Chunk(c, i, start, end, src + start, dst + start)


def vector_split(nv: int) -> Tuple[np.ndarray, np.ndarray]:
    """For an aligned chunk of ``nv`` whole vectors: the vectors the unrolled loop stores and those the remainder loop
    stores. Thread ``t`` owns vectors ``t + THREADS * j``; it runs ``K_t`` unrolled iterations (``j < K_t * UNROLL``), as
    many as keep its last vector of the iteration below ``nv``."""
    i = np.arange(nv, dtype=np.int64)
    t, j = i % THREADS, i // THREADS
    span = nv - (UNROLL - 1) * THREADS - t
    k = np.where(span > 0, (span + UNROLL * THREADS - 1) // (UNROLL * THREADS), 0)
    unrolled = j < k * UNROLL
    return i[unrolled], i[~unrolled]


def unrolled_vectors(nv: int) -> int:
    """How many of ``nv`` vectors the unrolled loop stores (the count of :func:`vector_split`, in closed form)."""
    if nv <= (UNROLL - 1) * THREADS:
        return 0
    t = np.arange(THREADS, dtype=np.int64)
    span = nv - (UNROLL - 1) * THREADS - t
    return int(np.where(span > 0, (span + UNROLL * THREADS - 1) // (UNROLL * THREADS), 0).sum()) * UNROLL


def chunk_paths(src: int, dst: int, length: int) -> Counter:
    """Bytes of one chunk moved by each path."""
    out: Counter = Counter()
    if (src | dst) % VEC:
        out["bytes"] = length
        return out
    nv = length // VEC
    u = unrolled_vectors(nv)
    out["unrolled"], out["vec16"], out["tail"] = u * VEC, (nv - u) * VEC, length - nv * VEC
    return +out


def path_report(rows, total_chunks: int, chunk_bytes: int) -> Counter:
    """Bytes moved by each path over the whole table."""
    out: Counter = Counter()
    for ch in chunks(rows, total_chunks, chunk_bytes):
        out.update(chunk_paths(ch.src, ch.dst, ch.end - ch.start))
    return out


def _region(memory: Dict[int, np.ndarray], addr: int, n: int) -> Tuple[int, np.ndarray]:
    for base, buf in memory.items():
        if base <= addr and addr + n <= base + buf.size:
            return base, buf
    raise AssertionError(f"[{addr:#x}, {addr + n:#x}) lies in no region")


def replay(rows, total_chunks: int, chunk_bytes: int, memory: Dict[int, np.ndarray]) -> Tuple[Dict[int, np.ndarray], Counter]:
    """Run the kernel on host ``memory`` (region base address -> uint8 array, written in place). Returns the number of
    stores per byte of every region and the bytes each path moved. Reads see the memory as it was before the launch."""
    before = {b: m.copy() for b, m in memory.items()}
    stores = {b: np.zeros(m.size, dtype=np.int32) for b, m in memory.items()}
    report: Counter = Counter()
    for ch in chunks(rows, total_chunks, chunk_bytes):
        n = ch.end - ch.start
        if n <= 0:
            continue
        sb, _ = _region(memory, ch.src, n)
        db, dbuf = _region(memory, ch.dst, n)
        s0, d0 = ch.src - sb, ch.dst - db
        src = before[sb][s0:s0 + n]
        parts: List[np.ndarray] = []
        paths = chunk_paths(ch.src, ch.dst, n)
        report.update(paths)
        if "bytes" in paths:
            parts.append(np.arange(n, dtype=np.int64))
        else:
            nv = n // VEC
            lanes = np.arange(VEC, dtype=np.int64)
            for vecs in vector_split(nv):
                parts.append((vecs[:, None] * VEC + lanes).ravel())
            parts.append(np.arange(nv * VEC, n, dtype=np.int64))
        for k in parts:
            dbuf[d0 + k] = src[k]
            stores[db][d0 + k] += 1
    return stores, report

