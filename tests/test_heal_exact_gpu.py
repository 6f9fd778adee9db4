"""The heal copy byte for byte: ``heal_copy_kernel`` against the CPU model of ``tests/_heal_ref.py`` at every alignment,
length, chunk size and grid; ``P2PTransport`` across processes (on two GPUs when there are two); and the FT-ZeRO-1
re-shard pulls against the state before each quorum change.

Destinations are carved from larger buffers pre-filled with random bytes, and comparisons are of bytes (``uint8``), never
of values: the data holds NaN payloads and -0.0."""

from __future__ import annotations

import json
import os
import select
import subprocess
import sys
import tempfile
from collections import Counter
from datetime import timedelta

import numpy as np
import pytest
import torch

from _heal_ref import PATHS, THREADS, UNROLL, VEC, chunks, path_report

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHUNKS = (16, 4 << 10, 1 << 20, 4 << 20, (1 << 20) + 8)  # the last is off the 16-byte grid
GRIDS = (1, 3, 128, 1024)
OFFSETS = (0, 1, 2, 4, 8, 15)
GAP = 64  # random bytes around every destination


@pytest.fixture(scope="module")
def K():
    from torchft_b200.ops import _native

    return _native.load()


def _lengths(chunk):
    return (1, 15, 16, 17, 65535, 65536, 65537, chunk - 1, chunk, chunk + 1, 3 * chunk + 5)


def _round(x, a=256):
    return (x + a - 1) // a * a


def alignment_case(chunk):
    """``(src_off, dst_off, n)`` relative to two 256-byte aligned buffers, and the buffer sizes: every src x dst offset of
    ``OFFSETS`` at every length of :func:`_lengths`, each destination with ``GAP`` random bytes on both sides."""
    rel, s_at, d_at = [], 0, 0
    for so in OFFSETS:
        for do in OFFSETS:
            for n in _lengths(chunk):
                rel.append((s_at + so, d_at + GAP + do, n))
                s_at = _round(s_at + so + n)
                d_at = _round(d_at + GAP + do + n + GAP)
    return rel, s_at, d_at


def packed_case(chunk, seed=5, n=2000):
    """About ``n`` entries of random length and source offset, packed back to back into one destination (neighbours share
    16-byte vectors); a few are longer than a chunk, a few are empty."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 3000, n)
    lens[rng.random(n) < 0.03] = 0
    big = rng.random(n) < 0.02
    lens[big] = rng.integers(60_000, 3 * min(chunk, 1 << 20) + 100_000, int(big.sum()))
    lens[rng.random(n) < 0.05] = 16 * rng.integers(1, 200)  # whole vectors ...
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]) + GAP
    src_size = 8 << 20
    soffs = rng.integers(0, src_size - int(lens.max()), n)
    soffs[rng.random(n) < 0.3] &= ~15  # ... and aligned sources, so some neighbours land on the vector paths
    rel = [(int(s), int(d), int(k)) for s, d, k in zip(soffs, starts, lens)]
    return rel, src_size, _round(int(starts[-1] + lens[-1]) + GAP)


def _fill(nbytes, seed):
    """Seeded random bytes on the device, with NaN payloads and -0.0 planted at fp32 and bf16 alignment."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = torch.randint(0, 256, (max(nbytes, 16),), dtype=torch.uint8, device="cuda", generator=g)
    w = b[: b.numel() // 4 * 4].view(torch.int32)
    w[::97] = 0x7FA00001              # signalling NaN with a payload
    w[1::89] = -(1 << 31)             # -0.0
    b[: b.numel() // 2 * 2].view(torch.int16)[5::83] = 0x7FC1  # bf16 NaN with a payload
    return b


def _copy_and_check(rel, src_size, dst_size, chunk, grids, seed):
    """Copy ``rel`` with every grid of ``grids``; the result must be the destination buffer as it was with each entry's
    source bytes sliced into place (independently of the kernel's table), and the source must be unchanged. Returns the
    CPU model's path report."""
    from torchft_b200.checkpointing.p2p_transport import copy_table, device_copy

    src = _fill(src_size, seed)
    assert src.data_ptr() % 256 == 0
    src0 = src.cpu().numpy()
    dst0 = _fill(dst_size, seed + 1).cpu().numpy()
    want = dst0.copy()
    for s, d, n in rel:
        want[d:d + n] = src0[s:s + n]
    report = None
    for blocks in grids:
        dst = torch.from_numpy(dst0).cuda()
        assert dst.data_ptr() % 256 == 0
        entries = [(src.data_ptr() + s, dst.data_ptr() + d, n) for s, d, n in rel]
        device_copy(entries, blocks=blocks, chunk_bytes=chunk)
        torch.cuda.synchronize()
        if report is None:
            report = path_report(*copy_table(entries, chunk), chunk)
        got = dst.cpu().numpy()
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (f"chunk {chunk}, {blocks} CTAs: {bad.size} bytes differ, first at destination offset "
                               f"{bad[0]} ({[(s, d, n) for s, d, n in rel if d <= bad[0] < d + n][:1] or 'outside every entry'})")
        del dst
    assert np.array_equal(src.cpu().numpy(), src0), "the copy wrote into its source"
    return report


@pytest.mark.parametrize("chunk", CHUNKS)
def test_every_alignment_and_length_at_every_grid(K, chunk):
    rel, src_size, dst_size = alignment_case(chunk)
    _copy_and_check(rel, src_size, dst_size, chunk, GRIDS, seed=10)


@pytest.mark.parametrize("chunk", CHUNKS)
def test_packed_table(K, chunk):
    rel, src_size, dst_size = packed_case(chunk)
    assert len(rel) == 2000
    _copy_and_check(rel, src_size, dst_size, chunk, (1, 128, 1024), seed=20)


def test_one_entry_larger_than_2_to_the_31_bytes(K):
    from torchft_b200.checkpointing.p2p_transport import CHUNK_BYTES, copy_table, device_copy

    n = (1 << 31) + 12345  # the last chunk is 771 vectors and a 9-byte tail
    free, _ = torch.cuda.mem_get_info()
    if free < 3 * n + (1 << 30):
        pytest.skip(f"needs {3 * n / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free")
    src = _fill(n, 30)
    keep = src.clone()
    dst = _fill(n + 2 * 4096, 31)
    edges = (dst[:4096].clone(), dst[4096 + n:].clone())
    entries = [(src.data_ptr(), dst.data_ptr() + 4096, n)]
    device_copy(entries)
    torch.cuda.synchronize()
    rows, total = copy_table(entries, CHUNK_BYTES)
    spans = [(c.start, c.end) for c in chunks(rows, total, CHUNK_BYTES)]
    assert spans[0] == (0, CHUNK_BYTES) and spans[-1] == ((total - 1) * CHUNK_BYTES, n) and total == 513
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert path_report(rows, total, CHUNK_BYTES) == Counter(unrolled=1 << 31, vec16=771 * 16, tail=9)
    assert torch.equal(dst[4096:4096 + n], src), "the entry's bytes"
    assert torch.equal(dst[:4096], edges[0]) and torch.equal(dst[4096 + n:], edges[1]), "bytes around the entry"
    assert torch.equal(src, keep), "the copy wrote into its source"


def test_every_kernel_path_at_every_chunk_size():
    """Which paths the cases above take, by the CPU model (buffers are 256-byte aligned, so their addresses are those
    offsets modulo 16). Chunks of fewer than 7 x 512 + 1 vectors can never enter the unrolled loop."""
    from torchft_b200.checkpointing.p2p_transport import copy_table

    for chunk in CHUNKS:
        took = Counter()
        for rel, _, _ in (alignment_case(chunk), packed_case(chunk)):
            entries = [(s, (1 << 40) + d, n) for s, d, n in rel]
            took.update(path_report(*copy_table(entries, chunk), chunk))
        print(f"chunk {chunk}: " + ", ".join(f"{p} {took[p]} B" for p in PATHS))
        reachable = set(PATHS) if chunk >= ((UNROLL - 1) * THREADS + 1) * VEC else set(PATHS) - {"unrolled"}
        assert {p for p in PATHS if took[p]} == reachable, (chunk, took)


def test_heal_copy(K):
    from torchft_b200.checkpointing.p2p_transport import device_copy

    torch.manual_seed(7)
    srcs = [torch.randn(n, device="cuda") for n in (1, 1000, 1 << 20, 12345)]
    srcs.append(torch.randint(0, 255, (777,), device="cuda", dtype=torch.uint8)[1:])  # unaligned
    dsts = [torch.empty_like(s) for s in srcs]
    device_copy([(s.data_ptr(), d.data_ptr(), s.numel() * s.element_size()) for s, d in zip(srcs, dsts)])
    torch.cuda.synchronize()
    for s, d in zip(srcs, dsts):
        assert torch.equal(s, d)


# ----------------------------------------------------------------------------- the heal across processes
def _bytes(t):
    return t.detach().contiguous().cpu().reshape(-1).view(torch.uint8)


class _Source:
    """``tests/_heal_source.py`` serving one seeded state; the worker is killed on exit if it has not finished."""

    def __init__(self, config, seed, env=None):
        self.device = 1 if torch.cuda.device_count() > 1 else 0
        self.err = tempfile.TemporaryFile()
        self.p = subprocess.Popen([sys.executable, os.path.join(HERE, "_heal_source.py"), "--config", config,
                                   "--seed", str(seed), "--device", str(self.device)],
                                  stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=self.err,
                                  env={**os.environ, **(env or {})})

    def served(self, timeout=300):
        ready, _, _ = select.select([self.p.stdout], [], [], timeout)
        line = self.p.stdout.readline() if ready else b""
        if not line:
            self.err.seek(0)
            raise AssertionError(f"the source printed nothing: {self.err.read().decode(errors='replace')[-3000:]}")
        return json.loads(line)

    def finish(self):
        self.p.stdin.write(b"done\n")
        self.p.stdin.flush()
        assert self.p.wait(timeout=60) == 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        if self.p.poll() is None:
            self.p.kill()
        self.p.wait()
        self.err.close()


def _sentinel_view(buf, at, shape, dtype):
    """A contiguous ``dtype`` tensor of ``shape`` inside uint8 ``buf`` at byte ``at``."""
    n = torch.Size(shape).numel() * torch.empty(0, dtype=dtype).element_size()
    return buf[at:at + n].view(dtype).view(shape)


def _receive_leaves(seed, env=None):
    from _heal_source import source_state

    from torchft_b200.checkpointing import P2PTransport

    want = source_state("leaves", seed, "cuda:0")
    # in-place targets: views inside a random sentinel buffer, at offsets that are not 16-byte aligned
    pool = _fill(1 << 20, seed + 100)
    pool0 = pool.clone()
    d = want["dtypes"]
    match = {"fp32": _sentinel_view(pool, 4100, (3, 5, 7), torch.float32),
             "bf16": _sentinel_view(pool, 9002, (3, 5, 7), torch.bfloat16),
             "u8": _sentinel_view(pool, 12001, (3, 5, 7), torch.uint8),
             "c64": _sentinel_view(pool, 16384, (3, 5, 7), torch.complex64),
             "transposed": _sentinel_view(pool, 20008, (41, 37), torch.float32),
             "odd": _sentinel_view(pool, 30002, (1, 13, 1), torch.int16)}
    wrong = {"dtype": _sentinel_view(pool, 40000, (3, 5, 7), torch.float32),        # int32 source
             "shape": _sentinel_view(pool, 50000, (5, 3, 7), torch.float64),        # (3, 5, 7) source
             "strided": _sentinel_view(pool, 60000, (7, 5, 3), torch.int64).permute(2, 1, 0)}
    assert not wrong["strided"].is_contiguous()
    host_target = torch.zeros(1024)
    targets = {"dtypes": {"float32": match["fp32"], "bfloat16": match["bf16"], "uint8": match["u8"],
                          "complex64": match["c64"], "int32": wrong["dtype"], "float64": wrong["shape"],
                          "int64": wrong["strided"]},
               "transposed": match["transposed"], "odd": match["odd"], "host": {"page": host_target}}
    outside = torch.ones(pool.numel(), dtype=torch.bool, device="cuda")
    for t in match.values():
        off = t.data_ptr() - pool.data_ptr()
        outside[off:off + t.numel() * t.element_size()] = False
    ptrs = {k: t.data_ptr() for k, t in match.items()}
    t = timedelta(seconds=60)
    with _Source("leaves", seed, env) as src:
        info = src.served()
        assert "error" not in info, info["error"]
        rx = P2PTransport(t, state_dict=lambda: targets)
        try:
            got = rx.recv_checkpoint(0, info["metadata"], info["step"], t)
            torch.cuda.synchronize()
        finally:
            rx.shutdown()
        src.finish()

    from torch.utils import _pytree as pytree

    flat_want, spec = pytree.tree_flatten(want)
    flat_got, spec_got = pytree.tree_flatten(got)
    assert spec == spec_got
    tensor_bytes = 0
    for (kp, w), g in zip(pytree.tree_flatten_with_path(want)[0], flat_got):
        name = pytree.keystr(kp)
        if isinstance(w, torch.Tensor):
            assert isinstance(g, torch.Tensor) and g.dtype == w.dtype and g.shape == w.shape, name
            assert g.is_cuda == w.is_cuda, name
            assert torch.equal(_bytes(g), _bytes(w)), name
            if w.is_cuda or w.numel() * w.element_size() >= 4096:
                tensor_bytes += w.numel() * w.element_size()
        else:
            assert g == w, name
    assert rx.last_recv_bytes == tensor_bytes
    # matching targets were written in place, the others were left alone and replaced by fresh tensors
    assert got["dtypes"]["float32"].data_ptr() == ptrs["fp32"] and got["dtypes"]["bfloat16"].data_ptr() == ptrs["bf16"]
    assert got["dtypes"]["uint8"].data_ptr() == ptrs["u8"] and got["dtypes"]["complex64"].data_ptr() == ptrs["c64"]
    assert got["transposed"].data_ptr() == ptrs["transposed"] and got["odd"].data_ptr() == ptrs["odd"]
    for key, tgt in (("int32", wrong["dtype"]), ("float64", wrong["shape"]), ("int64", wrong["strided"])):
        assert got["dtypes"][key].data_ptr() != tgt.data_ptr(), key
    assert torch.equal(pool[outside], pool0[outside]), "bytes around the in-place targets, or a refused target, changed"
    assert got["host"]["page"] is host_target
    assert not got["host"]["small_pinned"].is_cuda and not got["host"]["page_pinned"].is_cuda


def test_heal_across_processes_every_dtype_view_and_target(K):
    print(f"source on cuda:{1 if torch.cuda.device_count() > 1 else 0}, receiver on cuda:0")
    _receive_leaves(seed=1)


def test_heal_across_processes_with_expandable_segments(K):
    _receive_leaves(seed=2, env={"PYTORCH_CUDA_ALLOC_CONF": "expandable_segments:True"})


def test_heal_across_processes_of_the_zero1_payload_in_a_vmm_segment(K):
    from _heal_source import source_state

    from torchft_b200.checkpointing import P2PTransport

    want = source_state("zero1_vmm", 3, "cuda:0")
    param = _fill(want["param"].numel() * 2 + 32, 40)
    keep = param.clone()
    target = param[16:16 + want["param"].numel() * 2].view(torch.bfloat16)
    t = timedelta(seconds=60)
    with _Source("zero1_vmm", 3) as src:
        info = src.served()
        assert "error" not in info, info["error"]
        rx = P2PTransport(t, state_dict=lambda: {"param": target, "t": 0})
        try:
            got = rx.recv_checkpoint(0, info["metadata"], info["step"], t)
            torch.cuda.synchronize()
        finally:
            rx.shutdown()
        src.finish()
    assert got["t"] == 5 and got["param"].data_ptr() == target.data_ptr()
    assert torch.equal(_bytes(target), _bytes(want["param"]))
    assert torch.equal(param[:16], keep[:16]) and torch.equal(param[16 + target.numel() * 2:], keep[16 + target.numel() * 2:])
    assert rx.last_recv_bytes == target.numel() * 2


# ----------------------------------------------------------------------------- FT-ZeRO-1 re-shard pulls
def _state_bytes(reps):
    return [_bytes(x) for x in reps.full_state()] + [_bytes(reps.full_ema())]


@pytest.mark.parametrize("k,chain", [(2, (4, 3, 5, 8, 7, 6)), (3, (8, 6, 4, 7)), (1, (1, 2, 4, 8))])
@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("moments", ["fp32", "bf16"])
def test_reshard_pulls_keep_the_state_of_the_quorum_before(monkeypatch, k, chain, compact, moments):
    """Quorum changes in which every range keeps a live holder: after each, the state assembled from the new holders is
    the state of the old ones byte for byte (master, m, v and the EMA). Members that leave come back as fresh optimizers."""
    from _zero1_replicas import Replicas, raws

    from torchft_b200.parallel import zero1

    plans = []
    real = zero1.plan_quorum
    monkeypatch.setattr(zero1, "plan_quorum", lambda *a, **kw: plans.append(real(*a, **kw)) or plans[-1])
    md = torch.float32 if moments == "fp32" else torch.bfloat16
    reps = Replicas(max(chain), k=k, compact=compact, moment_dtype=md, ema_decay=0.9)
    members = list(range(chain[0]))
    reps.configure(members, 1)
    for epoch, size in enumerate(chain[1:], start=2):
        reps.step(raws(len(members), 100 + epoch))
        reps.settle()
        before = _state_bytes(reps)
        if size < len(members):
            assert len(members) - size < k, "a change that removes k holders can lose a range"
            drop = members[1::2][:len(members) - size]
            members = [m for m in members if m not in drop]
        else:
            for m in [m for m in range(max(chain)) if m not in members][:size - len(members)]:
                o = reps.make(reps.comms[m])  # a fresh process with the healed weights
                o.param.copy_(reps.opts[members[0]].param)
                o.seed_master()
                reps.opts[m] = o
                members.append(m)
        plans.clear()
        reps.configure(members, epoch)
        assert len(members) == size and plans
        for p in plans:
            assert all(not rp.lost for rp in p.values()), "a range lost its last holder"
        after = _state_bytes(reps)
        for name, a, b in zip(("master", "m", "v", "EMA"), before, after):
            assert torch.equal(a, b), f"{name} changed in the re-shard to {members}"
        assert all(reps.opts[m].lost_elements == 0 for m in members)
