"""Peer-memory collectives, W ranks of one quorum emulated in ONE process on ONE GPU
(``SymmetricComm.virtual_world(presignal=False)``: the ranks' kernels run concurrently on W streams and
synchronise through the real signal-pad protocol): staging rounds, multi-piece send/recv, the fp8 collectives
against their emulation, the pre-signalled mode, and the resiliency contract of the reference's
process_group_test.py:890-949: when a rank never shows up the survivors' collective fails within the timeout and
``errored()`` is latched. The plain all-reduce, reduce-scatter and push-exchange results are checked byte for byte in
``test_collectives_exact_gpu.py``.
"""

from __future__ import annotations

import pytest
import torch

import _q8_emulation as E
from _collectives import DEV, _ok, _run, _world

pytestmark = pytest.mark.gpu


def test_exchange_larger_than_staging_runs_in_rounds():
    comms = _world(4, staging=2 << 20)  # usable staging 1.5 MiB -> 384 KiB slots
    n = 1_000_003
    xs = [torch.full((n,), r + 1, dtype=torch.int32, device=DEV) for r in range(4)]
    outs = [torch.empty(4 * n, dtype=torch.int32, device=DEV) for _ in range(4)]
    _run(comms, lambda r, c, s: c.allgather_(outs[r], xs[r], stream=s))
    _ok(comms)
    assert all(torch.equal(o, torch.cat(xs)) for o in outs)


def test_send_recv_multi_piece_fifo():
    comms = _world(3, staging=4 << 20)  # 128 KiB mailboxes -> many pieces
    a = torch.arange(300_001, device=DEV, dtype=torch.float32)
    b = torch.arange(77, device=DEV, dtype=torch.int64)
    ra, rb = torch.empty_like(a), torch.empty_like(b)
    back = torch.empty_like(b)

    # (send and recv are different kernels; each has run once above would be needed under lazy module loading -- conftest
    # switches to eager loading for that reason)
    # one kernel per stream and phase: inside ONE process a second kernel queued behind a waiting one could be ordered
    # in front of the kernel it waits for (real ranks are separate processes with their own queues)
    _run(comms, lambda r, c, s: c.send_(a, 2, s) if r == 0 else c.recv_(ra, 0, s), ranks=(0, 2))
    _ok(comms)
    _run(comms, lambda r, c, s: c.send_(b, 2, s) if r == 0 else c.recv_(rb, 0, s), ranks=(0, 2))
    _run(comms, lambda r, c, s: c.send_(rb, 1, s) if r == 2 else c.recv_(back, 2, s), ranks=(1, 2))
    _ok(comms)
    assert torch.equal(ra, a) and torch.equal(rb, b) and torch.equal(back, b)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_q8_allreduce_and_reduce_scatter_within_reference_tolerance(world):
    comms = _world(world, staging=16 << 20)
    g = torch.Generator(device=DEV).manual_seed(9)
    for n, dtype in ((512, torch.float32), (100_000, torch.float32), ((1 << 20) + 24, torch.bfloat16)):
        a = [(torch.randn(n, device=DEV, generator=g) * 3).to(dtype) for _ in range(world)]
        b = [torch.randn(n, device=DEV, generator=g).to(dtype) for _ in range(world)]
        outs = [torch.empty(n, dtype=dtype, device=DEV) for _ in range(world)]
        _run(comms, lambda r, c, s: c.q8_allreduce_(outs[r], a[r], b[r], scale=1.0 / world, stream=s))
        _ok(comms)
        ref = sum(x.float() - y.float() for x, y in zip(a, b)) / world
        exact, _ = E.allreduce([E.pseudo_grad(x, y) for x, y in zip(a, b)], 1.0 / world)
        for o in outs:
            assert E.equal_bits(o, E.cast(exact, dtype)), E.first_mismatch(o, E.cast(exact, dtype))
            assert ((o.float() - ref).abs().mean() / ref.abs().mean()).item() <= 0.04  # collectives_test.py:186
        assert all(torch.equal(outs[0], o) for o in outs)
        se = ((n + world - 1) // world + 7) // 8 * 8
        rs = [torch.zeros(se, dtype=dtype, device=DEV) for _ in range(world)]
        _run(comms, lambda r, c, s: c.q8_reduce_scatter_(rs[r], a[r], se, scale=1.0 / world, stream=s))
        _ok(comms)
        tot = sum(x.float() for x in a) / world
        exact = E.reduce_scatter([E.load(x) for x in a], se, 1.0 / world)
        for r in range(world):
            valid = max(0, min(se, n - r * se))
            assert E.equal_bits(rs[r][:valid], E.cast(exact[r], dtype))
            if valid:
                want = tot[r * se: r * se + valid]
                assert ((rs[r][:valid].float() - want).abs().mean() / want.abs().mean()).item() <= 0.05  # :207


@pytest.mark.parametrize("world", [2, 8])
def test_q8_allreduce_large_message_pipeline_with_scratch_segment(world):
    """With a ``*_q8`` scratch segment the fp8 all-reduce runs as quantise -> handshake -> slice-reduce -> handshake ->
    gather+dequantise (sync-free kernels of any grid size): same numerics contract, same result on every rank."""
    n = (3 << 20) + 40
    comms = _world(world, segs={"buf": 1 << 20, "frag_q8": (n * 516 // 512 + 16 * 516 + 4096) * 3 // 2 + 8192})
    g = torch.Generator(device=DEV).manual_seed(21)
    for dtype in (torch.float32, torch.bfloat16):
        a = [(torch.randn(n, device=DEV, generator=g) * 2).to(dtype) for _ in range(world)]
        b = [torch.randn(n, device=DEV, generator=g).to(dtype) for _ in range(world)]
        outs = [torch.empty(n, dtype=dtype, device=DEV) for _ in range(world)]
        before = [c.launches for c in comms]
        _run(comms, lambda r, c, s: c.q8_allreduce_(outs[r], a[r], b[r], scale=1.0 / world, contribute=(r != 1 or world == 2), stream=s))
        _ok(comms)
        assert [c.launches - x for c, x in zip(comms, before)] == [5] * world  # 3 kernels + 2 handshakes, ONE pass
        quiet = None if world == 2 else 1
        ref = sum(x.float() - y.float() for r, (x, y) in enumerate(zip(a, b)) if r != quiet) / world
        exact, _, _ = E.allreduce_scratch([E.pseudo_grad(x, y) for x, y in zip(a, b)], 1.0 / world,
                                          [r != quiet for r in range(world)])
        for o in outs:
            assert E.equal_bits(o, E.cast(exact, dtype)), E.first_mismatch(o, E.cast(exact, dtype))
            assert ((o.float() - ref).abs().mean() / ref.abs().mean()).item() <= 0.04
        assert all(torch.equal(outs[0], o) for o in outs)


def test_dead_rank_latches_timeout_instead_of_hanging_then_abort_is_immediate():
    import time

    comms = _world(3, timeout=1.0)
    xs = [torch.ones(1 << 16, device=DEV) for _ in range(3)]
    t0 = time.monotonic()
    _run(comms, lambda r, c, s: c.allreduce_(xs[r], stream=s), ranks=(0, 1))  # rank 2 never launches
    took = time.monotonic() - t0
    assert 0.9 < took < 5.0
    for c in comms[:2]:
        e = c.errored()
        assert e is not None and "timeout waiting for replica rank 2" in str(e)
    # later kernels bail out immediately on the latched error (one timeout per failure, not one per queued kernel)
    t0 = time.monotonic()
    _run(comms, lambda r, c, s: c.allreduce_(xs[r], stream=s), ranks=(0, 1))
    assert time.monotonic() - t0 < 0.5


def test_host_abort_releases_spinning_kernels():
    import threading
    import time

    comms = _world(2, timeout=30.0)
    x = torch.ones(1 << 16, device=DEV)
    threading.Timer(0.3, comms[0].abort).start()
    t0 = time.monotonic()
    _run(comms, lambda r, c, s: c.allreduce_(x, stream=s), ranks=(0,))
    assert time.monotonic() - t0 < 5.0
    assert "aborted" in str(comms[0].errored())


def test_presignalled_world_emulates_ranks_one_kernel_at_a_time():
    """The profiler-friendly mode used by smoke(): run rank 0's kernel, then rank 1's, ... and still get the W-rank result."""
    from torchft_b200.bench_utils import collectives_selfcheck

    errs = collectives_selfcheck(world=4)
    assert errs["zero1_replicas_differ"] == 0
