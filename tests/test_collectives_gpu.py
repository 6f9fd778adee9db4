"""Every peer-memory collective kernel, W ranks of one quorum emulated in ONE process on ONE GPU
(``SymmetricComm.virtual_world(presignal=False)``: the ranks' kernels run concurrently on W streams and
synchronise through the real signal-pad protocol). Exact values per collective, as the reference's
process_group_test.py:143-492 does with rank threads, plus the resiliency contract of :890-949: when a rank
never shows up the survivors' collective fails within the timeout and ``errored()`` is latched.
"""

from __future__ import annotations

import pytest
import torch

import _q8_emulation as E
from _collectives import DEV, _ok, _run, _world

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_allreduce_paths_exact(world, dtype):
    comms = _world(world)
    g = torch.Generator(device=DEV).manual_seed(world)
    for n, plan in ((5, None), (4096, (0, 4)), (100_003, (1, 8)), (1 << 19, (1, 16)), (70_000, None)):
        xs = [torch.randint(-8, 8, (n,), device=DEV, generator=g).to(dtype) for _ in range(world)]  # exactly summable
        want = sum(x.float() for x in xs)
        # symmetric (zero-copy) path
        es = xs[0].element_size()
        views = [c.segment("buf")[: n * es].view(dtype) for c in comms]
        for v, x in zip(views, xs):
            v.copy_(x)

        def symm(r, c, s):
            c._force_plan = plan
            c.allreduce_(views[r], scale=0.5, stream=s)
            c._force_plan = None

        _run(comms, symm)
        _ok(comms)
        for v in views:
            assert torch.equal(v.float(), want * 0.5)
        # staged path (tensor outside symmetric memory), MAX, and a non-contributing rank
        ys = [x.clone() for x in xs]
        _run(comms, lambda r, c, s: c.allreduce_(ys[r], op=1, stream=s))
        for y in ys:
            assert torch.equal(y.float(), torch.stack([x.float() for x in xs]).max(0).values)
        zs = [x.clone() for x in xs]
        _run(comms, lambda r, c, s: c.allreduce_(zs[r], contribute=(r != 0), stream=s))
        _ok(comms)
        for z in zs:
            assert torch.equal(z.float(), want - xs[0].float())
    # random normal values: the sum is exact only in the kernels' order, rank 0 first, in fp32, then the scale and one
    # round-to-nearest-even cast, on every rank and for both plans
    n = 100_003
    xs = [torch.randn(n, device=DEV, generator=g).to(dtype) for _ in range(world)]
    want = _rank_order_sum(xs, 0.5).to(dtype)
    for plan in ((0, 16), (1, 8)):
        views = [c.segment("buf")[: n * xs[0].element_size()].view(dtype) for c in comms]
        for v, x in zip(views, xs):
            v.copy_(x)
        ys = [x.clone() for x in xs]

        def both(r, c, s):
            c._force_plan = plan
            c.allreduce_(views[r], scale=0.5, stream=s)
            c.allreduce_(ys[r], scale=0.5, stream=s)
            c._force_plan = None

        _run(comms, both)
        _ok(comms)
        for v, y in zip(views, ys):
            assert torch.equal(v, want) and torch.equal(y, want), plan


def _rank_order_sum(xs, scale):
    acc = xs[0].float()
    for x in xs[1:]:
        acc = acc + x.float()
    return acc * scale


@pytest.mark.parametrize("world", [2, 3, 8])
def test_allgather_broadcast_alltoall_exact(world):
    comms = _world(world)
    for n, dtype in ((7, torch.int64), (4096, torch.float32), (33_333, torch.bfloat16), (1 << 20, torch.uint8)):
        xs = [(torch.arange(n, device=DEV) * (r + 1) % 251).to(dtype) for r in range(world)]
        outs = [torch.empty(world * n, dtype=dtype, device=DEV) for _ in range(world)]
        _run(comms, lambda r, c, s: c.allgather_(outs[r], xs[r], stream=s))
        _ok(comms)
        want = torch.cat(xs)
        assert all(torch.equal(o, want) for o in outs)
        for root in (0, world - 1):
            bs = [x.clone() for x in xs]
            _run(comms, lambda r, c, s: c.broadcast_(bs[r], root, stream=s))
            assert all(torch.equal(b, xs[root]) for b in bs)
        m = n - n % world or world
        ins = [(torch.arange(m, device=DEV) + 1000 * r).to(torch.int32) for r in range(world)]
        a2a = [torch.empty(m, dtype=torch.int32, device=DEV) for _ in range(world)]
        _run(comms, lambda r, c, s: c.alltoall_(a2a[r], ins[r], stream=s))
        _ok(comms)
        c_ = m // world
        for r in range(world):
            assert torch.equal(a2a[r], torch.cat([ins[p][r * c_:(r + 1) * c_] for p in range(world)]))


def test_exchange_larger_than_staging_runs_in_rounds():
    comms = _world(4, staging=2 << 20)  # usable staging 1.5 MiB -> 384 KiB slots
    n = 1_000_003
    xs = [torch.full((n,), r + 1, dtype=torch.int32, device=DEV) for r in range(4)]
    outs = [torch.empty(4 * n, dtype=torch.int32, device=DEV) for _ in range(4)]
    _run(comms, lambda r, c, s: c.allgather_(outs[r], xs[r], stream=s))
    _ok(comms)
    assert all(torch.equal(o, torch.cat(xs)) for o in outs)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_reduce_scatter_exact(world):
    comms = _world(world, segs={"buf": 8 << 20})
    g = torch.Generator(device=DEV).manual_seed(3)
    for n, dtype in ((8, torch.float32), (1001, torch.float32), (65_536, torch.bfloat16)):
        ins = [torch.randint(-8, 8, (world * n,), device=DEV, generator=g).to(dtype) for _ in range(world)]
        outs = [torch.empty(n, dtype=dtype, device=DEV) for _ in range(world)]
        _run(comms, lambda r, c, s: c.reduce_scatter_(outs[r], ins[r], scale=0.25, stream=s))
        _ok(comms)
        tot = sum(x.float() for x in ins)
        for r in range(world):
            assert torch.equal(outs[r].float(), tot[r * n:(r + 1) * n] * 0.25)
        # zero-copy: input already in symmetric memory
        es = ins[0].element_size()
        views = [c.segment("buf")[: world * n * es].view(dtype) for c in comms]
        for v, x in zip(views, ins):
            v.copy_(x)
        _run(comms, lambda r, c, s: c.reduce_scatter_(outs[r], views[r], op=2, stream=s))
        _ok(comms)
        mn = torch.stack([x.float() for x in ins]).min(0).values
        for r in range(world):
            assert torch.equal(outs[r].float(), mn[r * n:(r + 1) * n])
    for n, dtype in ((1001, torch.float32), (65_536, torch.bfloat16), (4104, torch.float16)):
        ins = [torch.randn(world * n, device=DEV, generator=g).to(dtype) for _ in range(world)]
        outs = [torch.empty(n, dtype=dtype, device=DEV) for _ in range(world)]
        _run(comms, lambda r, c, s: c.reduce_scatter_(outs[r], ins[r], scale=0.25, stream=s))
        _ok(comms)
        want = _rank_order_sum(ins, 0.25).to(dtype)
        for r in range(world):
            assert torch.equal(outs[r], want[r * n:(r + 1) * n]), (n, dtype, r)


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
