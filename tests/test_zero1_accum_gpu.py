"""FT-ZeRO-1 gradient accumulation on ONE GPU: the accumulating reduce kernel modes against a PyTorch reference,
real signalling between micro-batches, clipping of the accumulated gradient, ``Zero1Optimizer`` across a change of
world, and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (see ``test_zero1_gpu.py``). Reference for a step of
``M`` micro-batches: ``s_m`` = fp32 sum of the ranks' bf16 gradients in rank order, ``reduced = bf16((((s_1 + s_2) +
...) + s_M) * scale)`` with ``scale = 1 / (contributors * M)`` in fp32.
"""

from __future__ import annotations

import pytest
import torch

from _zero1_replicas import NUMEL, UNITS, Replicas, kernel_world, raws, reduced, ref_adamw, trainer

pytestmark = pytest.mark.gpu

MAX_NORM = 50.0


def _scale(contributors, M):
    return 1.0 / (contributors * M)


def _accs(world, k):
    """Per rank: an fp32 accumulator (NaN-filled: every element must be written before it is read) and its offsets."""
    from torchft_b200.parallel.zero1 import ShardLayout, accum_offsets

    L = ShardLayout(tuple(UNITS), k)
    out = []
    for r in range(world):
        offs, n = accum_offsets(L, r, world)
        out.append((torch.full((n + 8,), float("nan"), device="cuda"), offs))
    return out


def _accum_reduce(world, k, micro, quiet=None, presignal=True, clip=False):
    """All micro-batches of one step through ``zero1_reduce_scatter_`` with the accumulator. Returns every rank's
    gradient segment afterwards and (``clip``) its per-unit sum-of-squares partials."""
    from torchft_b200.parallel.zero1 import accum_mode

    dev = torch.device("cuda", 0)
    comms = kernel_world(world, presignal)
    grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    gnorm = [c.segment("z1_gnorm")[: 8 * len(UNITS)].view(torch.float64) for c in comms]
    accs = _accs(world, k)
    M = len(micro)
    scale = _scale(world - (1 if quiet is not None else 0), M)
    order = ([quiet] if quiet is not None else []) + [r for r in range(world) if r != quiet]

    def rs(r, m, s):
        mode = accum_mode(m, M)
        acc, offs = accs[r]
        for u, (lo, hi) in enumerate(UNITS):
            gn = gnorm[r].data_ptr() + 8 * u if clip and mode == 3 else 0
            comms[r].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, scale, r != quiet, k, 4, s, gnorm=gn,
                                           acc=acc.data_ptr() + 4 * offs[u], acc_mode=mode)

    if presignal:
        for m, raw in enumerate(micro):
            for r in range(world):  # backward of micro-batch m rewrites every rank's gradient buffer
                grads[r].copy_(raw[r])
            if quiet is not None:
                grads[quiet].zero_()  # sequential emulation: the quiet rank's zeroing precedes everybody's reads
            torch.cuda.synchronize()
            for r in order:
                rs(r, m, None)
            torch.cuda.synchronize()
    else:
        # the trainer's order on every rank: backward (writes the gradient) on its compute stream behind the event
        # the comm stream recorded after the previous micro-batch's reduce-scatters, reduce-scatters on its comm stream
        compute = [torch.cuda.Stream(device=dev) for _ in comms]
        comm = [torch.cuda.Stream(device=dev) for _ in comms]
        done = [torch.cuda.Event() for _ in comms]
        torch.cuda.synchronize()
        for m, raw in enumerate(micro):
            for r in range(world):
                if m > 0:
                    compute[r].wait_event(done[r])
                with torch.cuda.stream(compute[r]):
                    grads[r].copy_(raw[r])
                comm[r].wait_stream(compute[r])
                rs(r, m, comm[r])
                done[r].record(comm[r])
        torch.cuda.synchronize()
    assert all(c.errored() is None for c in comms)
    return [g.clone() for g in grads], [x.clone() for x in gnorm]


def _check_holders(world, k, grads, want):
    from torchft_b200.parallel.zero1 import ShardLayout

    L = ShardLayout(tuple(UNITS), k)
    for u in range(len(UNITS)):
        for s in range(world):
            lo, hi = L.slice_bounds(u, world, s)
            for h in L.holders(u, world, s):
                assert torch.equal(grads[h][lo:hi], want[lo:hi]), f"holder {h} of unit {u} slice {s}"


# ----------------------------------------------------------------------------- the kernel modes vs the reference
@pytest.mark.parametrize("M", [2, 3])
@pytest.mark.parametrize("world,k", [(1, 1), (2, 2), (3, 2), (4, 3), (8, 1), (8, 2)])
def test_accumulated_reduce_matches_reference_bit_for_bit(world, k, M):
    quiet = 1 if world > 2 else None
    micro = raws(world, 10 * world + k + M, (1.0,) * M)
    grads, _ = _accum_reduce(world, k, micro, quiet=quiet)
    _check_holders(world, k, grads, reduced(micro, quiet))


def test_without_accumulator_the_launch_is_todays():
    """``acc = 0`` / ``acc_mode = 0`` is the plain launch: same number of launches, same bits."""
    world, k = 4, 2
    micro = raws(world, 3)
    out = []
    for kw in ({}, {"acc": 0, "acc_mode": 0}):
        comms = kernel_world(world)
        grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
        for r in range(world):
            grads[r].copy_(micro[0][r])
        torch.cuda.synchronize()
        before = [c.launches for c in comms]
        for r in range(world):
            for lo, hi in UNITS:
                comms[r].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0 / world, True, k, 4, None, **kw)
        torch.cuda.synchronize()
        out.append(([c.launches - b for c, b in zip(comms, before)], [g.clone() for g in grads]))
    assert out[0][0] == out[1][0]
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1]))
    _check_holders(world, k, out[0][1], reduced(micro))


def test_real_signalling_between_micro_batches_gives_the_presignalled_bits():
    """W = 4 ranks in flight at once; each rank overwrites its gradient with the next micro-batch only behind the event
    its comm stream recorded after the previous micro-batch's trailing handshakes."""
    world, k, M = 4, 2, 3
    micro = raws(world, 44, (1.0,) * M)
    seq, _ = _accum_reduce(world, k, micro)
    real, _ = _accum_reduce(world, k, micro, presignal=False)
    for r in range(world):
        assert torch.equal(seq[r], real[r]), f"rank {r}"
    _check_holders(world, k, real, reduced(micro))


@pytest.mark.parametrize("world,k", [(1, 1), (4, 2)])
def test_norm_of_the_accumulated_gradient(world, k):
    """The last micro-batch's sum-of-squares partials are bit-identical to those the M = 1 clipping path produces from
    ``reduced`` itself (rank 0 holding ``reduced``, every other rank zeros, scale 1), and their total is its norm."""
    M = 3
    micro = raws(world, 60 + world, (1.0,) * M)
    red = reduced(micro)
    grads, parts = _accum_reduce(world, k, micro, clip=True)
    _check_holders(world, k, grads, red)
    plain = [[red] + [torch.zeros_like(red)] * (world - 1)]
    comms = kernel_world(world)
    g = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    gn = [c.segment("z1_gnorm")[: 8 * len(UNITS)].view(torch.float64) for c in comms]
    for r in range(world):
        g[r].copy_(plain[0][r])
    torch.cuda.synchronize()
    for r in range(world):
        for u, (lo, hi) in enumerate(UNITS):
            comms[r].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0, True, k, 4, None, gnorm=gn[r].data_ptr() + 8 * u)
    torch.cuda.synchronize()
    for r in range(world):
        assert torch.equal(parts[r], gn[r]), f"partials of rank {r}"
    norm = float(red.double().norm())
    dev = float(sum(float(p.sum()) for p in parts)) ** 0.5
    assert abs(dev - norm) <= 1e-5 * norm


# ----------------------------------------------------------------------------- Zero1Optimizer
@pytest.mark.parametrize("compact", [False, True])
def test_optimizer_accumulates_through_a_change_of_world(compact):
    from torchft_b200.parallel.zero1 import ShardLayout, accum_elements, accum_offsets

    M, k = 3, 2
    reps = Replicas(4, compact=compact, min_world=3, grad_accum_steps=M)
    L = ShardLayout(tuple(UNITS), k)
    assert all(o.accum_bytes() == 4 * accum_elements(L, 3) for o in reps.opts)
    dev = torch.device("cuda", 0)
    rm, rmm, rv = reps.init.float(), torch.zeros(NUMEL, device=dev), torch.zeros(NUMEL, device=dev)
    t = 0
    seed = 100
    for members, epoch in (([0, 1, 2, 3], 1), ([0, 1, 3], 2), ([0, 1, 2, 3], 3)):
        if epoch == 3:  # member 2 rejoins from the healed weights
            reps.settle()
            o = reps.opts[2]
            o.param.copy_(reps.opts[0].param)
            if not compact:
                o.seed_master()
        reps.configure(members, epoch)
        world = len(members)
        for rank, i in enumerate(members):
            assert reps.opts[i]._acc_offsets == accum_offsets(L, rank, world)[0]
        for _ in range(2):
            seed += 1
            micro = raws(world, seed, (0.01,) * M)
            reps.step(micro)
            red = reduced(micro)
            t += 1
            ref_adamw(rm, rmm, rv, red.float(), t)
            assert reps.verdicts() == {i: True for i in members}
            for rank, i in enumerate(members):
                o = reps.opts[i]
                for lo, hi in L.held(rank, world):  # the update read exactly the reference's reduced gradient
                    assert torch.equal(o.grad[lo:hi], red[lo:hi]), f"member {i}, step {t}"
    reps.settle()
    for rank, i in enumerate(reps.members):
        o = reps.opts[i]
        assert o.t == t
        assert torch.equal(o.param, reps.opts[0].param)
        for (lo, hi), (master, m, v) in o.held_state().items():
            torch.testing.assert_close(master, rm[lo:hi], rtol=2e-5, atol=1e-6)
            torch.testing.assert_close(m, rmm[lo:hi], rtol=1e-5, atol=1e-7)
            torch.testing.assert_close(v, rv[lo:hi], rtol=1e-5, atol=1e-9)


def test_a_unit_short_of_micro_batches_vetoes_the_step():
    M, world = 3, 4
    reps = Replicas(world, min_world=3, grad_accum_steps=M)
    reps.configure([0, 1, 2, 3], 1)
    reps.step(raws(world, 5, (1.0,) * M))
    reps.settle()
    before = [(o.param.clone(), {r: tuple(x.clone() for x in s) for r, s in o.held_state().items()}) for o in reps.opts]
    reps.step(raws(world, 6, (1.0,) * M), skip=(1, M - 1))  # unit 1 never saw its last micro-batch
    assert reps.verdicts() == {i: False for i in range(world)}
    reps.settle()
    for o, (p, st) in zip(reps.opts, before):
        assert o.t == 1
        assert torch.equal(o.param, p)
        for r, s in o.held_state().items():
            assert all(torch.equal(a, b) for a, b in zip(s, st[r]))
    reps.step(raws(world, 7, (1.0,) * M))  # the counts start over: the next step commits
    assert reps.verdicts() == {i: True for i in range(world)}
    reps.settle()
    assert all(o.t == 2 for o in reps.opts)


def test_clipped_accumulation_matches_adamw_and_an_inf_in_an_early_micro_batch_vetoes():
    M, world, k = 3, 4, 2
    reps = Replicas(world, min_world=3, max_grad_norm=MAX_NORM, grad_accum_steps=M)
    reps.configure([0, 1, 2, 3], 1)
    dev = torch.device("cuda", 0)
    rm, rmm, rv = reps.init.float(), torch.zeros(NUMEL, device=dev), torch.zeros(NUMEL, device=dev)
    from torchft_b200.parallel.zero1 import ShardLayout

    L = ShardLayout(tuple(UNITS), k)
    t, clipped = 0, []
    for step, scale in enumerate((1.0, 0.01, 1.0, 1.0)):
        micro = raws(world, 200 + step, (scale,) * M)
        poisoned = step == 2
        if poisoned:
            micro[0][3][UNITS[1][0] + 9] = float("inf")  # micro-batch 0 of 3, rank 3
        reps.step(micro)
        red = reduced(micro)
        norms = [reps.opts[i].grad_norm.clone() for i in range(world)]
        assert all(torch.equal(n, norms[0]) for n in norms), "norm bits differ between ranks"
        if poisoned:
            assert float(norms[0]) == float("inf")
            assert reps.verdicts() == {i: False for i in range(world)}
            continue
        assert reps.verdicts() == {i: True for i in range(world)}
        norm = float(red.double().norm())
        assert abs(float(norms[0]) - norm) <= 1e-5 * norm
        coef = torch.clamp(MAX_NORM / (norms[0] + 1e-6), max=1.0)
        assert torch.equal(reps.opts[0]._clip[1], coef)
        clipped.append(bool(coef < 1))
        t += 1
        ref_adamw(rm, rmm, rv, red.float() * coef, t)
    reps.settle()
    assert any(clipped) and not all(clipped), clipped
    for rank, o in enumerate(reps.opts):
        assert o.t == t and o.nonfinite_steps == 1
        assert torch.equal(o.param, reps.opts[0].param)
        for lo, hi in L.held(rank, world):
            torch.testing.assert_close(o.master[lo:hi], rm[lo:hi], rtol=2e-5, atol=1e-6)


def test_accumulator_too_small_for_the_quorum_raises():
    from torch.distributed import PrefixStore

    from torchft_b200.parallel.symm_mem import SymmetricComm

    reps = Replicas(4, min_world=3, grad_accum_steps=2)
    SymmetricComm.virtual_quorum(reps.comms, [0, 1], 9)
    with pytest.raises(RuntimeError, match="accumulator bytes"):
        reps.opts[0]._on_configured(PrefixStore("q/9", reps.store), 0, 2, 9)


# ----------------------------------------------------------------------------- trainer
def _train(M, steps=3, tag="a", batch=4):
    with trainer("llama3_debug", f"z1acc_{tag}", grad_accum_steps=M) as tr:
        gen = torch.Generator().manual_seed(5)
        losses = []
        for _ in range(steps):
            tok = torch.randint(0, tr.cfg.vocab_size, (batch, 128), generator=gen).pin_memory()
            tgt = torch.randint(0, tr.cfg.vocab_size, (batch, 128), generator=gen).pin_memory()
            losses.append(tr.step(tok, tgt))
        assert tr.manager.current_step() == steps
        tr.join()
        torch.cuda.synchronize()
        return losses, tr.state_dict()["param"].clone(), (tr.zopt.accum_bytes() if M > 1 else 0)


def test_trainer_accumulating_two_micro_batches_matches_one_batch():
    l1, p1, _ = _train(1, tag="m1")
    l2, p2, acc_bytes = _train(2, tag="m2")
    assert acc_bytes == 4 * p1.numel()  # world 1: the accumulator covers the whole buffer
    assert abs(l1[0] - l2[0]) <= 2e-3 * abs(l1[0]), (l1, l2)  # same weights; bf16 GEMMs of half the rows
    torch.testing.assert_close(torch.tensor(l1), torch.tensor(l2), rtol=5e-3, atol=5e-3)
    diff = (p1.float() - p2.float()).abs()
    assert float(diff.max()) <= 8e-3 and float((diff > 0).float().mean()) < 0.25, (float(diff.max()), float((diff > 0).float().mean()))
    l3, p3, _ = _train(2, tag="m2b")
    assert l2 == l3 and torch.equal(p2, p3), "two accumulating runs with the same seed must be bit-identical"


def test_trainer_refuses_accumulation_without_zero1_and_an_indivisible_batch():
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    with pytest.raises(ValueError, match="grad_accum_steps"):
        FaultTolerantTrainer("llama3_debug", "unused:0", zero1=False, grad_accum_steps=2)
    with pytest.raises(ValueError, match="grad_accum_steps"):
        _train(3, steps=1, tag="bad", batch=4)
