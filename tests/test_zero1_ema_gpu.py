"""FT-ZeRO-1 EMA of the weights on ONE GPU: the kernel against its numpy specification bit for bit, against an fp64 EMA
of the device's own masters at every world, identical holders, a vetoed step, paged against flat state, kill / rejoin /
split commit / lost slices, checkpoints, the agreement check, ``ema_weights()`` and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (see ``_zero1_replicas.py``).
"""

from __future__ import annotations

import contextlib
import os
import threading
from datetime import timedelta

import numpy as np
import pytest
import torch

from _zero1_replicas import PG, UNITS, Replicas, bits, raws, trainer, warmup_cosine, widen

pytestmark = pytest.mark.gpu

BF16, FP32 = torch.bfloat16, torch.float32
DECAY = 0.9


def _c(decay=DECAY):
    from torchft_b200.parallel.zero1 import ema_coefficient

    return ema_coefficient(decay)


def _np(x):
    return x.contiguous().cpu().numpy()


# ----------------------------------------------------------------------------- the kernel, bit for bit
@pytest.mark.parametrize("moments", [FP32, BF16])
@pytest.mark.parametrize("paged", [False, True])
def test_kernel_ema_equals_the_numpy_specification(moments, paged):
    from torchft_b200.parallel.zero1 import bf16_sr_ema, ema_step

    world = 4
    reps = Replicas(world, k=2, compact=paged, moment_dtype=moments, ema_decay=DECAY)
    reps.configure(list(range(world)), 1)
    first = reps.full_ema()
    assert torch.equal(first.float(), reps.init.float()), "seeded with the master weights"
    for step in range(4):
        before = {(i, lo, hi): reps.get_ema(i, lo, hi) for i, lo, hi in reps.held()}
        reps.step(raws(world, 500 + step))
        reps.settle()
        t = reps.opts[0].t
        assert t == step + 1
        for (i, lo, hi), e0 in before.items():
            w = _np(reps.get(i, lo, hi)[0])
            e1 = reps.get_ema(i, lo, hi)
            if moments == FP32:
                want = ema_step(_np(e0), w, _c())
                assert (_np(e1).view(np.uint32) == want.view(np.uint32)).all(), f"member {i} {(lo, hi)} t={t}"
            else:
                want = bf16_sr_ema(ema_step(widen(bits(e0)), w, _c()), np.arange(lo, hi, dtype=np.uint64), t)
                assert (bits(e1) == want).all(), f"member {i} {(lo, hi)} t={t}"
            assert not torch.equal(e0, e1)


# ----------------------------------------------------------------------------- against fp64 at every world
CASES = [(w, k, paged) for w in (1, 2, 4, 8) for k in (1, 2) if k <= w for paged in (False, True)]


@pytest.mark.parametrize("world,k,paged", CASES)
def test_kernel_ema_follows_an_fp64_ema_of_the_device_masters(world, k, paged):
    """fp32 EMA: within a few fp32 ulps of the fp64 EMA of the masters the device produced (each step rounds three
    times, and the error contracts by d per step). Clipping and a schedule in some cases: they change ``w'`` only."""
    extras = {}
    if world == 4:
        extras = dict(max_grad_norm=5.0)
    if world == 8:
        extras = dict(lr_lambda=warmup_cosine, lr_steps=6)
    reps = Replicas(world, k=k, compact=paged, moment_dtype=FP32, ema_decay=DECAY, **extras)
    reps.configure(list(range(world)), 1)
    c = float(np.float32(1 - DECAY))
    ref = reps.init.double()
    for step in range(6):
        reps.step(raws(world, 40 * world + 7 * k + step))
        master = reps.full_state()[0]
        ref = ref + c * (master.double() - ref)
    got = reps.full_ema()
    assert got.dtype == FP32
    torch.testing.assert_close(got.double(), ref, rtol=1e-6, atol=1e-8)  # a few fp32 ulps of weights ~0.05
    moved = (got.double() - reps.init.double()).abs()
    assert float(moved.mean()) > 1e-4, "the EMA moved"
    assert all(o.t == 6 for o in reps.opts)


def test_bf16_ema_follows_the_fp64_ema_within_its_rounding_noise():
    world, steps = 2, 12
    reps = Replicas(world, k=2, moment_dtype=BF16, ema_decay=DECAY)
    reps.configure(list(range(world)), 1)
    c = float(np.float32(1 - DECAY))
    ref = reps.init.double()
    mag = ref.abs()  # each step rounds at the EMA's magnitude then: the noise is in ulps of the largest one it passed
    for step in range(steps):
        reps.step(raws(world, 900 + step))
        ref = ref + c * (reps.full_state()[0].double() - ref)
        mag = torch.maximum(mag, ref.abs())
    got = reps.full_ema().double()
    ulp = 2.0 ** (torch.floor(torch.log2(mag.clamp_min(1e-30))) - 7)  # one bf16 ulp
    dev = (got - ref) / ulp
    assert float(dev.abs().max()) < 10 and abs(float(dev.mean())) < 0.05 and float(dev.square().mean().sqrt()) < 2, \
        (float(dev.abs().max()), float(dev.mean()), float(dev.square().mean().sqrt()))


# ----------------------------------------------------------------------------- holders, vetoes, paging
def test_holders_agree_a_vetoed_step_leaves_the_ema_and_paged_equals_flat():
    world = 4
    runs = {}
    for moments in (FP32, BF16):
        for paged, blocks in ((False, 1), (False, 8), (True, 8)):
            reps = Replicas(world, k=2, blocks=blocks, compact=paged, moment_dtype=moments, ema_decay=DECAY)
            reps.configure(list(range(world)), 1)
            for step in range(4):
                rs = raws(world, 60 + step)
                if step == 2:
                    reps.settle()
                    before = [o.ema.clone() for o in reps.opts]
                    reps.step_vetoed_by_all(rs)
                    reps.settle()
                    for o, b in zip(reps.opts, before):
                        assert torch.equal(o.ema.view(torch.uint8), b.view(torch.uint8)), "a vetoed step moved the EMA"
                else:
                    reps.step(rs)
            runs[(moments, paged, blocks)] = (reps.full_ema(), reps.full_state()[0])
            assert all(o.t == 3 for o in reps.opts)
    for (moments, paged, blocks), (ema, master) in runs.items():
        ref_ema, ref_master = runs[(moments, False, 1)]
        assert torch.equal(ema, ref_ema) and torch.equal(master, ref_master), (moments, paged, blocks)


def test_without_an_ema_nothing_is_allocated_and_the_context_refuses():
    reps = Replicas(2, moment_dtype=FP32, ema_decay=None)
    reps.configure([0, 1], 1)
    o = reps.opts[0]
    assert o.ema is None and o._state_item() == 12 and o.state_bytes_allocated() == 12 * o.numel
    with pytest.raises(RuntimeError, match="no EMA"):
        o.held_ema()
    with pytest.raises(RuntimeError, match="no EMA"):
        with o.ema_weights():
            pass


# ----------------------------------------------------------------------------- faults
@pytest.mark.parametrize("compact", [False, True])
def test_kill_rejoin_and_split_commit_keep_the_ema_on_every_holder(compact):
    world = 4
    reps = Replicas(world, k=2, compact=compact, min_world=3, moment_dtype=BF16 if compact else FP32, ema_decay=DECAY)
    reps.configure([0, 1, 2, 3], 1)
    for step in range(2):
        reps.step(raws(4, 70 + step))
    src = reps.full_ema()
    reps.configure([0, 1, 3], 2)  # member 2 dies: its slices, EMA included, move to the survivors
    assert torch.equal(reps.full_ema(), src)
    reps.step(raws(3, 80))
    reps.settle()
    src = reps.full_ema()
    o = reps.make(reps.comms[2])  # ... and restarts with nothing but the weights
    o.param.copy_(reps.opts[0].param)
    o.seed_master()
    reps.opts[2] = o
    reps.configure([0, 1, 2, 3], 3)
    assert torch.equal(reps.full_ema(), src), "the joiner pulled its EMA slices with master, m and v"
    assert all(x.lost_elements == 0 for x in reps.opts)
    held = sum(hi - lo for lo, hi in reps.layout().held(2, 4))
    assert o.pulled_bytes == o._state_item() * held == (10 if compact else 16) * held  # master + m + v + EMA
    # a split commit: member 1 misses an update the others apply, then pulls their state at the next quorum
    reps.step(raws(4, 81), veto=[1])
    reps.settle()
    assert reps.opts[1].t + 1 == reps.opts[0].t
    others = {(lo, hi): reps.get_ema(i, lo, hi) for i, lo, hi in reps.held() if i != 1}
    reps.configure([0, 1, 2, 3], 4)
    for (lo, hi), e in others.items():
        for rank, i in enumerate(reps.members):
            if any(a <= lo and hi <= b for a, b in reps.opts[i]._holdings):
                assert torch.equal(reps.get_ema(i, lo, hi), e)
    reps.step(raws(4, 82))
    reps.full_ema()


def test_a_slice_lost_with_all_its_holders_is_reseeded_from_the_weights_and_counted():
    world = 3
    reps = Replicas(world, k=1, moment_dtype=FP32, ema_decay=DECAY)
    reps.configure([0, 1, 2], 1)
    for step in range(3):
        reps.step(raws(3, 110 + step))
    reps.settle()
    L = reps.layout()
    lost = L.held(2, 3)
    reps.configure([0, 1], 2)  # member 2 held its slices alone
    counted = sum(o.lost_elements for o in reps.opts[:2])
    assert counted == sum(hi - lo for lo, hi in lost) > 0
    ema = reps.full_ema()
    master = reps.full_state()[0]
    for lo, hi in lost:
        # re-seeded: the EMA restarts at the master, which restarts at the weights
        assert torch.equal(ema[lo:hi], master[lo:hi]) and torch.equal(master[lo:hi], reps.opts[0].param[lo:hi].float())


def test_mismatched_decays_raise_on_every_rank_before_anything_moves():
    for decay in ([DECAY, DECAY, 0.99], [DECAY, None, DECAY]):
        reps = Replicas(3, compact=True, moment_dtype=FP32, ema_decay=decay)
        before = [(o.t, list(o._holdings)) for o in reps.opts]
        errs = reps.configure_errors([0, 1, 2], 1)
        assert sorted(errs) == [0, 1, 2]
        for e in errs.values():
            assert isinstance(e, RuntimeError) and "disagree on the EMA" in str(e)
        for o, (t, hold) in zip(reps.opts, before):
            assert o.pulled_bytes == 0 and o.t == t and o._holdings == hold and not o._configured


# ----------------------------------------------------------------------------- checkpoints
def _saved(tmp_path, moments, decay=DECAY, world=4):
    live = Replicas(world, k=2, moment_dtype=moments, ema_decay=decay)
    live.configure(list(range(world)), 1)
    for step in range(2):
        live.step(raws(world, 90 + step))
    state = live.full_state()
    ema = live.full_ema() if decay is not None else None
    for o in live.opts:
        assert o.save(str(tmp_path), {"step": o.t, "batches_committed": 0}) == 2
    for o in live.opts:
        o.wait_checkpoint()
    return live, state, ema


@pytest.mark.parametrize("saved,restored", [(FP32, FP32), (BF16, BF16), (FP32, BF16), (BF16, FP32)])
@pytest.mark.parametrize("compact", [False, True])
def test_restore_at_another_world_keeps_or_converts_the_ema(tmp_path, saved, restored, compact):
    from torchft_b200.checkpointing.sharded import read_header, sections

    live, (master, m, v), ema = _saved(tmp_path, saved)
    h = read_header(os.path.join(tmp_path, "z1_step_2.w4.r0.bin"))
    ms = 2 if saved == BF16 else 4
    assert h["ema"] == {"decay": DECAY} and h["sections"] == sections(h["elements"], ms, ema=True)
    assert os.path.getsize(h["path"]) == h["data"] + (6 + 3 * ms) * h["elements"]
    back = Replicas(3, k=2, compact=compact, min_world=3, moment_dtype=restored, ema_decay=DECAY)
    for o in back.opts:
        assert o.restore(str(tmp_path))["step"] == 2
    back.configure([0, 1, 2], 1)
    assert torch.equal(back.full_state()[0], master)
    assert torch.equal(back.full_ema(), ema.to(restored))  # same type: the file's bits; otherwise converted
    assert all(o.lost_elements == 0 for o in back.opts)
    back.step(raws(3, 95))
    back.full_ema()


def test_restore_from_files_without_an_ema_seeds_it_from_the_master_weights(tmp_path, caplog):
    live, (master, _, _), _ = _saved(tmp_path, FP32, decay=None)
    from torchft_b200.checkpointing.sharded import read_header

    assert "ema" not in read_header(os.path.join(tmp_path, "z1_step_2.w4.r0.bin"))
    back = Replicas(2, k=2, compact=True, min_world=2, moment_dtype=FP32, ema_decay=DECAY)
    for o in back.opts:
        o.restore(str(tmp_path))
    with caplog.at_level("WARNING"):
        back.configure([0, 1], 1)
    assert "no EMA of the weights" in caplog.text
    assert torch.equal(back.full_ema(), master) and torch.equal(back.full_state()[0], master)
    # and a run without an EMA ignores a file's EMA section
    d2 = tmp_path / "with"
    _saved(d2, FP32)
    plain = Replicas(2, k=2, moment_dtype=FP32, ema_decay=None)
    for o in plain.opts:
        o.restore(str(d2))
    plain.configure([0, 1], 1)
    plain.step(raws(2, 97))
    plain.full_state()


def test_save_update_and_restore_raise_inside_ema_weights(tmp_path):
    reps = Replicas(2, k=2, moment_dtype=FP32, ema_decay=DECAY)
    reps.configure([0, 1], 1)
    reps.step(raws(2, 5))
    reps.settle()
    o = reps.opts[0]
    with o.ema_weights():
        for call in (lambda: o.update(), lambda: o.save(str(tmp_path)), lambda: o.restore(str(tmp_path))):
            with pytest.raises(RuntimeError, match="inside ema_weights"):
                call()
    o.update()  # allowed again after the exit


# ----------------------------------------------------------------------------- ema_weights()
@pytest.mark.parametrize("moments,world,k,paged", [(FP32, 4, 2, False), (BF16, 4, 2, True), (FP32, 1, 1, False),
                                                    (BF16, 3, 3, False)])
def test_ema_weights_puts_bf16_ema_in_every_param_and_restores_the_weights_bit_for_bit(moments, world, k, paged):
    reps = Replicas(world, k=k, compact=paged, moment_dtype=moments, ema_decay=DECAY)
    reps.configure(list(range(world)), 1)
    for step in range(3):
        reps.step(raws(world, 130 + step))
    reps.step(raws(world, 133), sync=False)  # the last update may still be queued when the context is entered
    reps.settle()
    params = [o.param.clone() for o in reps.opts]
    assert all(torch.equal(p, params[0]) for p in params)
    ema = reps.full_ema()
    want = ema if moments == BF16 else ema.bfloat16()  # fp32: rounded to nearest; bf16: as it is
    with contextlib.ExitStack() as stack:
        for o in reps.opts:
            stack.enter_context(o.ema_weights())
        torch.cuda.synchronize()
        for o in reps.opts:
            assert torch.equal(o.param, want)
        assert not torch.equal(want, params[0])
    torch.cuda.synchronize()
    for o, p in zip(reps.opts, params):
        assert torch.equal(o.param.view(torch.int16), p.view(torch.int16))
    reps.step(raws(world, 134))  # training goes on from the same weights
    reps.full_ema()


def test_ema_weights_waits_for_every_peer_before_it_pushes_with_real_signalling():
    """Two ranks on their own streams, signalling each other for real (W = k = 2: the last update ends without a
    handshake). Rank 1 is slow: it still reads its ``param`` (an evaluation) when rank 0 enters the context, and again
    when rank 0 leaves it. Rank 0's pushes of bf16(EMA) and then of bf16(master) must wait for rank 1 both times."""
    from torch.distributed import HashStore, PrefixStore

    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import Zero1Optimizer

    numel = UNITS[-1][1]
    seg = {"z1_param": numel * 2, "z1_grad": numel * 2, **{x: numel * 4 for x in ("z1_master", "z1_m", "z1_v", "z1_ema")}}
    comms = SymmetricComm.virtual_world(2, seg, presignal=False, timeout=timedelta(seconds=20))
    init = (torch.randn(numel, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9)) * 0.05).bfloat16()
    opts = [Zero1Optimizer(PG(c), numel, units=UNITS, replication=2, blocks=4, ema_decay=DECAY) for c in comms]
    for o in opts:
        o.param.copy_(init)
        o.seed_master()
    store = HashStore()
    ts = [threading.Thread(target=o._on_configured, args=(PrefixStore("q/1", store), r, 2, 1)) for r, o in enumerate(opts)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    for o in opts:
        o.ema.copy_(init.float() + 1.0)  # an EMA whose bf16 differs from the weights everywhere
        o.bind_stream(torch.cuda.Stream())
    torch.cuda.synchronize()
    want = (init.float() + 1.0).bfloat16()
    cur = [torch.cuda.Stream(), torch.cuda.Stream()]
    # one round without a slow rank first, so that no first-launch cost (loading the kernels) falls into the window below
    for r in (1, 0, 1, 0):
        with torch.cuda.stream(cur[r]):
            c = opts[r].ema_weights()
            c.__enter__()
            c.__exit__(None, None, None)
    torch.cuda.synchronize()
    slow = int(2e8)  # clock cycles, about 0.1 s: far longer than rank 0's launches take to reach rank 1
    ctx = [o.ema_weights() for o in opts]
    with torch.cuda.stream(cur[1]):
        torch.cuda._sleep(slow)
        before = opts[1].param.clone()
        ctx[1].__enter__()
    with torch.cuda.stream(cur[0]):
        ctx[0].__enter__()
        inside0 = opts[0].param.clone()
        ctx[0].__exit__(None, None, None)
    with torch.cuda.stream(cur[1]):
        torch.cuda._sleep(slow)
        inside1 = opts[1].param.clone()
        ctx[1].__exit__(None, None, None)
    torch.cuda.synchronize()
    assert all(c.errored() is None for c in comms)
    assert torch.equal(before, init), "a peer's EMA reached this rank's param before it entered the context"
    assert torch.equal(inside0, want) and torch.equal(inside1, want), "a peer's refresh reached param inside the context"
    for o in opts:
        assert torch.equal(o.param, init)


# ----------------------------------------------------------------------------- trainer
def test_trainer_ema_matches_an_fp64_ema_of_its_masters_and_evaluates_it(monkeypatch, tmp_path):
    monkeypatch.delenv("TORCHFT_B200_Z1_EMA_DECAY", raising=False)
    decay = 0.8
    with trainer("llama3_tiny", "z1ema_ema", lr=1e-3, ema_decay=decay) as tr:
        gen = torch.Generator().manual_seed(5)
        tok = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
        tgt = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
        zo = tr.zopt
        c = float(np.float32(1 - decay))
        ref = {r: x[0].double() for r, x in zo.held_state().items()}
        for _ in range(5):
            tr.step(tok, tgt)
            tr.manager.state_dict()  # resolve the step: held_state is its masters
            tr.join()
            ref = {r: ref[r] + c * (x[0].double() - ref[r]) for r, x in zo.held_state().items()}
        assert zo.t == 5
        ema = zo.held_ema()
        for r, e in ema.items():
            torch.testing.assert_close(e.double(), ref[r], rtol=1e-6, atol=1e-9)
        assert zo.state_bytes_allocated() == 16 * zo.numel
        weights = tr.flat.param.clone()
        with torch.no_grad():
            train_logits = tr.model(tok.cuda()[:, :16]).float()
        with tr.ema_weights():
            with torch.no_grad():
                ema_logits = tr.model(tok.cuda()[:, :16]).float()
            want = torch.cat([ema[r] for r in sorted(ema)]).bfloat16()
            assert torch.equal(tr.flat.param, want)
            for call in (lambda: tr.step(tok, tgt), lambda: tr.step_async(tok, tgt),
                         lambda: tr.step_device(tok.cuda(), tgt.cuda()), lambda: tr.save_checkpoint(str(tmp_path))):
                with pytest.raises(RuntimeError, match="inside ema_weights"):
                    call()
        torch.cuda.synchronize()
        assert torch.equal(tr.flat.param.view(torch.int16), weights.view(torch.int16))
        assert not torch.equal(ema_logits, train_logits), "the evaluation saw the EMA weights"
        with torch.no_grad():
            assert torch.equal(tr.model(tok.cuda()[:, :16]).float(), train_logits)
        tr.step(tok, tgt)  # training continues from the same weights
        tr.manager.state_dict()
        assert zo.t == 6


def test_trainer_takes_the_decay_from_the_environment_and_refuses_the_classic_pipeline(monkeypatch):
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    monkeypatch.setenv("TORCHFT_B200_Z1_EMA_DECAY", "0.99")
    with trainer("llama3_tiny", "z1ema_env", lr=1e-3) as tr:
        assert tr.zopt.ema_decay == 0.99 and tr.zopt.ema is not None and tr.zopt.ema.dtype == FP32
    for pipe in (dict(zero1=False), dict(backend="nccl")):
        with pytest.raises(ValueError, match="ema_decay"):
            FaultTolerantTrainer("llama3_tiny", "unused:0", ema_decay=0.99, **pipe)
