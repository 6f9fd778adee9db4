"""FT-ZeRO-1 learning-rate schedules and weight-decay exemptions on ONE GPU: the update kernel against
``torch.optim.AdamW`` with two parameter groups and ``LambdaLR``, neutral settings, vetoed steps, a kill and a rejoin,
a restore, the agreement check and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (see ``_zero1_replicas.py``). The reference steps
its scheduler once per committed step, on the same reduced gradients, in fp32.
"""

from __future__ import annotations

import numpy as np
import pytest
import torch

from _zero1_replicas import HP, NUMEL, STEPS, UNITS, Replicas, raws, reduced, trainer, warmup_cosine

pytestmark = pytest.mark.gpu

LR, B1, B2, EPS, WD = HP
# exempt ranges in every unit: short and long ones, across slice and page bounds, one ending at a unit's end
NO_DECAY = ((8, 64), (4096, 20000), (UNITS[1][0] + 800, UNITS[1][0] + 1600), (UNITS[2][0] + 16, UNITS[2][1]))
SCHED = dict(lr_lambda=warmup_cosine, lr_steps=STEPS, no_decay=NO_DECAY)  # the schedule and exemptions of most tests


def _mask(ranges):
    m = torch.zeros(NUMEL, dtype=torch.bool, device="cuda")
    for lo, hi in ranges:
        m[lo:hi] = True
    return m


class Ref:
    """fp32 ``torch.optim.AdamW`` over the flat vector in two groups (decay / no decay) with ``LambdaLR``; the scheduler
    steps after every committed update and holds its last value past ``steps`` entries."""

    def __init__(self, init, lam, steps, no_decay):
        self.mask = _mask(no_decay)
        w = init.float()
        self.pd = torch.nn.Parameter(w[~self.mask].clone())
        self.pn = torch.nn.Parameter(w[self.mask].clone())
        groups = [{"params": [self.pd], "weight_decay": WD}, {"params": [self.pn], "weight_decay": 0.0}]
        self.opt = torch.optim.AdamW(groups, lr=LR, betas=(B1, B2), eps=EPS, foreach=False)
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda i: lam(min(i, steps - 1)))

    def step(self, g):
        self.pd.grad = g[~self.mask].clone()
        self.pn.grad = g[self.mask].clone()
        self.opt.step()
        self.sched.step()

    def state(self):
        out = []
        for get in (lambda p: p.detach(), lambda p: self.opt.state[p]["exp_avg"], lambda p: self.opt.state[p]["exp_avg_sq"]):
            x = torch.empty(NUMEL, device="cuda")
            x[~self.mask] = get(self.pd)
            x[self.mask] = get(self.pn)
            out.append(x)
        return out


def _check(reps, ref, weights=True):
    """Every member's weights are equal; its held state matches the reference; holders of a slice agree bit for bit.

    ``weights=False`` for the first step after a re-shard: the pre-signalled virtual world runs each member's launches
    to the end before the next member's, so a later member's refresh (the ungated re-broadcast of its pre-update
    masters) can overwrite weights that an earlier holder of the same slice has already updated. Concurrent ranks order
    every refresh before any update through the handshakes; here the copy heals at the next update."""
    from torchft_b200.parallel.zero1 import ShardLayout

    reps.settle()
    torch.cuda.synchronize()
    rm, rmm, rv = ref.state()
    first = reps.opts[reps.members[0]]
    held = {}
    for rank, i in enumerate(reps.members):
        o = reps.opts[i]
        assert not weights or torch.equal(o.param, first.param), f"weights of member {i}"
        held[rank] = o.held_state()
        for (lo, hi), (master, m, v) in held[rank].items():
            torch.testing.assert_close(master, rm[lo:hi], rtol=2e-5, atol=1e-7)
            torch.testing.assert_close(m, rmm[lo:hi], rtol=1e-5, atol=1e-7)
            torch.testing.assert_close(v, rv[lo:hi], rtol=1e-5, atol=1e-9)
    world = len(reps.members)
    L = ShardLayout(tuple(reps.units), reps.k)

    def at(rank, lo, hi):
        for (a, b), xs in held[rank].items():
            if a <= lo and hi <= b:
                return [x[lo - a:hi - a] for x in xs]
        raise AssertionError(f"rank {rank} does not hold [{lo}, {hi})")

    for u in range(len(reps.units)):
        for s in range(world):
            lo, hi = L.slice_bounds(u, world, s)
            if hi == lo:
                continue
            hs = L.holders(u, world, s)
            for h in hs[1:]:
                for a, b in zip(at(hs[0], lo, hi), at(h, lo, hi)):
                    assert torch.equal(a, b), f"holders {hs} of unit {u} slice {s}"
            assert not weights or torch.equal(first.param[lo:hi], at(hs[0], lo, hi)[0].bfloat16())


# ----------------------------------------------------------------------------- kernels vs the reference
CASES = [(w, k, paged) for w in (1, 2, 4, 8) for k in (1, 2) if k <= w for paged in (False, True)]


@pytest.mark.parametrize("world,k,paged", CASES)
def test_scheduled_update_with_exemptions_matches_adamw_with_lambda_lr(world, k, paged):
    clip = world == 4 or (world == 8 and paged)
    reps = Replicas(world, k=k, compact=paged, max_grad_norm=5.0 if clip else None, **SCHED)
    reps.configure(list(range(world)), 1)
    ref = Ref(reps.init, warmup_cosine, STEPS, NO_DECAY)
    clipped = []
    for step in range(STEPS + 2):  # two updates past the end of the table
        rs = raws(world, 100 * world + 10 * k + step, (1.0 if step % 2 else 0.01,))
        reps.step(rs)
        g = reduced(rs).float()
        if clip:
            coef = reps.opts[0]._clip[1].clone()
            clipped.append(float(coef) < 1)
            g = g * coef
        ref.step(g)
        assert all(o.t == step for o in reps.opts)  # settles lazily, at the next step
    assert all(o.lr_at(STEPS + 2) == o.lr_at(STEPS) for o in reps.opts)
    _check(reps, ref)
    assert all(o.t == STEPS + 2 for o in reps.opts)
    if clip:
        assert any(clipped) and not all(clipped), clipped


@pytest.mark.parametrize("world,paged", [(1, False), (2, True), (4, False), (4, True)])
def test_neutral_schedule_and_no_exemptions_change_nothing(world, paged):
    """A lambda that is always 1.0 and no exempt ranges: the same bits as the launch without either."""
    runs = []
    for lam in (None, lambda i: 1.0):
        reps = Replicas(world, compact=paged, lr_lambda=lam, lr_steps=3)
        reps.configure(list(range(world)), 1)
        for step in range(5):
            reps.step(raws(world, 7 + step))
        reps.settle()
        runs.append([(o.param.clone(), o.held_state()) for o in reps.opts])
    assert runs[1][0][1], "something is held"
    for (pa, ha), (pb, hb) in zip(*runs):
        assert torch.equal(pa, pb)
        assert ha.keys() == hb.keys()
        for r in ha:
            for x, y in zip(ha[r], hb[r]):
                assert torch.equal(x, y)


def test_vetoed_steps_do_not_advance_the_schedule():
    world = 4
    lam = [1.0, 0.25, 2.0, 0.5, 1.5, 0.75].__getitem__  # a wrong rate anywhere shows in the state
    reps = Replicas(world, max_grad_norm=float("inf"), **{**SCHED, "lr_lambda": lam, "lr_steps": 6})
    reps.configure(list(range(world)), 1)
    ref = Ref(reps.init, lam, 6, NO_DECAY)
    plan = [None, "veto", None, "nonfinite", None]
    committed = 0
    for step, what in enumerate(plan):
        rs = raws(world, 60 + step)
        if what == "nonfinite":
            rs[0][2][UNITS[1][0] + 100] = float("inf")
        if what == "veto":
            reps.step_vetoed_by_all(rs)
        else:
            reps.step(rs)
        reps.settle()
        if what is None:
            committed += 1
            ref.step(reduced(rs).float())
        for o in reps.opts:
            assert o.t == committed, (step, what)
            assert o.lr_at(o.t + 1) == float(np.float32(LR * lam(committed)))
    assert reps.opts[0].nonfinite_steps == 1
    _check(reps, ref)

    # a split commit: member 1 misses an update the others apply, then adopts their count at the next quorum
    rs = raws(world, 70)
    reps.step(rs, veto=[1])
    reps.settle()
    ref.step(reduced(rs).float())
    assert reps.opts[1].t == committed and all(reps.opts[i].t == committed + 1 for i in (0, 2, 3))
    reps.configure(list(range(world)), 2)
    assert all(o.t == committed + 1 for o in reps.opts)
    for seed in (71, 72):
        rs = raws(world, seed)
        reps.step(rs)
        ref.step(reduced(rs).float())
        _check(reps, ref, weights=seed == 72)
    assert all(o.t == committed + 3 for o in reps.opts)


def test_kill_and_rejoin_keep_every_holder_on_the_schedule():
    world = 4
    lam = [1.0, 0.5, 2.0, 0.25, 1.5, 0.75, 1.25, 0.6].__getitem__  # a distinct rate per update
    reps = Replicas(world, k=2, **{**SCHED, "lr_lambda": lam, "lr_steps": 8})
    ref = Ref(reps.init, lam, 8, NO_DECAY)
    g = torch.Generator(device="cuda").manual_seed(3)

    def step():
        gstep = torch.randn(NUMEL, device="cuda", generator=g).bfloat16()  # the reduced gradient, identical everywhere
        reps.step([[gstep] * len(reps.members)], reduce=False)
        ref.step(gstep.float())

    reps.configure([0, 1, 2, 3], 1)
    step()
    step()
    reps.configure([0, 1, 3], 2)  # member 2 dies
    step()
    _check(reps, ref, weights=False)
    step()
    _check(reps, ref)
    o = reps.make(reps.comms[2])  # ... and restarts from the healed weights
    o.param.copy_(reps.opts[0].param)
    o.seed_master()
    reps.opts[2] = o
    reps.configure([0, 1, 2, 3], 3)
    tmax = reps.opts[0].t
    assert o.t == tmax == 4
    assert o.lr_at(o.t + 1) == float(np.float32(LR * lam(tmax)))
    step()  # the joiner's first update applies lr_{tmax + 1}
    _check(reps, ref, weights=False)
    assert all(x.t == tmax + 1 for x in reps.opts)
    step()
    _check(reps, ref)
    assert all(x.lost_elements == 0 for x in reps.opts)


@pytest.mark.parametrize("world", [4, 2])
def test_restore_continues_the_schedule(tmp_path, world):
    g = torch.Generator(device="cuda").manual_seed(8)
    grads = [torch.randn(NUMEL, device="cuda", generator=g).bfloat16() for _ in range(4)]
    live = Replicas(4, **SCHED)
    ref = Ref(live.init, warmup_cosine, STEPS, NO_DECAY)
    live.configure([0, 1, 2, 3], 1)
    for gs in grads[:2]:
        live.step([[gs] * 4], reduce=False)
        ref.step(gs.float())
    live.settle()
    for o in live.opts:
        assert o.save(str(tmp_path), {"step": o.t, "batches_committed": 0}) == 2
    for o in live.opts:
        o.wait_checkpoint()
    for gs in grads[2:]:  # the uninterrupted run
        live.step([[gs] * 4], reduce=False)
        ref.step(gs.float())
    live.settle()

    back = Replicas(world, **SCHED)
    for o in back.opts:
        assert o.restore(str(tmp_path))["step"] == 2 and o.t == 2
    back.configure(list(range(world)), 1)
    for gs in grads[2:]:
        back.step([[gs] * world], reduce=False)
    back.settle()
    assert all(o.t == 4 for o in back.opts)
    if world == 4:
        for a, b in zip(live.opts, back.opts):
            assert torch.equal(a.param, b.param)
            ha, hb = a.held_state(), b.held_state()
            assert ha.keys() == hb.keys()
            for r in ha:
                for x, y in zip(ha[r], hb[r]):
                    assert torch.equal(x, y), r
    _check(back, ref)


@pytest.mark.parametrize("what", ["lambda", "no_decay", "schedule_on_one_rank"])
def test_mismatched_schedules_raise_on_every_rank_before_anything_moves(what):
    world = 3
    kw = {"lambda": dict(lr_lambda=[warmup_cosine, warmup_cosine, lambda i: 1.0]),
          "no_decay": dict(no_decay=[NO_DECAY, NO_DECAY, NO_DECAY[:2]]),
          "schedule_on_one_rank": dict(lr_lambda=[warmup_cosine, None, warmup_cosine])}[what]
    reps = Replicas(world, compact=what == "no_decay", **{**SCHED, **kw})
    before = [(o.t, list(o._holdings)) for o in reps.opts]
    errs = reps.configure_errors([0, 1, 2], 1)
    assert sorted(errs) == [0, 1, 2]
    for e in errs.values():
        assert isinstance(e, RuntimeError) and "disagree" in str(e)
    for o, (t, hold) in zip(reps.opts, before):
        assert o.pulled_bytes == 0 and o.t == t and o._holdings == hold and not o._configured


# ----------------------------------------------------------------------------- trainer
def _train(tag, steps=3, lr=3e-4, **kw):
    with trainer("llama3_tiny", f"z1sched_{tag}", lr=lr, **kw) as tr:
        torch.cuda.synchronize()
        start = (tr.zopt.param.clone(), tr.zopt.master.clone())
        gen = torch.Generator().manual_seed(5)
        losses, lrs, ts = [], [], []
        for _ in range(steps):
            tok = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
            tgt = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
            losses.append(tr.step(tok, tgt))
            lrs.append(tr.last_lr())
            ts.append(tr.zopt.t)
        tr.manager.state_dict()  # settles the last verdict
        lrs.append(tr.last_lr())
        ts.append(tr.zopt.t)
        tr.join()
        torch.cuda.synchronize()
        where = {n: (o, p.numel(), p.ndim) for (n, p) in tr.model.named_parameters()
                 for q, o in zip(tr.flat.params, tr.flat.offsets) if q is p}
        return {"loss": losses, "lr": lrs, "t": ts, "start": start, "param": tr.zopt.param.clone(),
                "master": tr.zopt.master.clone(), "where": where}


def test_trainer_with_a_constant_schedule_reproduces_the_trainer_without_one():
    a = _train("plain")
    b = _train("const", lr_lambda=lambda i: 1.0, lr_steps=10)
    assert a["loss"] == b["loss"]
    assert torch.equal(a["param"], b["param"]) and torch.equal(a["master"], b["master"])
    assert all(x is None or x == float(np.float32(3e-4)) for x in a["lr"])


def test_trainer_reports_the_rate_of_the_last_resolved_update():
    lam = [0.5, 1.0, 0.75, 0.25].__getitem__
    r = _train("lr", steps=4, lr=1e-3, lr_lambda=lam, lr_steps=4)
    assert r["t"][-1] == 4
    for t, x in zip(r["t"], r["lr"]):
        assert x is None if t == 0 else x == float(np.float32(1e-3 * lam(t - 1))), (t, x)
    assert r["lr"][-1] == float(np.float32(1e-3 * 0.25))


def test_trainer_with_a_zero_first_rate_leaves_the_weights_alone():
    r = _train("zero", steps=1, lr_lambda=lambda i: 0.0 if i == 0 else 1.0, lr_steps=2)
    assert r["t"][-1] == 1
    assert torch.equal(r["param"], r["start"][0]) and torch.equal(r["master"], r["start"][1])


def test_trainer_exempts_the_norm_gains_from_weight_decay():
    lr = 1e-2
    a = _train("decay", steps=1, lr=lr)
    b = _train("nodecay", steps=1, lr=lr, no_decay=lambda n, p: p.ndim == 1)
    assert a["t"][-1] == b["t"][-1] == 1
    gains = torch.zeros_like(a["master"], dtype=torch.bool)
    for n, (o, numel, ndim) in a["where"].items():
        if ndim == 1:
            gains[o:o + numel] = True
    assert int(gains.sum()) > 0
    assert torch.equal(a["master"][~gains], b["master"][~gains]), "every matrix element is unchanged"
    w0 = a["start"][1][gains]
    torch.testing.assert_close(b["master"][gains] - a["master"][gains], lr * WD * w0, rtol=1e-3, atol=1e-7)


def test_trainer_refuses_schedules_and_exemptions_on_the_classic_pipeline():
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    for kw in (dict(lr_lambda=lambda i: 1.0, lr_steps=4), dict(no_decay=lambda n, p: p.ndim == 1)):
        for pipe in (dict(zero1=False), dict(backend="nccl")):
            with pytest.raises(ValueError, match="lr_lambda and no_decay"):
                FaultTolerantTrainer("llama3_tiny", "unused:0", **pipe, **kw)


def test_kernel_constant_matches_the_python_cap():
    from torchft_b200.ops import _native
    from torchft_b200.parallel.zero1 import MAX_NO_DECAY

    assert _native.load().ZERO1_MAX_NO_DECAY == MAX_NO_DECAY
