"""FT-ZeRO-1 bf16 moments on ONE GPU: the device rounding against its numpy specification bit for bit, one update against
the fp32 reference, bit-identical holders at any grid and paging through a vetoed step, thirty steps against fp32
moments, kill / rejoin / re-shard, the agreement check, checkpoints across moment types, and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (see ``_zero1_replicas.py``).
"""

from __future__ import annotations

import os
from datetime import timedelta

import numpy as np
import pytest
import torch

from _zero1_replicas import HP, PG, Replicas, ref_adamw
from test_zero1_sched_gpu import NUMEL, UNITS, _configure_errors, _raws, _reduced, _step_vetoed_by_all

pytestmark = pytest.mark.gpu

LR, B1, B2, EPS, WD = HP
BF16, FP32 = torch.bfloat16, torch.float32


class MReplicas(Replicas):
    """:class:`Replicas` whose optimizers keep ``moments`` (a dtype, or one per member) and launch updates of at most
    ``blocks`` CTAs; ``lam`` / ``lr_steps`` add a learning-rate schedule."""

    def __init__(self, n, moments=BF16, blocks=4, lam=None, lr_steps=0, units=UNITS, **kw):
        self.moments, self.blocks, self.lam, self.lr_steps = moments, blocks, lam, lr_steps
        super().__init__(n, units, **kw)

    def make(self, comm):
        from torchft_b200.parallel.zero1 import Zero1Optimizer

        md = self.moments[self.comms.index(comm)] if isinstance(self.moments, list) else self.moments
        return Zero1Optimizer(PG(comm), self.numel, units=self.units, lr=LR, betas=(B1, B2), eps=EPS, weight_decay=WD,
                              replication=self.k, blocks=self.blocks, compact=self.compact, min_world=self.min_world,
                              page_shift=8, max_grad_norm=self.max_norm, grad_accum_steps=self.M, lr_lambda=self.lam,
                              lr_steps=self.lr_steps, moment_dtype=md)

    def layout(self):
        from torchft_b200.parallel.zero1 import ShardLayout

        return ShardLayout(tuple(self.units), self.k)

    def held(self):
        """``(member, lo, hi)`` over every range a member of the current quorum holds."""
        L, world = self.layout(), len(self.members)
        return [(i, lo, hi) for rank, i in enumerate(self.members) for lo, hi in L.held(rank, world)]

    def get(self, i, lo, hi):
        """(master, m, v) of member ``i`` over ``[lo, hi)``, through its page table."""
        o = self.opts[i]
        torch.cuda.synchronize()
        pieces = o._pieces(o._table_host, lo, hi)
        return tuple(torch.cat([x[at:at + b - a] for a, b, at in pieces]) for x in (o.master, o.m, o.v))

    def put(self, m, v):
        """Write the flat vectors ``m`` and ``v`` into every holder's moments."""
        for i, lo, hi in self.held():
            o = self.opts[i]
            for a, b, at in o._pieces(o._table_host, lo, hi):
                o.m[at:at + b - a].copy_(m[a:b])
                o.v[at:at + b - a].copy_(v[a:b])
        torch.cuda.synchronize()

    def full_state(self):
        """(master, m, v) over the whole vector assembled from the holders, which must agree bit for bit."""
        self.settle()
        o0 = self.opts[self.members[0]]
        out = [torch.zeros(self.numel, dtype=x.dtype, device="cuda") for x in (o0.master, o0.m, o0.v)]
        seen = torch.zeros(self.numel, dtype=torch.bool, device="cuda")
        for i, lo, hi in self.held():
            got = self.get(i, lo, hi)
            for name, x, y in zip(("master", "m", "v"), out, got):
                had = seen[lo:hi]
                assert torch.equal(x[lo:hi][had].view(torch.uint8), y[had].view(torch.uint8)), \
                    f"holders disagree on {name} over {(lo, hi)} (member {i})"
                x[lo:hi] = y
            seen[lo:hi] = True
        assert bool(seen.all())
        return out


def _bits(x):
    """bf16 tensor -> numpy uint16 bit patterns."""
    assert x.dtype == BF16
    return x.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def _widen(bits):
    return (bits.astype(np.uint32) << np.uint32(16)).view(np.float32)


def _random_moments(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = (torch.randn(NUMEL, device="cuda", generator=g) * 0.02).bfloat16()
    v = (torch.randn(NUMEL, device="cuda", generator=g) * 0.02).square().bfloat16()
    return m, v


def _assert_neighbour(stored, ref, slack, what):
    """``stored`` (bf16) is one of the two bf16 neighbours of some value within ``slack`` of the fp32 ``ref``. The kernel
    and the reference contract ``b * x + (1 - b) * y`` into FMAs differently, and the kernel takes ``1 - b`` in fp32 where
    the reference rounds the double, so the two fp32 moments differ by a few ulps of the larger addend (more than that
    many ulps of the result when the addends cancel)."""
    def towards(x, away):
        bits = x.contiguous().view(torch.int32)
        return ((bits + 0xFFFF if away else bits) & ~0xFFFF).view(torch.float32)

    lo_f, hi_f = ref - slack, ref + slack
    lo = torch.where(lo_f >= 0, towards(lo_f, False), towards(lo_f, True))  # the largest bf16 <= lo_f
    hi = torch.where(hi_f >= 0, towards(hi_f, True), towards(hi_f, False))  # the smallest bf16 >= hi_f
    s = stored.float()
    ok = (s >= lo) & (s <= hi)
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} stored moments are not a bf16 neighbour of the reference"


# ----------------------------------------------------------------------------- the rounding, bit for bit
@pytest.mark.parametrize("paged", [False, True])
def test_device_rounding_equals_the_numpy_specification(paged):
    """A zero gradient makes ``m' = fp32(b1 * m)`` and ``v' = fp32(b2 * v)`` single exactly rounded products."""
    from torchft_b200.parallel.zero1 import bf16_sr

    world = 4
    reps = MReplicas(world, k=2, compact=paged)
    reps.configure(list(range(world)), 1)
    reps.put(*_random_moments(1))
    zero = torch.zeros(NUMEL, dtype=BF16, device="cuda")
    seen_t = []
    for t0 in (0, 999):
        for o in reps.opts:
            o._set_t(t0)
        torch.cuda.synchronize()
        for _ in range(2):
            before = {(i, lo, hi): reps.get(i, lo, hi) for i, lo, hi in reps.held()}
            reps.step([[zero] * world], reduce=False)
            reps.settle()
            t = reps.opts[0].t
            seen_t.append(t)
            for (i, lo, hi), (_, m0, v0) in before.items():
                _, m1, v1 = reps.get(i, lo, hi)
                e = np.arange(lo, hi, dtype=np.uint64)
                want_m = bf16_sr(np.float32(B1) * _widen(_bits(m0)), e, t, 0)
                want_v = bf16_sr(np.float32(B2) * _widen(_bits(v0)), e, t, 1)
                assert (_bits(m1) == want_m).all(), f"m of member {i} over {(lo, hi)} at t={t}"
                assert (_bits(v1) == want_v).all(), f"v of member {i} over {(lo, hi)} at t={t}"
                assert (_bits(m1) != _bits(m0)).any()
    assert seen_t == [1, 2, 1000, 1001]


def test_device_rounding_hashes_the_full_64_bit_element_index():
    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import bf16_sr

    n, off, t = 8 * 1000, (1 << 33) + 8 * 3, 77
    c = SymmetricComm.virtual_world(1, {"z1_param": n * 2, "z1_grad": n * 2}, presignal=True)[0]
    g = torch.Generator(device="cuda").manual_seed(4)
    master = torch.randn(n, device="cuda", generator=g)
    m = torch.randn(n, device="cuda", generator=g).bfloat16()
    v = torch.randn(n, device="cuda", generator=g).square().bfloat16()
    m0, v0 = _bits(m), _bits(v)
    grad = torch.zeros(n, dtype=BF16, device="cuda")
    gate = torch.tensor([1, t], dtype=torch.int32, device="cuda")
    c.zero1_update_("z1_param", 0, grad.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), n, HP, gate, 1, 0, 4,
                    state_off=off, moment_dtype=BF16)
    torch.cuda.synchronize()
    e = np.arange(n, dtype=np.uint64) + np.uint64(off)
    assert (_bits(m) == bf16_sr(np.float32(B1) * _widen(m0), e, t, 0)).all()
    assert (_bits(v) == bf16_sr(np.float32(B2) * _widen(v0), e, t, 1)).all()
    assert (_bits(m) != bf16_sr(np.float32(B1) * _widen(m0), e - np.uint64(1 << 33), t, 0)).any()
    with pytest.raises(RuntimeError, match="16 B aligned"):
        c.zero1_update_("z1_param", 0, grad.data_ptr(), master.data_ptr(), m.data_ptr() + 2, v.data_ptr(), n - 8, HP,
                        gate, 1, 0, 4, moment_dtype=BF16)


# ----------------------------------------------------------------------------- one update against the fp32 reference
CASES = [(w, k) for w in (1, 2, 4, 8) for k in (1, 2) if k <= w]


@pytest.mark.parametrize("world,k", CASES)
def test_one_update_stores_a_neighbour_of_the_fp32_moment_and_the_fp32_weights(world, k):
    reps = MReplicas(world, k=k, compact=world in (2, 8))
    reps.configure(list(range(world)), 1)
    m0, v0 = _random_moments(10 * world + k)
    reps.put(m0, v0)
    raw = _raws(world, 5 * world + k)
    reps.step([raw])
    reps.settle()
    master, m, v = reps.init.float(), m0.float(), v0.float()
    g = _reduced(raw).float()
    ulp = 2.0 ** -21  # four fp32 ulps of the larger addend; a bf16 ulp is 2^13 times that
    slack_m = torch.maximum((B1 * m).abs(), ((1 - B1) * g).abs()) * ulp
    slack_v = torch.maximum(B2 * v, (1 - B2) * g * g) * ulp
    ref_adamw(master, m, v, g, 1)
    first = reps.opts[0]
    for i, lo, hi in reps.held():
        gm, gmm, gv = reps.get(i, lo, hi)
        # the weights come from the fp32 moments, before they are rounded: the tolerance of the fp32-moment update
        torch.testing.assert_close(gm, master[lo:hi], rtol=2e-5, atol=1e-7)
        _assert_neighbour(gmm, m[lo:hi], slack_m[lo:hi], "m")
        _assert_neighbour(gv, v[lo:hi], slack_v[lo:hi], "v")
        if k == 1:
            # with buddies, the pre-signalled virtual world lets a later member's refresh after the re-shard overwrite
            # weights an earlier holder has already updated (see test_zero1_sched_gpu._check); they heal at the next update
            assert torch.equal(reps.opts[i].param, first.param)
            assert torch.equal(first.param[lo:hi], gm.bfloat16())
    reps.full_state()  # holders agree
    assert all(o.t == 1 for o in reps.opts)


# ----------------------------------------------------------------------------- the same bits everywhere
def test_holders_grids_and_paging_give_the_same_bits_and_a_vetoed_step_leaves_every_byte():
    world = 4
    runs = {}
    for paged, blocks in ((False, 1), (False, 8), (True, 8), (True, 1)):
        reps = MReplicas(world, k=2, compact=paged, blocks=blocks)
        reps.configure(list(range(world)), 1)
        for step in range(5):
            raw = _raws(world, 40 + step)
            if step == 2:
                reps.settle()
                torch.cuda.synchronize()
                before = [[x.clone() for x in (o.master, o.m, o.v, o.param)] for o in reps.opts]
                _step_vetoed_by_all(reps, raw)
                reps.settle()
                for o, b in zip(reps.opts, before):
                    for x, y in zip((o.master, o.m, o.v, o.param), b):
                        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), "a vetoed step changed state"
                assert all(o.t == 2 for o in reps.opts)
            else:
                reps.step([raw])
        state = reps.full_state()  # asserts that the holders of every slice agree
        assert all(o.t == 4 for o in reps.opts)
        assert state[1].dtype == BF16 and state[2].dtype == BF16
        runs[(paged, blocks)] = state + [reps.opts[0].param.clone()]
    ref = runs[(False, 1)]
    for key, st in runs.items():
        for name, x, y in zip(("master", "m", "v", "param"), ref, st):
            assert torch.equal(x, y), f"{name} differs between flat state on one CTA and {key}"


# ----------------------------------------------------------------------------- a short run against fp32 moments
@pytest.mark.parametrize("extras", [False, True])
def test_thirty_steps_stay_close_to_fp32_moments(extras):
    """bf16 moments carry a relative error of about 2^-9 each, so one step's weight change is off by a fraction of a
    per cent of lr; over 32 steps the masters stay within lr * steps * 2^-5 = 1e-2 at the worst element and 1e-3 on
    average (the weights themselves move by up to lr * steps = 0.32)."""
    world, steps = 2, 32
    kw = dict(max_norm=2.0, lam=lambda i: min(1.0, (i + 1) / 8), lr_steps=8) if extras else {}
    out = {}
    for md in (FP32, BF16):
        reps = MReplicas(world, moments=md, k=2, **kw)
        reps.configure(list(range(world)), 1)
        for step in range(steps):
            reps.step([_raws(world, 300 + step)])
        out[md] = reps.full_state()
        assert all(o.t == steps for o in reps.opts)
    d = (out[FP32][0] - out[BF16][0]).abs()
    moved = (out[FP32][0] - reps.init.float()).abs()
    assert float(moved.mean()) > 0.003, "the run moved the weights"
    assert float(d.max()) < 1e-2 and float(d.mean()) < 1e-3, (float(d.max()), float(d.mean()))
    assert float(d.max()) > 0, "the two runs are not the same run"
    torch.testing.assert_close(out[BF16][2].float(), out[FP32][2], rtol=0.05, atol=1e-6)


# ----------------------------------------------------------------------------- kill, rejoin, re-shard
@pytest.mark.parametrize("compact", [False, True])
def test_kill_rejoin_and_reshard_move_bf16_moments_bit_for_bit(compact):
    world = 4
    pulled = {}
    for md in (BF16, FP32):
        reps = MReplicas(world, moments=md, k=2, compact=compact, min_world=3)
        reps.configure([0, 1, 2, 3], 1)
        for step in range(2):
            reps.step([_raws(4, 70 + step)])
        src = reps.full_state()
        reps.configure([0, 1, 3], 2)  # member 2 dies: its slices move to the survivors
        got = reps.full_state()
        for name, x, y in zip(("master", "m", "v"), src, got):
            assert torch.equal(x, y), f"{name} after the kill"
        reps.step([_raws(3, 80)])
        reps.settle()
        src = reps.full_state()
        o = reps.make(reps.comms[2])  # ... and restarts with nothing but the weights
        o.param.copy_(reps.opts[0].param)
        o.seed_master()
        reps.opts[2] = o
        reps.configure([0, 1, 2, 3], 3)
        got = reps.full_state()
        for name, x, y in zip(("master", "m", "v"), src, got):
            assert torch.equal(x, y), f"{name} after the rejoin"
        assert o.t == 3 and all(x.lost_elements == 0 for x in reps.opts)
        reps.step([_raws(4, 81)])
        reps.full_state()
        pulled[md] = [x.pulled_bytes for x in reps.opts]
        assert o.pulled_bytes == o._state_item() * sum(hi - lo for lo, hi in reps.layout().held(2, 4))
        assert o.state_bytes_held() == o._state_item() * sum(hi - lo for lo, hi in reps.layout().held(2, 4))
        assert o.state_bytes_allocated() == o._state_item() * o.master.numel()
    assert reps.opts[0]._state_item() == 12 and sum(pulled[BF16]) > 0
    assert [12 * b for b in pulled[BF16]] == [8 * f for f in pulled[FP32]], "8 bytes per pulled element instead of 12"


def test_mixed_moment_types_raise_on_every_rank_before_anything_moves():
    reps = MReplicas(3, moments=[BF16, FP32, BF16], compact=True)
    before = [(o.t, list(o._holdings)) for o in reps.opts]
    errs = _configure_errors(reps, [0, 1, 2], 1)
    assert sorted(errs) == [0, 1, 2]
    for e in errs.values():
        assert isinstance(e, RuntimeError) and "disagree on the type of the optimizer moments" in str(e)
    for o, (t, hold) in zip(reps.opts, before):
        assert o.pulled_bytes == 0 and o.t == t and o._holdings == hold and not o._configured


# ----------------------------------------------------------------------------- checkpoints
def _saved(tmp_path, md, world=4):
    live = MReplicas(world, moments=md, k=2)
    live.configure(list(range(world)), 1)
    for step in range(2):
        live.step([_raws(world, 90 + step)])
    state = live.full_state()
    for o in live.opts:
        assert o.save(str(tmp_path), {"step": o.t, "batches_committed": 0}) == 2
    for o in live.opts:
        o.wait_checkpoint()
    return live, state


@pytest.mark.parametrize("saved,restored", [(BF16, BF16), (FP32, BF16), (BF16, FP32)])
@pytest.mark.parametrize("compact", [False, True])
def test_restore_at_another_world_keeps_or_converts_the_moments(tmp_path, saved, restored, compact):
    live, (master, m, v) = _saved(tmp_path, saved)
    back = MReplicas(3, moments=restored, k=2, compact=compact, min_world=3)
    for o in back.opts:
        assert o.restore(str(tmp_path)) == {"step": 2, "batches_committed": 0} and o.t == 2
    back.configure([0, 1, 2], 1)
    gmaster, gm, gv = back.full_state()
    assert gm.dtype == restored and gv.dtype == restored
    assert torch.equal(gmaster, master)
    # same type: the file's bits; fp32 -> bf16: round to nearest; bf16 -> fp32: exact
    assert torch.equal(gm, m.to(restored)) and torch.equal(gv, v.to(restored))
    assert all(o.lost_elements == 0 for o in back.opts)
    back.step([_raws(3, 95)])
    back.full_state()
    assert all(o.t == 3 for o in back.opts)


def test_checkpoint_files_of_both_types_have_the_layout_their_header_names(tmp_path):
    from torchft_b200.checkpointing.sharded import read_header, sections

    for md, item in ((FP32, 4), (BF16, 2)):
        d = tmp_path / str(item)
        live, (master, m, v) = _saved(d, md)
        for r, o in enumerate(live.opts):
            path = os.path.join(d, f"z1_step_2.w4.r{r}.bin")
            h = read_header(path)
            n = h["elements"]
            assert ("moments" in h) == (md == BF16)
            assert h["sections"] == sections(n, item)
            if md == FP32:  # the layout fp32 files have always had, byte for byte
                assert h["sections"] == {"param": 0, "master": 2 * n, "m": 6 * n, "v": 10 * n}
            assert os.path.getsize(path) == h["data"] + (6 + 2 * item) * n
            assert o.snapshot_bytes() == (6 + 2 * item) * n
            raw = np.fromfile(path, dtype=np.uint8, offset=h["data"])
            for name, x in (("param", o.param), ("master", master), ("m", m), ("v", v)):
                want = torch.cat([x[lo:hi] for lo, hi, _ in h["ranges"]]).contiguous().view(torch.uint8).cpu().numpy()
                at = h["sections"][name]
                assert (raw[at:at + want.size] == want).all(), (name, r)


# ----------------------------------------------------------------------------- trainer
def _train(tag, steps=10, **kw):
    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    lh = local_lighthouse()
    tr = FaultTolerantTrainer("llama3_tiny", loopback(lh.address()), replica_id=f"z1mom_{tag}_0",
                              timeout=timedelta(seconds=30), lr=1e-3, **kw)
    try:
        gen = torch.Generator().manual_seed(5)
        tok = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
        tgt = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
        losses = [tr.step(tok, tgt) for _ in range(steps)]
        tr.manager.state_dict()
        tr.join()
        torch.cuda.synchronize()
        return {"loss": losses, "t": tr.zopt.t, "dtype": tr.zopt.m.dtype, "bytes": tr.zopt.state_bytes_allocated(),
                "numel": tr.zopt.numel, "master": tr.zopt.master.clone()}
    finally:
        tr.shutdown()
        lh.shutdown()


def test_trainer_with_bf16_moments_follows_the_fp32_trainer(monkeypatch):
    monkeypatch.delenv("TORCHFT_B200_Z1_MOMENTS", raising=False)
    a = _train("fp32")
    b = _train("bf16", moment_dtype=BF16)
    monkeypatch.setenv("TORCHFT_B200_Z1_MOMENTS", "bf16")
    c = _train("env")
    assert a["dtype"] == FP32 and b["dtype"] == BF16 and c["dtype"] == BF16
    assert a["t"] == b["t"] == c["t"] == 10
    assert a["bytes"] == 12 * a["numel"] and b["bytes"] == 8 * b["numel"]
    assert b["loss"] == c["loss"] and torch.equal(b["master"], c["master"]), "the rounding is a function of (e, t) alone"
    assert a["loss"][-1] < a["loss"][0], "the run learns its batch"
    torch.testing.assert_close(torch.tensor(b["loss"]), torch.tensor(a["loss"]), rtol=2e-2, atol=2e-2)


def test_trainer_refuses_a_moment_type_on_the_classic_pipeline():
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    for pipe in (dict(zero1=False), dict(backend="nccl")):
        with pytest.raises(ValueError, match="moment_dtype"):
            FaultTolerantTrainer("llama3_tiny", "unused:0", moment_dtype=BF16, **pipe)
