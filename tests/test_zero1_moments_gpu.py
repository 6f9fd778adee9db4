"""FT-ZeRO-1 bf16 moments on ONE GPU: the device rounding against its numpy specification bit for bit, one update against
the fp32 reference, bit-identical holders at any grid and paging through a vetoed step, thirty steps against fp32
moments, kill / rejoin / re-shard, the agreement check, checkpoints across moment types, and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (see ``_zero1_replicas.py``).
"""

from __future__ import annotations

import os

import numpy as np
import pytest
import torch

from _zero1_replicas import HP, NUMEL, Replicas, bits, raws, reduced, ref_adamw, trainer, widen
from _zero1_state import State

pytestmark = pytest.mark.gpu

LR, B1, B2, EPS, WD = HP
BF16, FP32 = torch.bfloat16, torch.float32


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
    reps = Replicas(world, k=2, compact=paged, moment_dtype=BF16)
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
                want_m = bf16_sr(np.float32(B1) * widen(bits(m0)), e, t, 0)
                want_v = bf16_sr(np.float32(B2) * widen(bits(v0)), e, t, 1)
                assert (bits(m1) == want_m).all(), f"m of member {i} over {(lo, hi)} at t={t}"
                assert (bits(v1) == want_v).all(), f"v of member {i} over {(lo, hi)} at t={t}"
                assert (bits(m1) != bits(m0)).any()
    assert seen_t == [1, 2, 1000, 1001]


def test_device_rounding_hashes_the_full_64_bit_element_index():
    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import bf16_sr

    n, off, t = 8 * 1000, (1 << 33) + 8 * 3, 77
    c = SymmetricComm.virtual_world(1, {"z1_param": n * 2, "z1_grad": n * 2}, presignal=True)[0]
    g = torch.Generator(device="cuda").manual_seed(4)
    st = State(n, [(0, n)], None, off, "bf16", 0)
    st.put(0, n, torch.randn(n, device="cuda", generator=g), torch.randn(n, device="cuda", generator=g).bfloat16(),
           torch.randn(n, device="cuda", generator=g).square().bfloat16())
    m, v = st.m, st.v
    m0, v0 = bits(m), bits(v)
    grad = torch.zeros(n, dtype=BF16, device="cuda")
    gate = torch.tensor([1, t], dtype=torch.int32, device="cuda")
    c.zero1_update_("z1_param", 0, grad.data_ptr(), nelem=n, hyper=HP, gate=gate, replication=1, mode=0, blocks=4,
                    **st.args())
    torch.cuda.synchronize()
    e = np.arange(n, dtype=np.uint64) + np.uint64(off)
    assert (bits(m) == bf16_sr(np.float32(B1) * widen(m0), e, t, 0)).all()
    assert (bits(v) == bf16_sr(np.float32(B2) * widen(v0), e, t, 1)).all()
    assert (bits(m) != bf16_sr(np.float32(B1) * widen(m0), e - np.uint64(1 << 33), t, 0)).any()
    with pytest.raises(RuntimeError, match="16 B aligned"):
        c.zero1_update_("z1_param", 0, grad.data_ptr(), nelem=n - 8, hyper=HP, gate=gate, replication=1, mode=0,
                        blocks=4, **{**st.args(), "m": st.m.data_ptr() + 2})


# ----------------------------------------------------------------------------- one update against the fp32 reference
CASES = [(w, k) for w in (1, 2, 4, 8) for k in (1, 2) if k <= w]


@pytest.mark.parametrize("world,k", CASES)
def test_one_update_stores_a_neighbour_of_the_fp32_moment_and_the_fp32_weights(world, k):
    reps = Replicas(world, k=k, compact=world in (2, 8), moment_dtype=BF16)
    reps.configure(list(range(world)), 1)
    m0, v0 = _random_moments(10 * world + k)
    reps.put(m0, v0)
    rs = raws(world, 5 * world + k)
    reps.step(rs)
    reps.settle()
    master, m, v = reps.init.float(), m0.float(), v0.float()
    g = reduced(rs).float()
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
        reps = Replicas(world, k=2, blocks=blocks, compact=paged, moment_dtype=BF16)
        reps.configure(list(range(world)), 1)
        for step in range(5):
            rs = raws(world, 40 + step)
            if step == 2:
                reps.settle()
                torch.cuda.synchronize()
                before = [[x.clone() for x in (o.master, o.m, o.v, o.param)] for o in reps.opts]
                reps.step_vetoed_by_all(rs)
                reps.settle()
                for o, b in zip(reps.opts, before):
                    for x, y in zip((o.master, o.m, o.v, o.param), b):
                        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), "a vetoed step changed state"
                assert all(o.t == 2 for o in reps.opts)
            else:
                reps.step(rs)
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
    kw = dict(max_grad_norm=2.0, lr_lambda=lambda i: min(1.0, (i + 1) / 8), lr_steps=8) if extras else {}
    out = {}
    for md in (FP32, BF16):
        reps = Replicas(world, k=2, moment_dtype=md, **kw)
        reps.configure(list(range(world)), 1)
        for step in range(steps):
            reps.step(raws(world, 300 + step))
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
        reps = Replicas(world, k=2, compact=compact, min_world=3, moment_dtype=md)
        reps.configure([0, 1, 2, 3], 1)
        for step in range(2):
            reps.step(raws(4, 70 + step))
        src = reps.full_state()
        reps.configure([0, 1, 3], 2)  # member 2 dies: its slices move to the survivors
        got = reps.full_state()
        for name, x, y in zip(("master", "m", "v"), src, got):
            assert torch.equal(x, y), f"{name} after the kill"
        reps.step(raws(3, 80))
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
        reps.step(raws(4, 81))
        reps.full_state()
        pulled[md] = [x.pulled_bytes for x in reps.opts]
        assert o.pulled_bytes == o._state_item() * sum(hi - lo for lo, hi in reps.layout().held(2, 4))
        assert o.state_bytes_held() == o._state_item() * sum(hi - lo for lo, hi in reps.layout().held(2, 4))
        assert o.state_bytes_allocated() == o._state_item() * o.master.numel()
    assert reps.opts[0]._state_item() == 12 and sum(pulled[BF16]) > 0
    assert [12 * b for b in pulled[BF16]] == [8 * f for f in pulled[FP32]], "8 bytes per pulled element instead of 12"


def test_mixed_moment_types_raise_on_every_rank_before_anything_moves():
    reps = Replicas(3, compact=True, moment_dtype=[BF16, FP32, BF16])
    before = [(o.t, list(o._holdings)) for o in reps.opts]
    errs = reps.configure_errors([0, 1, 2], 1)
    assert sorted(errs) == [0, 1, 2]
    for e in errs.values():
        assert isinstance(e, RuntimeError) and "disagree on the type of the optimizer moments" in str(e)
    for o, (t, hold) in zip(reps.opts, before):
        assert o.pulled_bytes == 0 and o.t == t and o._holdings == hold and not o._configured


# ----------------------------------------------------------------------------- checkpoints
def _saved(tmp_path, md, world=4):
    live = Replicas(world, k=2, moment_dtype=md)
    live.configure(list(range(world)), 1)
    for step in range(2):
        live.step(raws(world, 90 + step))
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
    back = Replicas(3, k=2, compact=compact, min_world=3, moment_dtype=restored)
    for o in back.opts:
        assert o.restore(str(tmp_path)) == {"step": 2, "batches_committed": 0} and o.t == 2
    back.configure([0, 1, 2], 1)
    gmaster, gm, gv = back.full_state()
    assert gm.dtype == restored and gv.dtype == restored
    assert torch.equal(gmaster, master)
    # same type: the file's bits; fp32 -> bf16: round to nearest; bf16 -> fp32: exact
    assert torch.equal(gm, m.to(restored)) and torch.equal(gv, v.to(restored))
    assert all(o.lost_elements == 0 for o in back.opts)
    back.step(raws(3, 95))
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
    with trainer("llama3_tiny", f"z1mom_{tag}", lr=1e-3, **kw) as tr:
        gen = torch.Generator().manual_seed(5)
        tok = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
        tgt = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=gen).pin_memory()
        losses = [tr.step(tok, tgt) for _ in range(steps)]
        tr.manager.state_dict()
        tr.join()
        torch.cuda.synchronize()
        return {"loss": losses, "t": tr.zopt.t, "dtype": tr.zopt.m.dtype, "bytes": tr.zopt.state_bytes_allocated(),
                "numel": tr.zopt.numel, "master": tr.zopt.master.clone()}


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
