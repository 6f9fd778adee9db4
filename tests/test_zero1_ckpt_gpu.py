"""FT-ZeRO-1 durable checkpoints on ONE GPU: save under the next step, restore at another world and into compact state,
partial restarts next to a live replica, fallback and refusal on real files, and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (pre-signalled, see ``test_zero1_gpu.py``); every
rank launches on the current stream, the snapshot copies run on the optimizer's own stream.
"""

from __future__ import annotations

import os

import pytest
import torch

from _zero1_replicas import Replicas, raws, seeded_weights, trainer

pytestmark = pytest.mark.gpu

# large enough that the snapshot copy is still running when the next step's update is enqueued
UNITS = [(0, 8 * 131072), (8 * 131072, 8 * 131072 + 8 * 50021), (8 * 131072 + 8 * 50021, 8 * 131072 + 8 * 50028)]
NUMEL = UNITS[-1][1]
K = 2


def _step(reps, seed):
    """Gradients, reduce-scatters, verdicts and updates of one step are enqueued; nothing waits for the device."""
    reps.step(raws(len(reps.members), seed, (0.01,), NUMEL), sync=False)


def _state(reps):
    """(master, m, v) over the whole vector, assembled from the holders, and the weights."""
    return reps.full_state(), reps.opts[reps.members[0]].param.clone()


def _check_against(reps, ref, param):
    reps.settle()
    for i in reps.members:
        o = reps.opts[i]
        assert torch.equal(o.param, param), f"weights of member {i}"
        for (lo, hi), arrs in o.held_state().items():
            for name, a, r in zip(("master", "m", "v"), arrs, ref):
                assert torch.equal(a, r[lo:hi]), f"{name} of member {i} over {(lo, hi)}"


def _chain(world):
    """Quorums a live run of 4 goes through to reach ``world`` without losing state (k = 2)."""
    return {4: [[0, 1, 2, 3]], 3: [[0, 1, 2]], 1: [[0, 2], [0]]}[world]


@pytest.mark.parametrize("world,compact", [(4, False), (3, False), (1, False), (3, True)])
def test_save_under_the_next_step_and_restore_at_another_world(tmp_path, world, compact):
    live = Replicas(4, UNITS, k=K)
    live.configure([0, 1, 2, 3], 1)
    _step(live, 11)
    _step(live, 12)
    ref, param = _state(live)
    assert not torch.isnan(ref[0]).any()
    assert live.save(str(tmp_path)) == 2
    _step(live, 13)  # immediately: the update of each unit waits for that unit's snapshot copy, not for the host
    for o in live.opts:
        o.wait_checkpoint()
    live.settle()
    assert all(o.t == 3 for o in live.opts)
    assert sorted(os.listdir(tmp_path)) == [f"z1_step_2.w4.r{r}.bin" for r in range(4)]

    back = Replicas(world, UNITS, k=K, compact=compact, min_world=3 if compact else 1)
    for o in back.opts:
        o.master.fill_(float("nan"))  # a re-shard must fill every held element
        assert o.restore(str(tmp_path)) == {"step": 2, "batches_committed": 0}
        assert torch.equal(o.param, param) and o.t == 2
    back.configure(list(range(world)), 1)
    _check_against(back, ref, param)
    assert all(o.lost_elements == 0 for o in back.opts)
    assert sum(o.disk_read_elements for o in back.opts) == sum(
        sum(hi - lo for lo, hi in o.layout.held(r, world)) for r, o in enumerate(back.opts))

    # a live run that changed 4 -> world at T = 2 and the restored one agree bit for bit two steps later
    ctl = Replicas(4, UNITS, k=K)
    ctl.configure([0, 1, 2, 3], 1)
    _step(ctl, 11)
    _step(ctl, 12)
    for e, members in enumerate(_chain(world)):
        ctl.configure(members, 2 + e)
    for seed in (21, 22):
        _step(ctl, seed)
        _step(back, seed)
    st, p = _state(ctl)
    _check_against(back, st, p)
    assert all(o.t == 4 for o in back.opts) and all(ctl.opts[i].lost_elements == 0 for i in ctl.members)


def test_partial_restart_pulls_from_the_live_replica_and_reads_the_rest(tmp_path):
    from torchft_b200.parallel.zero1 import intersect_ranges, subtract_ranges, total

    live = Replicas(4, UNITS, k=K)
    live.configure([0, 1, 2, 3], 1)
    _step(live, 31)
    _step(live, 32)
    ref, param = _state(live)
    live.save(str(tmp_path))
    for o in live.opts:
        o.wait_checkpoint()
    for r in (1, 2, 3):  # these processes restart; member 0 stays alive at T = 2
        o = live.make(live.comms[r])
        o.param.zero_()
        for a in (o.master, o.m, o.v):
            a.fill_(float("nan"))
        assert o.restore(str(tmp_path))["step"] == 2
        live.opts[r] = o
    live.configure([0, 1, 2, 3], 2)
    _check_against(live, ref, param)
    L = live.opts[0].layout
    for r in (1, 2, 3):
        o = live.opts[r]
        assert o.pulled_bytes == 12 * total(intersect_ranges(L.held(r, 4), L.held(0, 4)))
        assert o.disk_read_elements == total(subtract_ranges(L.held(r, 4), L.held(0, 4))) > 0
        assert o.lost_elements == 0
    assert live.opts[0].pulled_bytes == 0 and live.opts[0].disk_read_elements == 0


def test_missing_and_torn_files_fall_back_and_a_mismatch_refuses(tmp_path):
    live = Replicas(2, UNITS, k=K)
    live.configure([0, 1], 1)
    _step(live, 41)
    live.save(str(tmp_path))
    _step(live, 42)
    live.save(str(tmp_path))
    _step(live, 43)
    live.save(str(tmp_path))  # keep = 2: step 1's files are pruned
    for o in live.opts:
        o.wait_checkpoint()
    _, p2 = _state(live)  # the weights of step 3
    assert sorted(os.listdir(tmp_path)) == [f"z1_step_{t}.w2.r{r}.bin" for t in (2, 3) for r in (0, 1)]

    def restore_one():
        o = Replicas(1, UNITS, k=K).opts[0]
        return o.restore(str(tmp_path)), o

    sd, o = restore_one()
    assert sd["step"] == 3 and torch.equal(o.param, p2)
    with open(tmp_path / "z1_step_3.w2.r1.bin", "r+b") as f:  # torn: step 3 is incomplete
        f.truncate(os.path.getsize(tmp_path / "z1_step_3.w2.r1.bin") // 2)
    sd, o = restore_one()
    assert sd["step"] == 2 and o.t == 2
    os.remove(tmp_path / "z1_step_2.w2.r0.bin")  # missing: nothing is complete
    sd, o = restore_one()
    assert sd is None and o.t == 0 and torch.equal(o.param, seeded_weights(NUMEL))
    # another unit split (as with another optimizer_blocks) refuses before touching anything
    other = Replicas(1, [(0, UNITS[1][0]), (UNITS[1][0], NUMEL)], k=K).opts[0]
    with pytest.raises(ValueError, match="units"):
        other.restore(str(tmp_path))
    assert other.t == 0 and torch.equal(other.param, seeded_weights(NUMEL))


# ----------------------------------------------------------------------------- trainer
def _batches(cfg, n):
    gen = torch.Generator().manual_seed(9)
    return [(torch.randint(0, cfg.vocab_size, (2, 128), generator=gen).pin_memory(),
             torch.randint(0, cfg.vocab_size, (2, 128), generator=gen).pin_memory()) for _ in range(n)]


def test_trainer_resumes_bit_identically_where_the_durable_checkpointer_route_does_not(tmp_path):
    from torchft_b200.checkpointing import DurableCheckpointer

    sharded, classic = str(tmp_path / "sharded"), str(tmp_path / "classic")
    with trainer("llama3_debug", "z1ckpt_a") as tr:
        data = _batches(tr.cfg, 5)
        for tok, tgt in data[:3]:
            tr.step(tok, tgt)
        assert tr.save_checkpoint(sharded) == 3
        dc = DurableCheckpointer(tr.manager, tr.state_dict, tr.load_state_dict, classic)
        assert dc.maybe_save(force=True)
        dc.wait()
        live = [tr.step(tok, tgt) for tok, tgt in data[3:]]
        tr.wait_checkpoint()
        with pytest.raises(RuntimeError, match="before the first step"):
            tr.restore_checkpoint(sharded)
        tr.join()
        p_live = tr.zopt.param.clone()
        assert tr.manager.current_step() == 5

    with trainer("llama3_debug", "z1ckpt_b") as tr:
        assert tr.restore_checkpoint(sharded) == 3
        assert tr.manager.current_step() == 3
        resumed = [tr.step(tok, tgt) for tok, tgt in data[3:]]
        tr.join()
        assert resumed == live
        assert torch.equal(tr.zopt.param, p_live)
        assert tr.manager.current_step() == 5 and tr.zopt.lost_elements == 0

    # the route this exists to replace: weights and t come back, master / m / v do not, so training continues from
    # the initial master weights with zero moments
    with trainer("llama3_debug", "z1ckpt_c") as tr:
        assert DurableCheckpointer(tr.manager, tr.state_dict, tr.load_state_dict, classic).restore() == 3
        for tok, tgt in data[3:]:
            tr.step(tok, tgt)
        tr.join()
        assert not torch.equal(tr.zopt.param, p_live)


def test_trainer_refusals(tmp_path):
    with trainer("llama3_debug", "z1ckpt_classic", zero1=False) as tr:
        with pytest.raises(ValueError, match="FT-ZeRO-1"):
            tr.save_checkpoint(str(tmp_path))
        with pytest.raises(ValueError, match="FT-ZeRO-1"):
            tr.restore_checkpoint(str(tmp_path))
    with trainer("llama3_debug", "z1ckpt_empty") as tr:
        assert tr.restore_checkpoint(str(tmp_path / "nothing")) is None
