"""FT-ZeRO-1 kernels on ONE GPU: a W-rank quorum is emulated in-process (``SymmetricComm.virtual_world``).

``presignal=True`` runs the ranks' kernels one after the other (exact W-rank result, profiler/sanitizer friendly);
``presignal=False`` launches them concurrently on W streams so the signal-pad protocol runs for real.
Reference for the numerics: plain PyTorch fp32 AdamW on the fp32-accumulated, bf16-rounded mean gradient.
"""

from __future__ import annotations

import pytest
import torch

from _zero1_replicas import HP, NUMEL, UNITS, kernel_world, reduced, ref_adamw, trainer
from _zero1_state import State

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world,k", [(2, 2), (3, 2), (8, 2), (8, 1), (4, 3)])
def test_reduce_scatter_commit_update_match_reference(world, k):
    from torchft_b200.parallel.zero1 import ShardLayout

    dev = torch.device("cuda", 0)
    comms = kernel_world(world)
    L = ShardLayout(tuple(UNITS), k)
    g = torch.Generator(device=dev).manual_seed(11)
    grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    params = [c.segment("z1_param")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    for p in params:
        p.copy_(init)
    state = [State.seeded(init) for _ in comms]
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    rm, rmm, rv = init.float(), torch.zeros(NUMEL, device=dev), torch.zeros(NUMEL, device=dev)
    quiet = 1 if world > 2 else None  # a healing / spare rank whose gradients must count as zeros
    contributors = world - (1 if quiet is not None else 0)

    for step in range(1, 4):
        raw = [(torch.randn(NUMEL, device=dev, generator=g) * (r + 1)).bfloat16() for r in range(world)]
        for r in range(world):
            grads[r].copy_(raw[r])
        if quiet is not None:
            grads[quiet].zero_()  # sequential emulation: the quiet rank's in-kernel zeroing must precede rank 0's reads
        red = reduced([raw], quiet)

        # one-kernel-at-a-time emulation: the quiet rank zeroes its buffer inside its kernel, which on real hardware
        # happens before anybody's push (barrier 1) -- so its kernel goes first here
        order = ([quiet] if quiet is not None else []) + [r for r in range(world) if r != quiet]
        for r in order:
            for lo, hi in UNITS:
                comms[r].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0 / contributors, r != quiet, k, 4)
        torch.cuda.synchronize()
        for r in range(world):
            for lo, hi in L.held(r, world):
                assert torch.equal(grads[r][lo:hi], red[lo:hi]), f"rank {r} held range [{lo},{hi}) step {step}"

        seqs = [c.zero1_commit_(gates[r], True, True) for r, c in enumerate(comms)]
        for r, c in enumerate(comms):
            for lo, hi in UNITS:
                c.zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP,
                                gate=gates[r], replication=k, mode=0, blocks=4, **state[r].args(lo))
        torch.cuda.synchronize()
        assert all(c.errored() is None for c in comms)
        assert all(c.verdict(s) is True for c, s in zip(comms, seqs))
        assert all(int(gt[0]) == 1 and int(gt[1]) == step for gt in gates)

        ref_adamw(rm, rmm, rv, red.float(), step)
        for r in range(1, world):
            assert torch.equal(params[0], params[r]), "weights must be bit-identical across replicas"
        # the bf16 weights are the rounded masters of their primary holders
        master = [st.master for st in state]
        for r in range(world):
            for lo, hi in L.primary(r, world):
                assert torch.equal(params[0][lo:hi], master[r][lo:hi].bfloat16())
            for lo, hi in L.held(r, world):
                torch.testing.assert_close(master[r][lo:hi], rm[lo:hi], rtol=2e-5, atol=1e-7)
                torch.testing.assert_close(state[r].m[lo:hi], rmm[lo:hi], rtol=1e-5, atol=1e-7)
                torch.testing.assert_close(state[r].v[lo:hi], rv[lo:hi], rtol=1e-5, atol=1e-9)
        # holders of the same slice computed bit-identical state
        for u in range(len(UNITS)):
            for s in range(world):
                lo, hi = L.slice_bounds(u, world, s)
                hs = L.holders(u, world, s)
                for h in hs[1:]:
                    assert torch.equal(master[hs[0]][lo:hi], master[h][lo:hi])


def test_gate_zero_skips_update_and_refresh_rebroadcasts_masters():
    dev = torch.device("cuda", 0)
    world, k = 4, 2
    comms = kernel_world(world)
    params = [c.segment("z1_param")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    state = [State.seeded(torch.full((NUMEL,), 1.5, device=dev)) for _ in comms]
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    for p, gr in zip(params, grads):
        p.fill_(9.0)
        gr.fill_(1.0)
    # a vetoed step: nothing may change
    for r, c in enumerate(comms):
        seq = c.zero1_commit_(gates[r], False, True)
        for lo, hi in UNITS:
            c.zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP, gate=gates[r],
                            replication=k, mode=0, blocks=4, **state[r].args(lo))
        torch.cuda.synchronize()
        assert c.verdict(seq) is False
    assert all(int(gt[0]) == 0 and int(gt[1]) == 0 for gt in gates)
    assert all(bool((p == 9.0).all()) for p in params) and all(bool((st.master == 1.5).all()) for st in state)
    # refresh (mode 1): ungated re-broadcast of bf16(master) of the primary slices, state untouched
    for r, c in enumerate(comms):
        for lo, hi in UNITS:
            c.zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP, gate=gates[r],
                            replication=k, mode=1, blocks=4, **state[r].args(lo))
    torch.cuda.synchronize()
    assert all(bool((p == 1.5).all()) for p in params) and all(bool((st.m == 0).all()) for st in state)


@pytest.mark.parametrize("world", [2, 8])
def test_commit_verdict_is_unanimous_with_real_signalling(world):
    """Concurrent launch on W streams (presignal off): one rank's veto must reach every rank's gate."""
    dev = torch.device("cuda", 0)
    comms = kernel_world(world, presignal=False)
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    streams = [torch.cuda.Stream(device=dev) for _ in comms]
    for veto in (None, world - 1, None):
        seqs = []
        for r, c in enumerate(comms):
            with torch.cuda.stream(streams[r]):
                seqs.append(c.zero1_commit_(gates[r], r != veto, True, streams[r]))
        torch.cuda.synchronize()
        want = veto is None
        assert [c.verdict(s) for c, s in zip(comms, seqs)] == [want] * world
        assert all(int(gt[0]) == int(want) for gt in gates)
        assert all(c.errored() is None for c in comms)
    assert all(int(gt[1]) == 2 for gt in gates)  # two committed steps


def test_concurrent_ranks_full_pipeline_in_one_process():
    """All W ranks' kernels in flight at once on W streams: real barriers, same result as the reference."""
    dev = torch.device("cuda", 0)
    world, k = 4, 2
    comms = kernel_world(world, presignal=False)
    g = torch.Generator(device=dev).manual_seed(5)
    grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    params = [c.segment("z1_param")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    raw = [torch.randn(NUMEL, device=dev, generator=g).bfloat16() for _ in comms]
    init = torch.randn(NUMEL, device=dev, generator=g).bfloat16()
    state = [State.seeded(init) for _ in comms]
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    for r in range(world):
        grads[r].copy_(raw[r])
        params[r].copy_(init)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=dev) for _ in comms]
    for r, c in enumerate(comms):
        s = streams[r]
        with torch.cuda.stream(s):
            for lo, hi in UNITS:
                c.zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0 / world, True, k, 2, s)
            c.zero1_commit_(gates[r], True, True, s)
            for lo, hi in UNITS:
                c.zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP,
                                gate=gates[r], replication=k, mode=0, blocks=2, stream=s, **state[r].args(lo))
    torch.cuda.synchronize()
    assert all(c.errored() is None for c in comms)
    rm, rmm, rv = init.float(), torch.zeros(NUMEL, device=dev), torch.zeros(NUMEL, device=dev)
    ref_adamw(rm, rmm, rv, reduced([raw]).float(), 1)
    for r in range(world):
        assert torch.equal(params[0], params[r])
    torch.testing.assert_close(params[0].float(), rm.bfloat16().float(), rtol=0, atol=2e-2)
    assert (params[0] != rm.bfloat16()).float().mean() < 1e-3  # at most a stray 1-ulp rounding difference


def test_trainer_zero1_matches_classic_adamw_at_world_one():
    out = []
    for zero1 in (False, True):
        with trainer("llama3_debug", f"z1eq_{int(zero1)}", bucket_mb=1.0, zero1=zero1) as tr:
            gen = torch.Generator().manual_seed(5)
            losses = []
            for _ in range(4):
                tok = torch.randint(0, tr.cfg.vocab_size, (2, 128), generator=gen).pin_memory()
                tgt = torch.randint(0, tr.cfg.vocab_size, (2, 128), generator=gen).pin_memory()
                losses.append(tr.step(tok, tgt))
            assert tr.manager.current_step() == 4
            sd = tr.state_dict()
            torch.cuda.synchronize()
            out.append((losses, sd["param"].clone()))
    (l0, p0), (l1, p1) = out
    # the same update rule with the same fp32 bias corrections (1 - b^t of the fp32 betas, rounded once) on both sides
    diff = (p0.float() - p1.float()).abs()
    assert torch.equal(p0, p1), (float(diff.max()), float((diff > 0).float().mean()))
    assert l0 == l1, (l0, l1)
