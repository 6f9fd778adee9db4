"""FT-ZeRO-1 global gradient-norm clipping on ONE GPU: the reduce / commit / update kernels with clipping against a
PyTorch reference, the unanimous veto of a non-finite step, compact state, ``Zero1Optimizer`` and the trainer.

Ranks are emulated in-process with ``SymmetricComm.virtual_world`` (see ``test_zero1_gpu.py``). Reference: fp32 AdamW
on ``reduced.float() * coef``, where ``reduced`` is the fp32-accumulated, bf16-rounded mean gradient, ``norm`` its L2
norm in fp64 and ``coef = min(1, max_norm / (norm + 1e-6))`` in fp32, as ``torch.nn.utils.clip_grad_norm_`` computes it.
"""

from __future__ import annotations

import pytest
import torch

from _zero1_replicas import HP, NUMEL, SHIFT, UNITS, Replicas, kernel_world, raws, reduced, ref_adamw, trainer
from _zero1_state import State

pytestmark = pytest.mark.gpu

MAX_NORM = 50.0
STEP_SCALES = (1.0, 0.01, 1.0)  # norms of a few hundred, a few units, a few hundred: clipped, not clipped, clipped


def _coef(max_norm, norm):
    """torch's clip coefficient in fp32 from an fp32 norm tensor."""
    return torch.clamp(max_norm / (norm + 1e-6), max=1.0)


def _pipeline(world, k, steps, max_norm, presignal=True, quiet=None, paged=False, seed=1):
    """Reduce-scatter -> commit -> update for every step of ``steps`` (``steps[step][rank]``) on fresh ranks, with
    clipping when ``max_norm`` is not None. Returns one record per step: verdicts, step counts, the [norm, coef] pair and
    the host-ring norm of every rank, and the weights and (full-size) state of every rank after the step."""
    dev = torch.device("cuda", 0)
    comms = kernel_world(world, presignal)
    g = torch.Generator(device=dev).manual_seed(seed)
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    params = [c.segment("z1_param")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    gnorm = [c.segment("z1_gnorm").data_ptr() for c in comms]
    state = [State.seeded(init, SHIFT if paged else None, seed * 10 + r) for r in range(world)]
    for p in params:
        p.copy_(init)
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    clip = [torch.zeros(2, dtype=torch.float32, device=dev) for _ in comms]
    streams = [torch.cuda.Stream(device=dev) for _ in comms]
    contributors = world - (1 if quiet is not None else 0)
    order = ([quiet] if quiet is not None else []) + [r for r in range(world) if r != quiet]
    seqs = {}

    def rs(r, s):
        for u, (lo, hi) in enumerate(UNITS):
            comms[r].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0 / contributors, r != quiet, k, 4, s,
                                           gnorm=gnorm[r] + 8 * u if max_norm is not None else 0)

    def commit(r, s):
        kw = {} if max_norm is None else dict(gnorm="z1_gnorm", nunits=len(UNITS), max_norm=max_norm, norm=clip[r])
        seqs[r] = comms[r].zero1_commit_(gates[r], True, True, s, **kw)

    def upd(r, s):
        coef = clip[r].data_ptr() + 4 if max_norm is not None else 0
        for lo, hi in UNITS:
            comms[r].zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP,
                                   gate=gates[r], replication=k, mode=0, blocks=4, stream=s, coef=coef,
                                   **state[r].args(lo))

    out = []
    for raw in steps:
        for r in range(world):
            grads[r].copy_(raw[r])
        if presignal and quiet is not None:
            grads[quiet].zero_()  # sequential emulation: the quiet rank's zeroing must precede everybody's reads
        torch.cuda.synchronize()
        if presignal:
            for r in order:
                rs(r, None)
            for r in range(world):
                commit(r, None)
            for r in range(world):
                upd(r, None)
        else:
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    rs(r, streams[r])
                    commit(r, streams[r])
                    upd(r, streams[r])
        torch.cuda.synchronize()
        assert all(c.errored() is None for c in comms)
        out.append({"verdict": [comms[r].verdict(seqs[r]) for r in range(world)],
                    "t": [int(gt[1]) for gt in gates],
                    "clip": [c.clone() for c in clip],
                    "host_norm": [comms[r].grad_norm(seqs[r]) if max_norm is not None else None for r in range(world)],
                    "params": [p.clone() for p in params],
                    "state": [st.get(0, NUMEL) for st in state]})
    return out


# ----------------------------------------------------------------------------- kernels vs the reference
@pytest.mark.parametrize("world,k", [(w, k) for w in (2, 3, 4, 8) for k in (1, 2, 3) if k <= w])
def test_clipped_pipeline_matches_reference(world, k):
    from torchft_b200.parallel.zero1 import ShardLayout

    dev = torch.device("cuda", 0)
    L = ShardLayout(tuple(UNITS), k)
    quiet = 1 if world > 2 else None  # a healing / spare rank whose gradients count as zeros
    steps = raws(world, 100 + world * 3 + k, STEP_SCALES)
    recs = _pipeline(world, k, steps, MAX_NORM, quiet=quiet)
    g = torch.Generator(device=dev).manual_seed(1)  # the seeded initial weights of _pipeline
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    rm, rmm, rv = init.float(), torch.zeros(NUMEL, device=dev), torch.zeros(NUMEL, device=dev)
    clipped = []
    for step, (raw, rec) in enumerate(zip(steps, recs), start=1):
        red = reduced([raw], quiet)
        norm = float(red.double().norm())
        for r in range(world):
            assert torch.equal(rec["clip"][r], rec["clip"][0]), f"norm / coef bits of rank {r}, step {step}"
            assert rec["host_norm"][r] == float(rec["clip"][0][0])
        dev_norm = rec["clip"][0][0]
        assert abs(float(dev_norm) - norm) <= 1e-5 * norm, (float(dev_norm), norm)
        assert torch.equal(rec["clip"][0][1], _coef(MAX_NORM, dev_norm)), "coef = min(1, max_norm / (norm + 1e-6))"
        coef = _coef(MAX_NORM, torch.tensor(norm, dtype=torch.float32, device=dev))
        clipped.append(bool(coef < 1))
        assert rec["verdict"] == [True] * world and rec["t"] == [step] * world
        ref_adamw(rm, rmm, rv, red.float() * coef, step)
    assert any(clipped) and not all(clipped), clipped
    last = recs[-1]
    for r in range(1, world):
        assert torch.equal(last["params"][0], last["params"][r]), "weights must be bit-identical across replicas"
    for r in range(world):
        master, m, v = last["state"][r]
        for lo, hi in L.primary(r, world):
            assert torch.equal(last["params"][0][lo:hi], master[lo:hi].bfloat16())
        for lo, hi in L.held(r, world):
            torch.testing.assert_close(master[lo:hi], rm[lo:hi], rtol=2e-5, atol=1e-7)
            torch.testing.assert_close(m[lo:hi], rmm[lo:hi], rtol=1e-5, atol=1e-7)
            torch.testing.assert_close(v[lo:hi], rv[lo:hi], rtol=1e-5, atol=1e-9)
    for u in range(len(UNITS)):
        for s in range(world):
            lo, hi = L.slice_bounds(u, world, s)
            hs = L.holders(u, world, s)
            for h in hs[1:]:
                for a, b in zip(last["state"][hs[0]], last["state"][h]):
                    assert torch.equal(a[lo:hi], b[lo:hi]), f"holders {hs} of unit {u} slice {s}"


@pytest.mark.parametrize("world,k", [(2, 2), (4, 2)])
def test_infinite_max_norm_changes_nothing(world, k):
    """max_norm = inf computes the norm but never scales: weights and state equal a run without clipping, bit for bit."""
    from torchft_b200.parallel.zero1 import ShardLayout

    L = ShardLayout(tuple(UNITS), k)
    quiet = 1 if world > 2 else None
    steps = raws(world, 7 + world, STEP_SCALES)
    off = _pipeline(world, k, steps, None, quiet=quiet)
    inf = _pipeline(world, k, steps, float("inf"), quiet=quiet)
    for a, b in zip(off, inf):
        assert all(float(c[1]) == 1.0 for c in b["clip"])
        for r in range(world):
            assert torch.equal(a["params"][r], b["params"][r])
            for lo, hi in L.held(r, world):
                for x, y in zip(a["state"][r], b["state"][r]):
                    assert torch.equal(x[lo:hi], y[lo:hi])


def test_real_signalling_gives_the_same_norm_bits_and_weights():
    """W = 4 ranks in flight at once on four streams against the pre-signalled sequential run."""
    world, k = 4, 2
    steps = raws(world, 21, STEP_SCALES)
    seq = _pipeline(world, k, steps, MAX_NORM)
    real = _pipeline(world, k, steps, MAX_NORM, presignal=False)
    for a, b in zip(seq, real):
        assert b["verdict"] == [True] * world
        for r in range(world):
            assert torch.equal(a["clip"][r], b["clip"][r])
            assert torch.equal(a["params"][r], b["params"][r])


@pytest.mark.parametrize("poison", ["inf", "nan"])
def test_nonfinite_gradient_vetoes_the_step_on_every_rank(poison):
    world, k = 4, 2
    steps = raws(world, 33, scales=(1.0, 1.0, 1.0))
    lo, hi = UNITS[1]
    steps[1][2][lo + 100] = float(poison)  # one element of one unit of one rank's raw gradient, step 2
    recs = _pipeline(world, k, steps, MAX_NORM, presignal=False)
    before, bad, after = recs
    assert before["verdict"] == [True] * world and before["t"] == [1] * world
    assert bad["verdict"] == [False] * world, "the veto must reach every rank"
    assert bad["t"] == [1] * world, "t must not advance"
    for r in range(world):
        norm = float(bad["clip"][r][0])
        assert (norm == float("inf")) if poison == "inf" else (norm != norm)
        assert torch.equal(bad["params"][r], before["params"][r])
        for x, y in zip(bad["state"][r], before["state"][r]):
            assert torch.equal(x, y)
    assert after["verdict"] == [True] * world and after["t"] == [2] * world


@pytest.mark.parametrize("world", [2, 4, 8])
def test_paged_update_with_clipping_matches_flat(world):
    k = 2
    steps = raws(world, 50 + world, STEP_SCALES)
    flat = _pipeline(world, k, steps, MAX_NORM, seed=4)
    paged = _pipeline(world, k, steps, MAX_NORM, paged=True, seed=4)
    _check_paged_vs_flat(world, k, flat, paged)


def _check_paged_vs_flat(world, k, flat, paged):
    from torchft_b200.parallel.zero1 import ShardLayout

    L = ShardLayout(tuple(UNITS), k)
    for step, (a, b) in enumerate(zip(flat, paged)):
        for r in range(world):
            assert torch.equal(a["clip"][r], b["clip"][r])
            assert torch.equal(a["params"][r], b["params"][r]), f"weights of rank {r}, step {step}"
            for lo, hi in L.held(r, world):
                for name, x, y in zip(("master", "m", "v"), a["state"][r], b["state"][r]):
                    assert torch.equal(x[lo:hi], y[lo:hi]), f"{name} of rank {r} on [{lo}, {hi}), step {step}"


# ----------------------------------------------------------------------------- Zero1Optimizer
def test_optimizer_reports_norms_one_step_late_and_counts_nonfinite_steps():
    """Through enqueue / update / wait / resolved in the Manager's order: a step's verdict (and norm) is settled when
    the next step starts."""
    world = 4
    opts = Replicas(world, max_grad_norm=MAX_NORM).opts
    steps = raws(world, 77, scales=(1.0, 0.01, 1.0, 1.0, 1.0))
    steps[2][3][UNITS[0][0] + 5] = float("inf")  # step 3 is poisoned
    norms, pending = [], None
    for step, raw in enumerate(steps):
        if pending is not None:  # the Manager books the previous step at the start of this one
            for o, s in zip(opts, pending):
                o.resolved(o.wait(s))
            for o in opts:
                assert o.last_grad_norm == norms[-1]
        for o, g in zip(opts, raw):
            o.grad.copy_(g)
        torch.cuda.synchronize()
        for o in opts:
            for u in range(len(UNITS)):
                o.reduce_scatter(u, 1.0 / world, True)
        pending = [o.enqueue(True) for o in opts]
        for o in opts:
            o.update()
        torch.cuda.synchronize()
        ref = float(reduced([raw]).double().norm())
        dev_norm = float(opts[0].grad_norm)
        assert dev_norm == ref == float("inf") if step == 2 else abs(dev_norm - ref) <= 1e-5 * ref, (step, dev_norm, ref)
        norms.append(dev_norm)
        assert all(torch.equal(o.grad_norm, opts[0].grad_norm) for o in opts)
    for o, s in zip(opts, pending):
        o.resolved(o.wait(s))
    for o in opts:
        assert o.last_grad_norm == norms[-1]
        assert o.nonfinite_steps == 1
        assert o.t == len(steps) - 1  # the poisoned step was not applied
    assert all(torch.equal(o.param, opts[0].param) for o in opts)


def test_optimizer_at_world_one_scales_in_place_and_norms_the_whole_buffer():
    opts = Replicas(1, max_grad_norm=1.0).opts
    o = opts[0]
    dev = torch.device("cuda", 0)
    raw = torch.randn(NUMEL, device=dev, generator=torch.Generator(device=dev).manual_seed(9)).bfloat16()
    o.grad.copy_(raw)
    for u in range(len(UNITS)):
        o.reduce_scatter(u, 0.5, True)
    seq = o.enqueue(True)
    o.update()
    o.resolved(o.wait(seq))
    reduced = (raw.float() * 0.5).bfloat16()
    assert torch.equal(o.grad, reduced), "the world-1 reduce launch scales in place like grad.mul_(scale)"
    norm = float(reduced.double().norm())
    assert abs(o.last_grad_norm - norm) <= 1e-5 * norm
    assert o.t == 1 and o.nonfinite_steps == 0
    assert float(o._clip[1]) == float(_coef(1.0, o._clip[0]))


# ----------------------------------------------------------------------------- trainer
def _train(max_grad_norm, steps=4, tag="a", read_grad=False):
    with trainer("llama3_debug", f"z1clip_{tag}", max_grad_norm=max_grad_norm) as tr:
        gen = torch.Generator().manual_seed(5)
        losses, reported, grad_norms = [], [], []
        for _ in range(steps):
            tok = torch.randint(0, tr.cfg.vocab_size, (2, 128), generator=gen).pin_memory()
            tgt = torch.randint(0, tr.cfg.vocab_size, (2, 128), generator=gen).pin_memory()
            losses.append(tr.step(tok, tgt))
            reported.append(tr.last_grad_norm())
            if read_grad:
                torch.cuda.synchronize()
                grad_norms.append(float(tr.flat.grad.double().norm()))
        tr.join()
        torch.cuda.synchronize()
        return losses, tr.state_dict()["param"].clone(), reported, grad_norms


def test_trainer_with_infinite_max_norm_reproduces_the_trainer_without_clipping():
    l0, p0, r0, _ = _train(None, tag="off")
    l1, p1, r1, _ = _train(float("inf"), tag="inf")
    assert l0 == l1
    assert torch.equal(p0, p1)
    assert all(x is None for x in r0) and all(x is not None for x in r1[1:])


def test_trainer_reports_the_norm_of_the_reduced_gradient_deterministically():
    la, pa, ra, ga = _train(0.05, steps=5, tag="c1", read_grad=True)
    lb, pb, rb, _ = _train(0.05, steps=5, tag="c2")
    # step n resolves step n - 1's verdict: the norm reported after step n is that of step n - 1's gradient
    for n in range(1, 5):
        assert abs(ra[n] - ga[n - 1]) <= 1e-5 * ga[n - 1], (n, ra[n], ga[n - 1])
    assert ga[0] > 0.05  # the threshold really clips
    assert ra == rb and la == lb and torch.equal(pa, pb), "two fresh trainers with the same seed: identical norm bits"


def test_trainer_refuses_clipping_on_the_classic_pipeline():
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    with pytest.raises(ValueError, match="max_grad_norm"):
        FaultTolerantTrainer("llama3_debug", "unused:0", zero1=False, max_grad_norm=1.0)
