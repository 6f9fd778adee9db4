"""FT-ZeRO-1 global token mean on ONE GPU: the commit kernel's count exchange and the update it scales, against the CPU
specification (``token_mean_commit``) and fp32 AdamW on ``reduced(...) * coef``; the unanimous veto of mismatched
shapes; and the trainer against an fp64 gradient of the mean over every valid target of the step.

Ranks are emulated in-process with ``SymmetricComm.virtual_world``. In a pre-signalled world every flag reads "arrived"
but nothing is exchanged, so each step first writes every rank's published slot, which is what a peer's arrival
guarantees; the real-signalling runs exchange them for real."""

from __future__ import annotations

import math
import struct
from datetime import timedelta

import pytest
import torch

from _zero1_replicas import HP, NUMEL, UNITS, PG, raws, reduced, ref_adamw, trainer
from _zero1_state import State

pytestmark = pytest.mark.gpu

MAX_NORM = 50.0
SLOT = 32  # bytes of one published slot (n, rows, loss bits, pad)
C = 4096   # the row count c = B * S of one micro-batch in the kernel tests


def _world(n, presignal, state=False):
    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import GNORM_UNITS

    seg = {"z1_grad": NUMEL * 2, "z1_param": NUMEL * 2, "z1_gnorm": GNORM_UNITS * 8, "z1_tokmean": 2 * SLOT}
    if state:
        seg.update({x: NUMEL * 4 for x in ("z1_master", "z1_m", "z1_v")})
    return SymmetricComm.virtual_world(n, seg, presignal=presignal, timeout=timedelta(seconds=20))


def _publish(comm, parity, n, loss, rows):
    """Write a rank's published slot directly (pre-signalled worlds: what the peer's arrival would guarantee)."""
    words = torch.tensor(struct.unpack("<4q", struct.pack("<QQdQ", n, rows, loss, 0)), dtype=torch.int64)
    comm.segment("z1_tokmean")[parity * SLOT:(parity + 1) * SLOT].view(torch.int64).copy_(words)


def _counts(world, M, quiet, step):
    """Uneven valid-target counts per rank (one rank with none) and fp64 loss sums; the quiet rank publishes 0s."""
    rows = M * C
    n = [(rows * (r + 1 + step)) // (world + 2) for r in range(world)]
    if world > 1:
        n[world - 1] = 0  # a rank whose every target is ignored
    loss = [2.5 * x + 0.1 * (r + 1) / 3 for r, x in enumerate(n)]
    return n, loss, [rows] * world


def _partials_norm(gnorms, world):
    """The fp32 norm the commit kernel forms from the ranks' per-unit fp64 partials (unit order, then rank order)."""
    sq = 0.0
    for r in range(world):
        s = 0.0
        for x in gnorms[r][: len(UNITS)].tolist():
            s += x
        sq += s
    return float(torch.tensor(math.sqrt(sq), dtype=torch.float32))


def _pipeline(world, k, steps, clip, tm=True, presignal=True, quiet=None, counts=None, seed=1):
    """Reduce-scatter (``M = len(steps[i])`` micro-batches) -> commit -> update for every step on fresh ranks. Returns
    one record per step with every rank's verdict, veto reason, [norm, coef], [loss, f], N, weights and state, plus
    what the ranks published and their pre-factor norm."""
    from torchft_b200.parallel.zero1 import ShardLayout, accum_mode, accum_offsets

    dev = torch.device("cuda", 0)
    comms = _world(world, presignal)
    g = torch.Generator(device=dev).manual_seed(seed)
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    grads = [c.segment("z1_grad")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    params = [c.segment("z1_param")[: NUMEL * 2].view(torch.bfloat16) for c in comms]
    gnorm = [c.segment("z1_gnorm").view(torch.float64) for c in comms]
    state = [State.seeded(init, None, seed * 10 + r) for r in range(world)]
    for p in params:
        p.copy_(init)
    L = ShardLayout(tuple(UNITS), k)
    accs = []
    for r in range(world):
        offs, n = accum_offsets(L, r, world)
        accs.append((torch.full((n + 8,), float("nan"), device=dev), offs))
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    coef = [torch.zeros(2, dtype=torch.float32, device=dev) for _ in comms]
    outs = [torch.zeros(2, dtype=torch.float32, device=dev) for _ in comms]
    ncount = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in comms]
    streams = [torch.cuda.Stream(device=dev) for _ in comms]
    P = world - (1 if quiet is not None else 0)
    order = ([quiet] if quiet is not None else []) + [r for r in range(world) if r != quiet]
    # every step's inputs exist before the first launch: with real signalling the steps are enqueued back to back, and
    # a copy from host memory on a stream behind a waiting handshake would block the host
    data = []
    for step, micro in enumerate(steps):
        n, loss, rows = (counts or _counts)(world, len(micro), quiet, step)
        data.append({"M": len(micro), "rows": rows,
                     "n_dev": [torch.tensor([n[r]], dtype=torch.int64, device=dev) for r in range(world)],
                     "l_dev": [torch.tensor([loss[r]], dtype=torch.float64, device=dev) for r in range(world)],
                     "pub": [(0, 0.0, rows[r]) if r == quiet else (n[r], loss[r], rows[r]) for r in range(world)]})
    seqs = [{} for _ in steps]
    snaps = [[{} for _ in range(world)] for _ in steps]  # per step and rank: what the step left, copied on its stream

    def rs(step, r, m, s):
        M = data[step]["M"]
        mode = accum_mode(m, M)
        if world == 1 and not clip and mode == 0:
            return  # what Zero1Optimizer does: scale 1 at world 1 is nothing to launch
        acc, offs = accs[r]
        for u, (lo, hi) in enumerate(UNITS):
            comms[r].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0 / (P * M), r != quiet, k, 4, s,
                                           gnorm=gnorm[r].data_ptr() + 8 * u if clip and mode in (0, 3) else 0,
                                           acc=acc.data_ptr() + 4 * offs[u] if mode else 0, acc_mode=mode)

    def commit(step, r, s):
        d = data[step]
        kw = dict(gnorm="z1_gnorm", nunits=len(UNITS), max_norm=MAX_NORM) if clip else {}
        if tm:
            kw.update(tokens="z1_tokmean", slot=step % 2, n_valid=d["n_dev"][r], loss_sum=d["l_dev"][r],
                      rows=d["rows"][r], divisor=P * d["rows"][r], contribute=r != quiet, token_out=outs[r],
                      token_count=ncount[r])
        if clip or tm:
            kw["norm"] = coef[r]
        seqs[step][r] = comms[r].zero1_commit_(gates[r], True, True, s, **kw)

    def upd(r, s):
        cf = coef[r].data_ptr() + 4 if clip or tm else 0
        for lo, hi in UNITS:
            comms[r].zero1_update_("z1_param", lo * 2, grads[r].data_ptr() + lo * 2, nelem=hi - lo, hyper=HP,
                                   gate=gates[r], replication=k, mode=0, blocks=4, stream=s, coef=cf,
                                   **state[r].args(lo))

    def snap(step, r, *what):
        x = snaps[step][r]
        for name in what:
            x[name] = {"gnorm": lambda: gnorm[r][: len(UNITS)].clone(), "coef": coef[r].clone, "out": outs[r].clone,
                       "N": ncount[r].clone, "t": lambda: gates[r][1:].clone(), "params": params[r].clone}[name]()

    if presignal:
        for step, micro in enumerate(steps):
            for m, raw in enumerate(micro):
                for r in range(world):
                    grads[r].copy_(raw[r])
                if quiet is not None:
                    grads[quiet].zero_()
                torch.cuda.synchronize()
                for r in order:
                    rs(step, r, m, None)
            for r in range(world):
                snap(step, r, "gnorm")
                if tm:
                    _publish(comms[r], step % 2, *data[step]["pub"][r])
            torch.cuda.synchronize()
            for r in range(world):
                commit(step, r, None)
                snap(step, r, "coef", "out", "N", "t")
            for r in range(world):
                upd(r, None)
            for r in range(world):
                snap(step, r, "params")  # after every rank's update: the peers' pushes land in this rank's weights
            torch.cuda.synchronize()
            assert all(c.errored() is None for c in comms)
    else:
        # every step of every rank enqueued at once, no host synchronisation between steps: a fast rank's commit c + 1
        # may run while a slow peer's commit c still reads the slots (each rank's launches keep the trainer's order; its
        # gradient copy for step c + 1 follows its update of step c, behind that step's trailing handshakes)
        torch.cuda.synchronize()
        for step, micro in enumerate(steps):
            assert len(micro) == 1
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    grads[r].copy_(micro[0][r])
                    rs(step, r, 0, streams[r])
                    snap(step, r, "gnorm")
                    commit(step, r, streams[r])
                    snap(step, r, "coef", "out", "N", "t")
                    upd(r, streams[r])
                    snap(step, r, "params")  # behind the update's trailing handshake: every peer's pushes have landed
        torch.cuda.synchronize()
        assert all(c.errored() is None for c in comms)
    recs = []
    for step, d in enumerate(data):
        x = snaps[step]
        recs.append({"verdict": [comms[r].verdict(seqs[step][r]) for r in range(world)],
                     "reason": [comms[r].commit_reason(seqs[step][r]) for r in range(world)] if tm else None,
                     "t": [int(x[r]["t"]) for r in range(world)], "coef": [x[r]["coef"] for r in range(world)],
                     "out": [x[r]["out"] for r in range(world)], "N": [int(x[r]["N"]) for r in range(world)],
                     "pre_norm": _partials_norm([x[r]["gnorm"] for r in range(world)], world) if clip else None,
                     "pub": d["pub"], "rows": d["rows"], "P": P, "params": [x[r]["params"] for r in range(world)],
                     "state": [st.get(0, NUMEL) for st in state] if step == len(data) - 1 else None})
    return recs


def _check_against_spec(world, k, steps, recs, clip, quiet):
    from torchft_b200.parallel.zero1 import ShardLayout, token_mean_commit

    dev = torch.device("cuda", 0)
    L = ShardLayout(tuple(UNITS), k)
    g = torch.Generator(device=dev).manual_seed(1)
    init = (torch.randn(NUMEL, device=dev, generator=g) * 0.05).bfloat16()
    rm, rmm, rv = init.float(), torch.zeros(NUMEL, device=dev), torch.zeros(NUMEL, device=dev)
    fmax = 1.0  # the test_zero1_clip_gpu tolerances, whose absolute parts scale with the gradient: m with f, v with f^2
    for step, (micro, rec) in enumerate(zip(steps, recs), start=1):
        fmax = max(fmax, float(rec["coef"][0][1]))
        assert rec["verdict"] == [True] * world and rec["t"] == [step] * world, rec["verdict"]
        assert rec["reason"] == [0] * world
        for r in range(world):
            spec = token_mean_commit(rec["pub"], rec["rows"][r], rec["P"] * rec["rows"][r],
                                     MAX_NORM if clip else None, rec["pre_norm"], own=r)
            assert not spec["veto"]
            assert rec["N"][r] == spec["N"], (r, rec["N"], spec)
            assert float(rec["out"][r][1]) == spec["f"] and float(rec["out"][r][0]) == spec["loss"], (r, spec)
            assert float(rec["coef"][r][1]) == spec["coef"], (r, float(rec["coef"][r][1]), spec)
            if clip:
                assert float(rec["coef"][r][0]) == spec["norm"]
            for x in ("coef", "out"):
                assert torch.equal(rec[x][r], rec[x][0]), f"{x} bits of rank {r}, step {step}"
        cf = rec["coef"][0][1]
        ref_adamw(rm, rmm, rv, reduced(micro, quiet).float() * cf, step)
    last = recs[-1]
    for r in range(1, world):
        assert torch.equal(last["params"][0], last["params"][r]), "weights must be bit-identical across replicas"
    for r in range(world):
        master, m, v = last["state"][r]
        for lo, hi in L.primary(r, world):
            assert torch.equal(last["params"][0][lo:hi], master[lo:hi].bfloat16())
        for lo, hi in L.held(r, world):
            torch.testing.assert_close(master[lo:hi], rm[lo:hi], rtol=2e-5, atol=1e-7)
            torch.testing.assert_close(m[lo:hi], rmm[lo:hi], rtol=1e-5, atol=1e-7 * fmax)
            torch.testing.assert_close(v[lo:hi], rv[lo:hi], rtol=1e-5, atol=1e-9 * fmax ** 2)


CASES = [(w, k, clip, M) for w in (1, 2, 3, 4, 8) for k in (1, 2) if k <= w for clip in (False, True) for M in (1, 3)]


@pytest.mark.parametrize("world,k,clip,M", CASES)
def test_token_mean_pipeline_matches_the_specification(world, k, clip, M):
    quiet = 1 if world > 2 else None  # a healing rank: no gradient and no targets
    scales = (1.0, 0.01, 1.0)
    steps = [raws(world, 300 + 7 * world + k + M + s, (sc,) * M) for s, sc in enumerate(scales)]  # steps[i][m][r]
    recs = _pipeline(world, k, steps, clip, quiet=quiet)
    _check_against_spec(world, k, steps, recs, clip, quiet)
    assert any(float(r["out"][0][1]) != 1.0 for r in recs), "uneven counts make f differ from 1"


def test_real_signalling_exchanges_the_same_counts_and_weights():
    """W = 4 ranks on four streams, every step enqueued back to back with no host synchronisation between steps, so a
    rank's commit of step c + 1 may run while a peer's commit of step c still reads the slots: the slots travel for
    real, alternate every step, and give what the sequential run gives."""
    world, k = 4, 2
    steps = [[x] for x in raws(world, 41, (1.0, 0.01, 1.0, 1.0))]
    for clip in (False, True):
        seq = _pipeline(world, k, steps, clip)
        real = _pipeline(world, k, steps, clip, presignal=False)
        _check_against_spec(world, k, steps, real, clip, None)
        for a, b in zip(seq, real):
            for r in range(world):
                for x in ("coef", "out", "params"):
                    assert torch.equal(a[x][r], b[x][r]), (clip, x, r)


@pytest.mark.parametrize("clip", [False, True])
def test_full_counts_change_no_bit(clip):
    """N = P * M * c everywhere: f = 1, and weights, state and norm are those of the same steps without the mode."""
    from torchft_b200.parallel.zero1 import ShardLayout

    world, k = 4, 2
    steps = [[x] for x in raws(world, 9, (1.0, 0.01, 1.0))]
    on = _pipeline(world, k, steps, clip, counts=lambda w, M, q, s: ([M * C] * w, [1.5 * M * C] * w, [M * C] * w))
    off = _pipeline(world, k, steps, clip, tm=False)
    L = ShardLayout(tuple(UNITS), k)
    for a, b in zip(off, on):
        assert all(float(o[1]) == 1.0 and float(o[0]) == 1.5 for o in b["out"])
        for r in range(world):
            if clip:
                assert torch.equal(a["coef"][r], b["coef"][r]), "norm and coefficient"
            assert torch.equal(a["params"][r], b["params"][r])
    for r in range(world):  # the state is recorded after the last step
        for lo, hi in L.held(r, world):
            for x, y in zip(off[-1]["state"][r], on[-1]["state"][r]):
                assert torch.equal(x[lo:hi], y[lo:hi])


def test_mismatched_rows_veto_on_every_rank_and_are_counted():
    """Four Zero1Optimizers with real signalling; at step 2 replica 2 publishes another M * B * S. Every rank vetoes,
    the state stays, the host counts and logs it, and the next step commits."""
    from torchft_b200.parallel.zero1 import Zero1Optimizer

    world = 4
    dev = torch.device("cuda", 0)
    comms = _world(world, presignal=False, state=True)
    streams = [torch.cuda.Stream(device=dev) for _ in comms]
    opts = []
    for c, s in zip(comms, streams):
        with torch.cuda.stream(s):
            o = Zero1Optimizer(PG(c), NUMEL, units=UNITS, replication=2, blocks=4, lr=HP[0], betas=HP[1:3], eps=HP[3],
                               weight_decay=HP[4], compact=False, global_token_mean=True)
        o.bind_stream(s)
        opts.append(o)
    init = (torch.randn(NUMEL, device=dev, generator=torch.Generator(device=dev).manual_seed(2)) * 0.05).bfloat16()
    for o in opts:
        o.param.copy_(init)
        o.seed_master()
    torch.cuda.synchronize()
    steps = raws(world, 61, (1.0, 1.0, 1.0))
    pending, snaps = None, []
    for step, raw in enumerate(steps):
        if pending is not None:
            for o, sq in zip(opts, pending):
                o.resolved(o.wait(sq))
        for o, g in zip(opts, raw):
            o.grad.copy_(g)
        # made before the launches: a copy from host memory on a stream behind a waiting handshake would block the host
        ns = [torch.tensor(C // 2 + r, device=dev) for r in range(world)]
        ls = [torch.tensor(1.0 * r, dtype=torch.float64, device=dev) for r in range(world)]
        torch.cuda.synchronize()
        pending = []
        for r, (o, s) in enumerate(zip(opts, streams)):
            with torch.cuda.stream(s):
                for u in range(len(UNITS)):
                    o.reduce_scatter(u, 1.0 / world, True)
                rows = C + (8 if step == 1 and r == 2 else 0)
                # at step 2 replica 3 also heals: it publishes 0 targets, and its vetoed step reports its own mean
                o.publish_tokens(ns[r], ls[r], rows, world, not (step == 1 and r == 3))
                pending.append(o.enqueue(True))
                o.update()
        torch.cuda.synchronize()
        snaps.append([(o.param.clone(), o.master.clone(), o.m.clone(), o.v.clone()) for o in opts])
        verdicts = [o.comm.verdict(sq) for o, sq in zip(opts, pending)]
        assert all(o.comm.errored() is None for o in opts)
        assert verdicts == [step != 1] * world, (step, verdicts)
        assert [o.comm.commit_reason(sq) for o, sq in zip(opts, pending)] == [1 if step == 1 else 0] * world
        if step == 1:
            for before, after in zip(snaps[0], snaps[1]):
                for x, y in zip(before, after):
                    assert torch.equal(x, y), "a vetoed step changes nothing"
            for r, o in enumerate(opts):  # a vetoed step reports the rank's own mean
                assert float(o._tok_out[0]) == float(torch.tensor((1.0 * r) / (C // 2 + r), dtype=torch.float32))
    for o, sq in zip(opts, pending):
        o.resolved(o.wait(sq))
    for o in opts:
        assert o.row_mismatch_steps == 1 and o.t == 2
    assert all(torch.equal(o.param, opts[0].param) for o in opts)


# ----------------------------------------------------------------------------- the trainer
B, S, DOC = 2, 128, 32


def _docs(M, seed, vocab, half_ignored=True):
    """Packed documents of DOC tokens (each one's last target -100); micro-batch 0 also ignores the second half of
    every row, so the micro-batches' counts of valid targets differ by about a factor of 2."""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, vocab, (M * B, S), generator=g)
    tgt = torch.randint(0, vocab, (M * B, S), generator=g)
    tgt[:, DOC - 1::DOC] = -100
    if half_ignored:
        tgt[:B, S // 2:] = -100
    cu = torch.arange(0, M * B * S + 1, DOC, dtype=torch.int32)
    return tok, tgt, cu


def _reference(model, tok, tgt, cu, M, dtype):
    """fp64 (or eager bf16) loss and gradients of sum(l) / N over the M micro-batches: reference_loss of each
    micro-batch weighted by its count."""
    from torchft_b200.data import slice_cu_seqlens
    from torchft_b200.models.reference import reference_loss

    N = int((tgt != -100).sum())
    loss, grads = 0.0, {}
    for m in range(M):
        t, y = tok[m * B:(m + 1) * B].cuda(), tgt[m * B:(m + 1) * B].cuda()
        n = int((y != -100).sum())
        lm, gm = reference_loss(model, t, y, dtype=dtype, cu_seqlens=slice_cu_seqlens(cu, m * B * S, (m + 1) * B * S))
        loss += lm * n / N
        for name, g in gm.items():
            g = g.double() * (n / N)
            grads[name] = g if name not in grads else grads[name] + g
    return loss, grads


def _applied_gradient(tr):
    """The gradient the update applied: the reduced bf16 gradient in the buffer times the commit kernel's coefficient."""
    torch.cuda.synchronize()
    where = {id(p): o for p, o in zip(tr.flat.params, tr.flat.offsets)}
    cf = tr.zopt._clip[1].float() if tr.global_token_mean else 1.0
    return {n: (tr.flat.grad[where[id(p)]:where[id(p)] + p.numel()].view(p.shape).float() * cf)
            for n, p in tr.model.named_parameters()}


def _worst(applied, g64, g16):
    """The model tests' criteria (FACTOR, MEDIAN of test_model_nodes_gpu): the worst per-row ratio and the worst median
    row error over the eager one divided by MEDIAN, over every parameter; both at most 1 pass."""
    from _node_ref import row_ratios
    from test_model_nodes_gpu import FACTOR, MEDIAN

    worst_ratio, worst_med = 0.0, 0.0
    for name, g in applied.items():
        ratio, eg, eb = row_ratios(g, g64[name], g16[name], FACTOR[False])
        worst_ratio = max(worst_ratio, float(ratio.max()))
        worst_med = max(worst_med, float(eg.median() / eb.median()) / MEDIAN[False])
    return worst_ratio, worst_med


def _one_step(monkeypatch, tag, tm, M=2, seed=4):
    """One step of a fresh trainer on the masks of :func:`_docs`. Returns the reported loss, each micro-batch's own loss
    (sum / (B * S)) at the same weights, the fp64 and eager bf16 losses and gradients of sum(l) / N, the applied
    gradient and N."""
    from test_model_nodes_gpu import _deterministic_attention

    with trainer("llama3_debug", tag, grad_accum_steps=M, global_token_mean=tm) as tr:
        tok, tgt, cu = _docs(M, seed, tr.cfg.vocab_size)
        # the references attend through an explicit mask, which the flash kernel of the deterministic context lacks
        l64, g64 = _reference(tr.model, tok, tgt, cu, M, torch.float64)
        l16, g16 = _reference(tr.model, tok, tgt, cu, M, torch.bfloat16)
        with _deterministic_attention(monkeypatch):
            own = []
            if tm:
                with torch.no_grad():
                    for m in range(M):
                        own.append(float(tr.model(tok[m * B:(m + 1) * B].cuda(), tgt[m * B:(m + 1) * B].cuda(),
                                                  cu_seqlens=_slice(cu, m), count_valid=False)))
            loss = tr.step(tok.pin_memory(), tgt.pin_memory(), cu)
            tr.join()
            return loss, own, (l64, l16), _applied_gradient(tr), (g64, g16), int((tgt != -100).sum())


def _slice(cu, m):
    from torchft_b200.data import slice_cu_seqlens

    return slice_cu_seqlens(cu, m * B * S, (m + 1) * B * S)


def test_trainer_applies_the_gradient_of_the_global_token_mean(monkeypatch):
    loss, own, (l64, l16), applied, (g64, g16), N = _one_step(monkeypatch, "tm_on", True)
    ratio, med = _worst(applied, g64, g16)
    print(f"[token mean] worst row ratio {ratio:.3g}, worst median ratio {med:.3g} (limits 1)")
    assert ratio <= 1 and med <= 1, (ratio, med)
    # the loss: sum of each micro-batch's loss * c in fp64, over N; and the fp64 model's within the model tests' bound
    total = 0.0
    for x in own:
        total += x * (B * S)
    assert abs(loss - total / N) <= 1e-6 * abs(total / N), (loss, total / N)
    assert abs(loss - l64) <= 4 * abs(l16 - l64) + 2.0 ** -9 * abs(l64), (loss, l64, l16)
    # without the option the same step weights the half-masked micro-batch's targets twice as much
    _, _, _, applied_off, _, _ = _one_step(monkeypatch, "tm_off", False)
    ratio_off, med_off = _worst(applied_off, g64, g16)
    print(f"[token mean] without the option: worst row ratio {ratio_off:.3g}, worst median ratio {med_off:.3g}")
    assert ratio_off > 3 and med_off > 3, (ratio_off, med_off)


def test_trainer_without_ignored_targets_changes_no_bit(monkeypatch):
    from test_model_nodes_gpu import _deterministic_attention

    out = []
    for tm in (False, True):
        with _deterministic_attention(monkeypatch), trainer("llama3_debug", f"tm_full_{int(tm)}",
                                                            global_token_mean=tm) as tr:
            gen = torch.Generator().manual_seed(5)
            losses = []
            for _ in range(3):
                tok = torch.randint(0, tr.cfg.vocab_size, (B, S), generator=gen).pin_memory()
                tgt = torch.randint(0, tr.cfg.vocab_size, (B, S), generator=gen).pin_memory()
                losses.append(tr.step(tok, tgt))
            tr.join()
            torch.cuda.synchronize()
            out.append((losses, tr.zopt.param.clone(), tr.zopt.master.clone(), tr.zopt.m.clone(), tr.zopt.v.clone()))
    assert out[0][0] == out[1][0]
    for a, b in zip(out[0][1:], out[1][1:]):
        assert torch.equal(a, b)


def test_trainer_accumulation_matches_one_batch_of_all_rows(monkeypatch):
    """grad_accum_steps=2 over B rows each against one step over 2 B rows, both with the option, on the masks above.
    With the tolerances of the accumulation test this would also pass without the option (AdamW normalises a reweighting
    away after one step): what the option fixes is shown by the gradient test above and the two-process test below."""
    from test_model_nodes_gpu import _deterministic_attention

    res = []
    for M in (2, 1):
        with _deterministic_attention(monkeypatch), trainer("llama3_debug", f"tm_acc{M}", grad_accum_steps=M,
                                                            global_token_mean=True) as tr:
            losses = []
            for step in range(3):
                tok, tgt, cu = _docs(2, 10 + step, tr.cfg.vocab_size)
                losses.append(tr.step(tok.pin_memory(), tgt.pin_memory(), cu))
            tr.join()
            torch.cuda.synchronize()
            res.append((losses, tr.zopt.param.clone()))
    (l2, p2), (l1, p1) = res
    assert abs(l1[0] - l2[0]) <= 2e-3 * abs(l1[0]), (l1, l2)
    torch.testing.assert_close(torch.tensor(l1), torch.tensor(l2), rtol=5e-3, atol=5e-3)
    diff = (p1.float() - p2.float()).abs()
    assert float(diff.max()) <= 8e-3 and float((diff > 0).float().mean()) < 0.25, (float(diff.max()),
                                                                                  float((diff > 0).float().mean()))


def test_two_replicas_with_different_masks_take_the_step_of_one_replica_on_both(tmp_path):
    """Two trainers in two processes on a local lighthouse, each training one micro-batch of every step with its own
    mask, against one trainer that trains both micro-batches with grad_accum_steps=2 (``_token_mean_replica.py``).
    The W = 2 reduce and the M = 2 accumulator perform the same fp32 operations in the same order (kAccLast), the
    divisors P * M * c agree (2 * 1 * B S and 1 * 2 * B S), and each replica adds its fp64 loss sums in micro-batch
    order as the commit kernel adds the ranks in rank order. So after 3 steps the weights and the optimizer state are
    bit-identical, and so is every reported loss."""
    import json
    import os
    import subprocess
    import sys

    from torchft_b200.bench_utils import local_lighthouse, loopback

    steps = 3
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_token_mean_replica.py")
    pair, alone = local_lighthouse(min_replicas=2), local_lighthouse(min_replicas=1)
    try:
        runs = {"0": pair, "1": pair, "all": alone}
        procs = {r: subprocess.Popen([sys.executable, script, "--lighthouse", loopback(lh.address()), "--replica", r,
                                      "--steps", str(steps), "--out", str(tmp_path / f"{r}.json")],
                                     stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                 for r, lh in runs.items()}
        logs = {r: p.communicate(timeout=600)[0] for r, p in procs.items()}
        for r, p in procs.items():
            assert p.returncode == 0, (r, logs[r][-4000:])
    finally:
        pair.shutdown()
        alone.shutdown()
    out = {r: json.loads((tmp_path / f"{r}.json").read_text()) for r in runs}
    for r in runs:
        assert out[r]["t"] == steps and out[r]["row_mismatch_steps"] == 0, out
    assert out["0"]["losses"] == out["1"]["losses"] == out["all"]["losses"], out
    for name in ("param", "master", "m", "v"):
        assert out["0"][name] == out["1"][name] == out["all"][name], (name, out)
