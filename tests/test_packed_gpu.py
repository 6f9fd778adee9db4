"""Packed documents on the GPU: the RoPE kernel at document positions against fp64, the model's isolation of documents
bit for bit (forward and backward), the model against an fp64 eager reference with an explicit block-diagonal mask,
activation checkpointing, the trainer's three step entry points and its micro-batch cut, and mutants that the checks
must catch."""

import dataclasses

import pytest
import torch

from _fp64 import _WORST, U, assert_close_elementwise  # noqa: F401
from _node_ref import bits_equal, row_ratios
from test_model_nodes_gpu import FACTOR, MEDIAN, _deterministic_attention, _equal_steps, _model_cfg
from test_model_ops_gpu import _rot_ref, _table_ref

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _cu(v):
    return torch.tensor(v, dtype=torch.int32)


def _cuts(B, S, lengths):
    """cu_seqlens of rows filled in order with documents of the given lengths (cycled), cut at every row end."""
    out, i = [0], 0
    for r in range(B):
        t = 0
        while t < S:
            n = min(lengths[i % len(lengths)], S - t)
            i += 1
            t += n
            out.append(r * S + t)
    return _cu(out)


# ------------------------------------------------------------------------------------------------ 1. the RoPE kernel
LAYOUTS = {
    # 300 one-token documents, then documents of 1 and 2 tokens and longer ones
    "one-token": lambda B, S: _cuts(B, S, [1] * 300 + [2, 1, 517]),
    # every row is two documents whose second ends on the row end
    "row-end": lambda B, S: _cuts(B, S, [S // 3, S]),
    # lengths that are not multiples of 8, 64 or 128
    "odd": lambda B, S: _cuts(B, S, [7, 63, 127, 129, 1001, 65, 9, 255, 2047]),
    "one-per-row": lambda B, S: _cuts(B, S, [S]),
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("B,S", [(1, 8192), (2, 4096)])
def test_rope_qkv_at_document_positions(B, S, D, layout):
    """Forward and backward against the fp64 rotation at cs[position in document], within 1 ulp plus the fp32 table's
    own error; v and dv bit-exact; with cu_seqlens = the row starts, bit for bit the path without positions."""
    from torchft_b200.data import document_positions
    from torchft_b200.ops import fused

    Hq, Hkv, theta = 32, 8, 5e5
    T, row = B * S, (Hq + 2 * Hkv) * D
    cu = LAYOUTS[layout](B, S)
    pos_h = document_positions(cu)
    pos = pos_h.cuda()
    cs = fused.rope_table(S, D, theta, torch.device("cuda"))
    cs64 = _table_ref(S, D, theta)
    err = (cs.double() - cs64).abs().amax(-1)
    gen = torch.Generator(device="cuda").manual_seed(S + D + len(layout))
    qkv0 = torch.randn(T, row, device="cuda", generator=gen).to(BF16)
    qkv = qkv0.clone().requires_grad_()
    q, k, v = fused.rope_qkv(qkv, cs, B, S, Hq, Hkv, D, positions=pos)
    assert torch.equal(v.reshape(T, Hkv * D), qkv0[:, (Hq + Hkv) * D:])
    dq = torch.randn(B, Hq, S, D, device="cuda", generator=gen).to(BF16).transpose(1, 2)
    dk = torch.randn(B, Hkv, S, D, device="cuda", generator=gen).to(BF16).transpose(1, 2)
    dv = torch.randn(B, Hkv, S, D, device="cuda", generator=gen).to(BF16).transpose(1, 2)
    torch.autograd.backward([q, k, v], [dq, dk, dv])
    dqkv = qkv.grad
    assert torch.equal(dqkv[:, (Hq + Hkv) * D:].view(B, S, Hkv, D), dv)
    qf, kf = q.reshape(T, Hq, D), k.reshape(T, Hkv, D)
    dqf, dkf = dq.reshape(T, Hq, D), dk.reshape(T, Hkv, D)
    tag = f"B={B} S={S} D={D} {layout}"
    for lo in range(0, T, 2048):
        hi = min(T, lo + 2048)
        p = pos[lo:hi].long()
        c64, e = cs64[p], err[p]
        packed = qkv0[lo:hi].view(hi - lo, Hq + 2 * Hkv, D)
        for name, got, x in (("q", qf[lo:hi], packed[:, :Hq]), ("k", kf[lo:hi], packed[:, Hq:Hq + Hkv])):
            ref, sl = _rot_ref(x, c64, e, 1.0)
            assert_close_elementwise(got, ref, ulps=1, abs_slack=sl, what=f"packed rope {name} {tag}")
        dpk = dqkv[lo:hi].view(hi - lo, Hq + 2 * Hkv, D)
        for name, got, g in (("dq", dpk[:, :Hq], dqf[lo:hi]), ("dk", dpk[:, Hq:Hq + Hkv], dkf[lo:hi])):
            ref, sl = _rot_ref(g, c64, e, -1.0)
            assert_close_elementwise(got, ref, ulps=1, abs_slack=sl, what=f"packed rope {name} {tag}")
    if layout == "one-per-row":
        plain = qkv0.clone().requires_grad_()
        q2, k2, v2 = fused.rope_qkv(plain, cs, B, S, Hq, Hkv, D)
        torch.autograd.backward([q2, k2, v2], [dq, dk, dv])
        for what, a, b in (("q", q, q2), ("k", k, k2), ("v", v, v2), ("dqkv", dqkv, plain.grad)):
            bits_equal(a, b, f"rope {what} {tag}: positions = row offsets vs no positions")
    _WORST.clear()


# ------------------------------------------------------------------------------------- varlen attention on this card
@pytest.mark.parametrize("D", [64, 128])
def test_varlen_attention_takes_gqa_and_the_strided_v_deterministically(D, monkeypatch):
    """The library's variable-length flash kernel takes 32 query heads over 8 KV heads and v as the strided view of the
    packed projection; its backward runs under deterministic algorithms and repeats bit for bit; at one document per row
    it is SDPA's causal attention up to rounding."""
    from torch.nn.attention.varlen import varlen_attn

    Hq, Hkv, B, S = 32, 8, 2, 2048
    T = B * S
    gen = torch.Generator(device="cuda").manual_seed(D)
    qkv = torch.randn(T, (Hq + 2 * Hkv) * D, device="cuda", generator=gen).to(BF16)
    do = torch.randn(T, Hq, D, device="cuda", generator=gen).to(BF16)
    cu = torch.tensor([0, S, 2 * S], dtype=torch.int32, device="cuda")

    def run():
        leaf = qkv.clone().requires_grad_()
        q = leaf[:, :Hq * D].view(T, Hq, D)
        k = leaf[:, Hq * D:(Hq + Hkv) * D].view(T, Hkv, D)
        v = leaf[:, (Hq + Hkv) * D:].view(T, Hkv, D)
        assert not v.is_contiguous()
        o = varlen_attn(q, k, v, cu, cu, S, S, window_size=(-1, 0))
        o.backward(do)
        return o.detach(), leaf.grad

    with _deterministic_attention(monkeypatch):
        o1, g1 = run()
        o2, g2 = run()
    bits_equal(o1, o2, f"varlen D={D}: two forwards")
    bits_equal(g1, g2, f"varlen D={D}: two deterministic backwards")
    leaf = qkv.clone().requires_grad_()
    sp = leaf.view(B, S, Hq + 2 * Hkv, D).transpose(1, 2)
    o = torch.nn.functional.scaled_dot_product_attention(sp[:, :Hq], sp[:, Hq:Hq + Hkv], sp[:, Hq + Hkv:],
                                                         is_causal=True, enable_gqa=True)
    o.transpose(1, 2).reshape(T, Hq, D).backward(do)
    o = o.transpose(1, 2).reshape(T, Hq, D).float()
    assert float((o1.float() - o).abs().max()) < 2e-2 * float(o.abs().max())
    assert float((g1.float() - leaf.grad.float()).abs().max()) < 5e-2 * float(leaf.grad.float().abs().max())


# -------------------------------------------------------------------------------------------- 2. isolation, forward
ISO = {"llama3_debug": (2, 512), "1b-2layer": (1, 2048)}


def _model(cfg):
    from torchft_b200.models.llama import Llama

    m = Llama(cfg, device="cuda")
    m.init_weights(0)
    return m


def _logits_and_losses(m, tok, tgt, cu):
    from torchft_b200.ops import fused

    with torch.no_grad():
        logits = m(tok, cu_seqlens=cu)
        V = logits.shape[-1]
        losses = fused.cross_entropy_inplace(logits.reshape(-1, V).clone(), tgt.reshape(-1))
    return logits.reshape(-1, V), losses


def _iso_layout(B, S):
    # row 0: documents 100, 37, 260, rest; other rows: two documents each
    cut = [0, 100, 137, 397, S] + [r * S + c for r in range(1, B) for c in (S // 2 - 11, S)]
    return _cu(cut)


def check_forward_isolation(name):
    """Changing the other documents' tokens leaves a document's logits and per-token losses unchanged, bit for bit."""
    cfg = _model_cfg(name)
    B, S = ISO[name]
    m = _model(cfg)
    cu = _iso_layout(B, S)
    gen = torch.Generator(device="cuda").manual_seed(21)
    tok = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=gen)
    tgt = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=gen)
    a, b = 137, 397  # the document under test
    tok2 = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=gen)
    tok2.view(-1)[a:b] = tok.view(-1)[a:b]
    la, sa = _logits_and_losses(m, tok, tgt, cu)
    lb, sb = _logits_and_losses(m, tok2, tgt, cu)
    bits_equal(la[a:b], lb[a:b], f"{name}: logits of a document whose neighbours changed")
    bits_equal(sa[a:b], sb[a:b], f"{name}: per-token losses of a document whose neighbours changed")
    assert not torch.equal(la[:a], lb[:a])


def check_forward_move(name, shift):
    """The same document at another offset of the row (same B*S) gives bit-identical logits."""
    cfg = _model_cfg(name)
    B, S = ISO[name]
    m = _model(cfg)
    L, a1 = min(300, S // 4), 100
    a2 = a1 + shift
    gen = torch.Generator(device="cuda").manual_seed(22)
    doc = torch.randint(0, cfg.vocab_size, (L,), device="cuda", generator=gen)
    out = []
    for a in (a1, a2):
        tok = torch.randint(0, cfg.vocab_size, (B, S), device="cuda", generator=gen)
        tok.view(-1)[a:a + L] = doc
        cu = _cu([0, a, a + L, S] + [r * S for r in range(2, B + 1)])
        logits, _ = _logits_and_losses(m, tok, torch.zeros_like(tok), cu)
        out.append(logits[a:a + L])
    bits_equal(out[0], out[1], f"{name}: logits of a document moved by {shift} tokens")


@pytest.mark.parametrize("name", list(ISO))
def test_forward_isolation_bit_for_bit(name):
    check_forward_isolation(name)


@pytest.mark.parametrize("shift", [256, 211])
@pytest.mark.parametrize("name", list(ISO))
def test_forward_moved_document_bit_for_bit(name, shift):
    check_forward_move(name, shift)


# ------------------------------------------------------------------------------------------- 3. isolation, backward
def check_backward_isolation(name, fp8=False):
    """Every other document's targets -100: every parameter gradient is unchanged, bit for bit, when the other
    documents' tokens change. The other documents draw from the upper half of the vocabulary and the document from the
    lower, so no embedding row is shared between them (the deterministic embedding backward sums a row's tokens in
    groups whose boundaries move when other tokens of the same id come and go)."""
    cfg = _model_cfg(name, fp8_linears=fp8)
    B, S = ISO[name]
    cu = _iso_layout(B, S)
    a, b = 137, 397
    V2 = cfg.vocab_size // 2
    gen = torch.Generator(device="cuda").manual_seed(23)
    doc = torch.randint(0, V2, (b - a,), device="cuda", generator=gen)
    tgt = torch.full((B, S), -100, dtype=torch.int64, device="cuda")
    tgt.view(-1)[a:b - 1] = doc[1:]
    steps = []
    for _ in range(2):
        tok = torch.randint(V2, cfg.vocab_size, (B, S), device="cuda", generator=gen)
        tok.view(-1)[a:b] = doc
        m = _model(cfg)
        loss = m(tok, tgt, cu_seqlens=cu)
        loss.backward()
        steps.append((loss.detach(), {n: p.grad for n, p in m.named_parameters()}))
    _equal_steps(steps[0], steps[1], f"{name} fp8={fp8}: other documents' tokens changed")


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name", list(ISO))
def test_backward_isolation_bit_for_bit(name, fp8, monkeypatch):
    with _deterministic_attention(monkeypatch):
        check_backward_isolation(name, fp8)


# ----------------------------------------------------------------------------------------------- 4./5. against fp64
def _packed_batch(cfg, B, S, seed):
    """Documents with log-uniform lengths from 1 to S, packed by data.pack_documents."""
    from torchft_b200.data import pack_documents

    g = torch.Generator().manual_seed(seed)
    docs = []
    while sum(len(d) for d in docs) < B * S:
        n = int(torch.exp(torch.rand((), generator=g) * torch.log(torch.tensor(float(S)))).item())
        docs.append(torch.randint(0, cfg.vocab_size, (max(n, 1),), generator=g).tolist())
    tok, tgt, cu = next(pack_documents(docs, B, S))
    return tok.cuda(), tgt.cuda(), cu


def check_against_fp64(cfg, tok, tgt, cu, ref_cu, tag):
    """test_model_rows_against_fp64's rule, with the model packed by ``cu`` and the references by ``ref_cu``."""
    from torchft_b200.models.reference import reference_loss
    from _node_ref import fp8_linear

    fp8 = cfg.fp8_linears
    m = _model(cfg)
    loss = m(tok, tgt, cu_seqlens=cu)
    loss.backward()
    lin = fp8_linear if fp8 else None
    l16, g16 = reference_loss(m, tok, tgt, dtype=torch.bfloat16, linear=lin, cu_seqlens=ref_cu)
    l64, g64 = reference_loss(m, tok, tgt, dtype=torch.float64, linear=lin, cu_seqlens=ref_cu)
    lr = abs(loss.item() - l64) / (FACTOR[fp8] * abs(l16 - l64) + 2.0 ** -9 * abs(l64))
    print(f"[packed rows] {tag} loss {loss.item():.9g} r64 {l64:.9g} b16 {l16:.9g} ratio {lr:.3g}")
    bad = []
    for pname, p in m.named_parameters():
        ratio, eg, eb = row_ratios(p.grad, g64[pname], g16[pname], FACTOR[fp8])
        i = int(ratio.argmax())
        med = float(eg.median() / eb.median())
        print(f"[packed rows] {tag} {pname}: worst row {i} ratio {float(ratio[i]):.3g}, median {med:.3g}")
        if float(ratio[i]) > 1 or med > MEDIAN[fp8]:
            bad.append((pname, i, float(ratio[i]), med))
        del g64[pname], g16[pname]
    assert lr <= 1, (tag, "loss", lr)
    assert not bad, (tag, bad)
    return loss.detach(), {n: p.grad for n, p in m.named_parameters()}


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name", list(ISO))
def test_packed_model_rows_against_fp64(name, fp8):
    cfg = _model_cfg(name, fp8_linears=fp8)
    tok, tgt, cu = _packed_batch(cfg, *ISO[name], seed=31)
    assert cu.numel() > 4
    check_against_fp64(cfg, tok, tgt, cu, cu, f"{name} fp8={fp8} documents={cu.numel() - 1}")


@pytest.mark.parametrize("name", list(ISO))
def test_one_document_per_row_matches_the_unpacked_step(name):
    """cu_seqlens = the row starts, against the unpacked fp64 reference by the same rule, on the batch that
    test_model_rows_against_fp64 judges the unpacked step on; bit equality with the unpacked step is reported, not
    required (the variable-length flash kernels round differently)."""
    from test_model_nodes_gpu import _batch, _step

    cfg = _model_cfg(name)
    B, S = ISO[name]
    tok, tgt = _batch(cfg, B, S, seed=17)
    packed = check_against_fp64(cfg, tok, tgt, _cu([r * S for r in range(B + 1)]), None, f"{name} one per row")
    plain = _step(cfg, tok, tgt)
    same = torch.equal(packed[0], plain[0]) and all(torch.equal(packed[1][n], plain[1][n]) for n in plain[1])
    print(f"[packed rows] {name}: one document per row bit-identical to the unpacked step: {same}")


# ------------------------------------------------------------------------------------- 6. activation checkpointing
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name", list(ISO))
def test_activation_checkpointing_changes_no_bit_of_a_packed_step(name, fp8, monkeypatch):
    cfg = _model_cfg(name, fp8_linears=fp8)
    tok, tgt, cu = _packed_batch(cfg, *ISO[name], seed=33)

    def step(c):
        m = _model(c)
        loss = m(tok, tgt, cu_seqlens=cu)
        loss.backward()
        return loss.detach(), {n: p.grad for n, p in m.named_parameters()}

    with _deterministic_attention(monkeypatch):
        ref = step(cfg)
        _equal_steps(step(cfg), ref, f"{name} fp8={fp8} packed: two runs")
        _equal_steps(step(dataclasses.replace(cfg, activation_checkpoint="full")), ref, f"{name} fp8={fp8} packed: ckpt")


# ---------------------------------------------------------------------------------------------------- 7. trainer
def _trainer_batches(vocab, n=3, B=2, S=256):
    g = torch.Generator().manual_seed(41)
    out = []
    for i in range(n):
        tok = torch.randint(0, vocab, (B, S), generator=g)
        cu = _cuts(B, S, [[37, 100, 5], [S], [1, 80, 300]][i])
        tgt = torch.randint(0, vocab, (B, S), generator=g)
        tgt.view(-1)[cu[1:].long() - 1] = -100
        out.append((tok.pin_memory(), tgt.pin_memory(), cu))
    return out


def test_trainer_packed_steps_through_every_entry_point(monkeypatch):
    """Three FT-ZeRO-1 steps of packed batches through step, step_async and step_device: all commit, with the same
    losses and the same parameter buffer, bit for bit."""
    from _zero1_replicas import trainer

    batches = _trainer_batches(2048)
    out = {}
    with _deterministic_attention(monkeypatch):
        for how in ("step", "step_async", "step_device"):
            with trainer("llama3_debug", f"packed_{how}", seed=0) as tr:
                losses = []
                for tok, tgt, cu in batches:
                    if how == "step":
                        losses.append(tr.step(tok, tgt, cu))
                    elif how == "step_async":
                        prev = tr.step_async(tok, tgt, cu)
                        if prev is not None:
                            losses.append(prev)
                    else:
                        losses.append(float(tr.step_device(tok.cuda(), tgt.cuda(), cu_seqlens=cu).item()))
                if how == "step_async":
                    losses.append(tr.last_loss())
                assert tr.manager.current_step() == 3
                tr.join()
                torch.cuda.synchronize()
                out[how] = (losses, tr.state_dict()["param"].clone())
    for how in ("step_async", "step_device"):
        assert out[how][0] == out["step"][0], (how, out[how][0], out["step"][0])
        bits_equal(out[how][1], out["step"][1], f"packed {how} vs step: parameter buffer after 3 steps")


def _accum_batch(vocab, S=128):
    """(4, S) packed: micro-batch 0 (rows 0-1) and micro-batch 1 (rows 2-3) with different layouts and the same number
    of documents, hence the same number of valid targets."""
    g = torch.Generator().manual_seed(42)
    tok = torch.randint(0, vocab, (4, S), generator=g)
    tgt = torch.randint(0, vocab, (4, S), generator=g)
    c0 = [0, 10, 50, S, S + 70, 2 * S]
    c1 = [0, 100, S, S + 1, S + 30, 2 * S]
    cu = _cu(c0 + [2 * S + c for c in c1[1:]])
    tgt.view(-1)[cu[1:].long() - 1] = -100
    assert int((tgt[:2] != -100).sum()) == int((tgt[2:] != -100).sum())
    return tok.pin_memory(), tgt.pin_memory(), cu


def _train_packed(M, tag, steps=3):
    from _zero1_replicas import trainer

    with trainer("llama3_debug", f"packed_acc_{tag}", grad_accum_steps=M) as tr:
        tok, tgt, cu = _accum_batch(tr.cfg.vocab_size)
        losses = [tr.step(tok, tgt, cu) for _ in range(steps)]
        assert tr.manager.current_step() == steps
        tr.join()
        torch.cuda.synchronize()
        return losses, tr.state_dict()["param"].clone()


def check_accumulation(tag):
    """grad_accum_steps=2 over a packed (2B, S) batch matches M = 1, with the tolerances of
    test_trainer_accumulating_two_micro_batches_matches_one_batch."""
    l1, p1 = _train_packed(1, f"{tag}1")
    l2, p2 = _train_packed(2, f"{tag}2")
    assert abs(l1[0] - l2[0]) <= 2e-3 * abs(l1[0]), (l1, l2)
    torch.testing.assert_close(torch.tensor(l1), torch.tensor(l2), rtol=5e-3, atol=5e-3)
    diff = (p1.float() - p2.float()).abs()
    assert float(diff.max()) <= 8e-3 and float((diff > 0).float().mean()) < 0.25, (float(diff.max()),
                                                                                 float((diff > 0).float().mean()))


def test_trainer_accumulating_packed_micro_batches_matches_one_batch():
    check_accumulation("ok")


def test_trainer_refuses_a_malformed_description_before_any_launch():
    from _zero1_replicas import trainer

    with trainer("llama3_debug", "packed_bad", grad_accum_steps=2) as tr:
        tok, tgt, cu = _accum_batch(tr.cfg.vocab_size)
        with pytest.raises(ValueError, match="row start"):
            tr.step(tok, tgt, _cu([0, 10, 2 * 128 + 5, 4 * 128]))


# ---------------------------------------------------------------------------------------------------- 8. mutants
def test_mutant_positions_as_row_offsets(monkeypatch):
    """RoPE at t - b*S instead of the position in the document: moving a document changes its logits."""
    from torchft_b200.ops import fused

    real = fused.rope_qkv
    monkeypatch.setattr(fused, "rope_qkv", lambda *a, positions=None, **k: real(*a, **k))
    with pytest.raises(AssertionError, match="moved"):
        check_forward_move("llama3_debug", 256)


def test_mutant_attention_as_row_causal_sdpa(monkeypatch):
    """Attention causal over the whole row: the other documents' tokens reach a document's logits."""
    from torchft_b200.models import llama

    B = ISO["llama3_debug"][0]

    def row_causal(q, k, v, cu, cu_k, max_q, max_k, window_size):
        T, H, D = q.shape
        sd = [t.reshape(B, T // B, t.shape[1], D).transpose(1, 2) for t in (q, k, v)]
        o = torch.nn.functional.scaled_dot_product_attention(*sd, is_causal=True, enable_gqa=True)
        return o.transpose(1, 2).reshape(T, H, D)

    monkeypatch.setattr(llama, "varlen_attn", row_causal)
    with pytest.raises(AssertionError, match="neighbours changed"):
        check_forward_isolation("llama3_debug")


def test_mutant_cu_seqlens_not_rebased_per_micro_batch(monkeypatch):
    """The second micro-batch handed the unsliced offsets: the model refuses it (it does not start at 0)."""
    from torchft_b200.parallel import trainer as trainer_mod

    monkeypatch.setattr(trainer_mod, "slice_cu_seqlens",
                        lambda cu, lo, hi: cu[(cu >= lo) & (cu <= hi)].to(torch.int32))
    with pytest.raises(ValueError, match="start at 0"):
        check_accumulation("mutant")
