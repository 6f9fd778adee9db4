"""Packed documents on the host: ``data.pack_documents``, the ``cu_seqlens`` rules of ``data.check_cu_seqlens``, the
position table and the per-micro-batch slice, and the eager reference's document mask. No GPU."""

import dataclasses

import numpy as np
import pytest
import torch

from torchft_b200.data import check_cu_seqlens, document_positions, pack_documents, slice_cu_seqlens


def _docs(seed, n, lo=1, hi=40, vocab=1000):
    g = np.random.default_rng(seed)
    return [g.integers(0, vocab, size=int(g.integers(lo, hi + 1))).tolist() for _ in range(n)]


def _pieces(tok, tgt, cu):
    """(tokens, targets) of every document of a packed batch, in order."""
    t, y, c = tok.reshape(-1).tolist(), tgt.reshape(-1).tolist(), cu.tolist()
    return [(t[a:b], y[a:b]) for a, b in zip(c, c[1:])]


# ------------------------------------------------------------------------------------------------ pack_documents
@pytest.mark.parametrize("B,S", [(2, 16), (1, 64), (3, 7)])
def test_pack_documents_keeps_every_document_in_order_with_shifted_targets(B, S):
    docs = _docs(0, 50)
    out = list(pack_documents(docs, B, S))
    stream, real = [], []
    for tok, tgt, cu in out:
        assert tok.shape == (B, S) and tgt.shape == (B, S) and tok.dtype == tgt.dtype == torch.int64
        assert cu.dtype == torch.int32 and cu.dim() == 1
        check_cu_seqlens(cu, B, S)
        assert set(range(0, B * S, S)) <= set(cu.tolist())  # every row start
        for t, y in _pieces(tok, tgt, cu):
            stream.append((t, y))
    # re-join split pieces: a piece whose last target is real continues into the next piece
    joined, cur_t, cur_y = [], [], []
    for t, y in stream:
        cur_t += t
        cur_y += y
        if y[-1] == -100:
            joined.append((cur_t, cur_y))
            cur_t, cur_y = [], []
    assert not cur_t
    for t, y in joined:
        if all(v == -100 for v in y) and all(v == 0 for v in t) and len(real) == len(docs):
            continue  # padding
        real.append((t, y))
    assert [t for t, _ in real] == docs
    for (t, y), d in zip(real, docs):
        assert y == d[1:] + [-100]  # the next token of the same document; -100 exactly at the document's end


def test_pack_documents_splits_at_a_row_end_and_restarts_positions():
    S = 8
    doc = list(range(1, 13))  # 12 tokens: 3 in row 0 after a 5-token document, 8 in row 1, 1 in row 2
    tok, tgt, cu = next(pack_documents([[100, 101, 102, 103, 104], doc], 3, S))
    assert cu.tolist() == [0, 5, 8, 16, 17, 24]
    assert tok[0].tolist() == [100, 101, 102, 103, 104, 1, 2, 3]
    assert tgt[0].tolist() == [101, 102, 103, 104, -100, 2, 3, 4]  # the first piece keeps its real last target
    assert tok[1].tolist() == list(range(4, 12)) and tgt[1].tolist() == list(range(5, 13))
    assert tok[2].tolist() == [12] + [0] * 7 and tgt[2].tolist() == [-100] * 8  # end of doc, then padding
    assert document_positions(cu).tolist() == [0, 1, 2, 3, 4, 0, 1, 2] + list(range(8)) + [0] + list(range(7))


def test_pack_documents_pads_the_tail_of_the_last_batch_one_document_per_row():
    tok, tgt, cu = next(pack_documents([[5, 6, 7]], 3, 4))
    assert cu.tolist() == [0, 3, 4, 8, 12]
    assert tok.reshape(-1).tolist() == [5, 6, 7] + [0] * 9
    assert tgt.reshape(-1).tolist() == [6, 7, -100] + [-100] * 9


def test_pack_documents_yields_full_batches_then_one_padded_and_skips_empty_documents():
    docs = [[1] * 10, [], [2] * 10, [3] * 5]
    out = list(pack_documents(docs, 1, 8))
    assert len(out) == 4  # 25 tokens in rows of 8
    assert [o[2].tolist() for o in out] == [[0, 8], [0, 2, 8], [0, 4, 8], [0, 1, 8]]
    assert list(pack_documents([], 2, 8)) == []
    with pytest.raises(ValueError):
        next(pack_documents([[1]], 0, 8))


def test_pack_documents_is_deterministic():
    docs = _docs(3, 40)
    a = list(pack_documents(docs, 2, 32))
    b = list(pack_documents(iter(docs), 2, 32))
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert all(torch.equal(u, v) for u, v in zip(x, y))


# ------------------------------------------------------------------------------------------- the cu_seqlens rules
def _cu(v):
    return torch.tensor(v, dtype=torch.int32)


def test_check_cu_seqlens_accepts_a_valid_description_and_returns_the_longest_document():
    assert check_cu_seqlens(_cu([0, 3, 8, 9, 16]), 2, 8) == 7
    assert check_cu_seqlens(_cu([0, 8, 16]), 2, 8) == 8


@pytest.mark.parametrize("cu,match", [
    ([0, 3, 8, 16], "torch.Tensor"),
    (torch.tensor([0, 8, 16], dtype=torch.int64), "int32"),
    (torch.tensor([[0, 8, 16]], dtype=torch.int32), "1-D"),
    (_cu([0]), "1-D"),
    (_cu([1, 8, 16]), "start at 0"),
    (_cu([0, 8, 15]), "end at B\\*S"),
    (_cu([0, 5, 5, 8, 16]), "strictly increasing"),
    (_cu([0, 9, 5, 8, 16]), "strictly increasing"),
    (_cu([0, 5, 12, 16]), "row start"),
])
def test_check_cu_seqlens_names_the_broken_rule(cu, match):
    with pytest.raises(ValueError, match=match):
        check_cu_seqlens(cu, 2, 8)


def test_check_cu_seqlens_refuses_a_device_tensor():
    meta = torch.tensor([0, 8, 16], dtype=torch.int32, device="meta")
    with pytest.raises(ValueError, match="CPU"):
        check_cu_seqlens(meta, 2, 8)


def test_positions_and_micro_batch_slices():
    cu = _cu([0, 3, 8, 10, 16, 24, 30, 32])
    assert document_positions(cu).tolist() == [0, 1, 2, 0, 1, 2, 3, 4, 0, 1, 0, 1, 2, 3, 4, 5] + list(range(8)) + \
        list(range(6)) + [0, 1]
    assert slice_cu_seqlens(cu, 0, 16).tolist() == [0, 3, 8, 10, 16]
    s = slice_cu_seqlens(cu, 16, 32)
    assert s.tolist() == [0, 8, 14, 16] and s.dtype == torch.int32
    check_cu_seqlens(s, 2, 8)


# ------------------------------------------------------------------------------------------- the eager reference
def _tiny():
    from torchft_b200.models.llama import CONFIGS, Llama

    cfg = dataclasses.replace(CONFIGS["llama3_tiny"], n_layers=1)
    m = Llama(cfg, device="cpu", dtype=torch.float32)
    m.init_weights(0)
    return m


def test_reference_with_one_document_per_row_is_the_causal_reference():
    from torchft_b200.models.reference import reference_loss

    m = _tiny()
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, m.cfg.vocab_size, (2, 16), generator=g)
    tgt = torch.randint(0, m.cfg.vocab_size, (2, 16), generator=g)
    l0, g0 = reference_loss(m, tok, tgt, dtype=torch.float64)
    l1, g1 = reference_loss(m, tok, tgt, dtype=torch.float64, cu_seqlens=_cu([0, 16, 32]))
    assert abs(l0 - l1) <= 1e-12 * abs(l0)
    for n in g0:
        torch.testing.assert_close(g1[n], g0[n], rtol=1e-10, atol=1e-14)


def test_reference_isolates_documents_and_restarts_positions():
    """A document alone in a row and the same document packed behind another give the same per-position values: the
    loss of a batch whose only valid targets are that document's is the same, and so is the gradient."""
    from torchft_b200.models.reference import reference_loss

    m = _tiny()
    g = torch.Generator().manual_seed(1)
    doc = torch.randint(0, m.cfg.vocab_size, (9,), generator=g)
    other = torch.randint(0, m.cfg.vocab_size, (7,), generator=g)
    dt = torch.randint(0, m.cfg.vocab_size, (9,), generator=g)
    alone = torch.cat([doc, other]).view(1, 16)
    behind = torch.cat([other, doc]).view(1, 16)
    ta = torch.cat([dt, torch.full((7,), -100)]).view(1, 16)
    tb = torch.cat([torch.full((7,), -100), dt]).view(1, 16)
    la, ga = reference_loss(m, alone, ta, dtype=torch.float64, cu_seqlens=_cu([0, 9, 16]))
    lb, gb = reference_loss(m, behind, tb, dtype=torch.float64, cu_seqlens=_cu([0, 7, 16]))
    assert abs(la - lb) <= 1e-12 * abs(la)
    for n in ga:
        torch.testing.assert_close(gb[n], ga[n], rtol=1e-9, atol=1e-13)
    lc, _ = reference_loss(m, behind, tb, dtype=torch.float64)  # without the mask the document sees `other`
    assert abs(lc - la) > 1e-6 * abs(la)
