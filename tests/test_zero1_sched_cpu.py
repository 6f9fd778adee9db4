"""FT-ZeRO-1 learning-rate schedules and weight-decay exemptions without a GPU: the fp32 rate table, its validation,
the per-unit split of the exempt ranges and the trainer's mapping of selected parameters to flat ranges."""

from __future__ import annotations

import math

import numpy as np
import pytest
import torch


def _warmup_cosine(warmup, total):
    def f(i):
        if i < warmup:
            return (i + 1) / warmup
        return 0.1 + 0.9 * 0.5 * (1 + math.cos(math.pi * min(1.0, (i - warmup) / max(1, total - warmup))))
    return f


def test_table_is_the_fp32_product_of_lr_and_the_lambda():
    from torchft_b200.parallel.zero1 import lr_schedule_table

    lr, lam = 3e-4, _warmup_cosine(5, 40)
    tab = lr_schedule_table(lr, lam, 40)
    assert tab.dtype == np.float32 and tab.shape == (40,)
    assert tab.tobytes() == np.array([np.float32(lr * lam(i)) for i in range(40)], dtype=np.float32).tobytes()


def test_table_matches_lambda_lr_stepped_after_every_step():
    from torchft_b200.parallel.zero1 import lr_schedule_table

    lr, lam = 1e-2, _warmup_cosine(3, 12)
    opt = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(1))], lr=lr)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lam)
    seen = []
    for _ in range(12):
        seen.append(np.float32(opt.param_groups[0]["lr"]))  # the rate this update applies
        opt.step()  # no gradients: changes nothing
        sched.step()
    assert lr_schedule_table(lr, lam, 12).tolist() == [float(x) for x in seen]


class _Opt:
    """The host side of ``Zero1Optimizer.lr_at`` without a process group."""

    def __init__(self, lr, lam=None, steps=0):
        from torchft_b200.parallel.zero1 import Zero1Optimizer, lr_schedule_table

        self.param_groups = [{"lr": lr}]
        self._lr_host = lr_schedule_table(lr, lam, steps) if lam is not None else None
        self.lr_at = Zero1Optimizer.lr_at.__get__(self)


def test_lr_at_clamps_past_the_end_and_before_the_first_update():
    lam = lambda i: 1.0 / (i + 1)  # noqa: E731
    o = _Opt(0.5, lam, 4)
    assert [o.lr_at(t) for t in (1, 2, 3, 4)] == [float(np.float32(0.5 / t)) for t in (1, 2, 3, 4)]
    assert o.lr_at(5) == o.lr_at(1000) == o.lr_at(4)
    assert o.lr_at(0) == o.lr_at(1)  # a refresh at t = 0 reads the first entry


def test_lr_at_without_a_schedule_is_the_current_fp32_rate():
    o = _Opt(0.1)
    assert o.lr_at(7) == float(np.float32(0.1))
    o.param_groups[0]["lr"] = 0.2
    assert o.lr_at(7) == float(np.float32(0.2))


@pytest.mark.parametrize("lam,steps,match", [
    (lambda i: 1.0, 0, "lr_steps"),
    (lambda i: 1.0, -3, "lr_steps"),
    (lambda i: -0.5 if i == 2 else 1.0, 5, "update 3"),
    (lambda i: float("nan"), 2, "update 1"),
    (lambda i: float("inf") if i == 1 else 1.0, 2, "update 2"),
])
def test_table_rejects_bad_schedules(lam, steps, match):
    from torchft_b200.parallel.zero1 import lr_schedule_table

    with pytest.raises(ValueError, match=match):
        lr_schedule_table(1e-3, lam, steps)


def test_a_zero_rate_is_allowed():
    from torchft_b200.parallel.zero1 import lr_schedule_table

    assert lr_schedule_table(1e-3, lambda i: 0.0 if i == 0 else 1.0, 3).tolist()[0] == 0.0


# ----------------------------------------------------------------------------- per-unit split
UNITS = [(0, 1024), (1024, 1024 + 256), (1280, 4096)]


def test_split_is_unit_relative_in_unit_order_and_merges_touching_ranges():
    from torchft_b200.parallel.zero1 import split_no_decay

    units = [UNITS[2], UNITS[0], UNITS[1]]  # forward order need not be offset order
    got = split_no_decay(units, [(1280, 1288), (0, 8), (1016, 1024), (1024, 1280), (8, 64), (4088, 4096)])
    assert got == [[(0, 8), (2808, 2816)], [(0, 64), (1016, 1024)], [(0, 256)]]


def test_split_accepts_ranges_at_unit_edges_and_whole_units():
    from torchft_b200.parallel.zero1 import split_no_decay

    assert split_no_decay(UNITS, [(0, 1024), (1280, 4096)]) == [[(0, 1024)], [], [(0, 2816)]]
    assert split_no_decay(UNITS, []) == [[], [], []]


@pytest.mark.parametrize("rs,match", [
    ([(1016, 1032)], "not inside one unit"),      # spans units 0 and 1
    ([(0, 4096)], "not inside one unit"),
    ([(4096, 4104)], "not inside one unit"),      # past the buffer
    ([(4, 16)], "multiples of 8"),
    ([(16, 20)], "multiples of 8"),
    ([(16, 16)], "non-empty"),
])
def test_split_rejects_misaligned_and_straddling_ranges(rs, match):
    from torchft_b200.parallel.zero1 import split_no_decay

    with pytest.raises(ValueError, match=match):
        split_no_decay(UNITS, rs)


def test_split_caps_the_ranges_per_unit():
    from torchft_b200.parallel.zero1 import MAX_NO_DECAY, split_no_decay

    four = [(16 * i, 16 * i + 8) for i in range(MAX_NO_DECAY)]
    assert len(split_no_decay(UNITS, four)[0]) == MAX_NO_DECAY
    with pytest.raises(ValueError, match="unit 0"):
        split_no_decay(UNITS, four + [(512, 520)])
    # the cap counts per unit after merging: touching ranges are one
    assert split_no_decay(UNITS, four + [(8, 16)])[0][0] == (0, 24)


def test_digest_tells_schedules_and_exemptions_apart():
    from torchft_b200.parallel.zero1 import lr_schedule_table, schedule_digest

    a = lr_schedule_table(1e-3, lambda i: 1.0, 4)
    b = lr_schedule_table(1e-3, lambda i: 1.0 if i < 3 else 0.5, 4)
    assert schedule_digest(a, [(0, 8)]) == schedule_digest(a.copy(), [(0, 8)])
    assert schedule_digest(a, [(0, 8), (8, 16)]) == schedule_digest(a, [(0, 16)])
    assert schedule_digest(a, []) != schedule_digest(b, [])
    assert schedule_digest(a, []) != schedule_digest(a, [(0, 8)])
    assert schedule_digest(None, [(0, 8)]) != schedule_digest(a, [(0, 8)])


# ----------------------------------------------------------------------------- trainer helper
def test_trainer_helper_covers_exactly_the_one_dimensional_parameters_of_llama3_tiny():
    from torchft_b200.models.llama import CONFIGS, FlatParams, Llama
    from torchft_b200.parallel.trainer import no_decay_ranges
    from torchft_b200.parallel.zero1 import merge_ranges, split_no_decay, subtract_ranges

    cfg = CONFIGS["llama3_tiny"]
    model = Llama(cfg, device="cpu")
    flat = FlatParams(model, device="cpu")
    rs = no_decay_ranges(flat, model, lambda n, p: p.ndim == 1)
    pad = lambda n: (n + FlatParams.ALIGN - 1) // FlatParams.ALIGN * FlatParams.ALIGN  # noqa: E731
    where = {id(p): o for p, o in zip(flat.params, flat.offsets)}
    gains = [(where[id(p)], where[id(p)] + pad(p.numel())) for n, p in model.named_parameters() if p.ndim == 1]
    others = [(where[id(p)], where[id(p)] + pad(p.numel())) for n, p in model.named_parameters() if p.ndim != 1]
    assert len(gains) == 2 * cfg.n_layers + 1
    assert rs == merge_ranges(gains), "every gain with its padding, merged"
    assert merge_ranges(gains + others) == [(0, flat.numel)]
    assert subtract_ranges(rs, gains) == [] and all(not subtract_ranges([o], rs) == [] for o in others)
    # the exempt elements are exactly the gains' elements plus their padding
    mask = torch.zeros(flat.numel, dtype=torch.bool)
    for lo, hi in rs:
        mask[lo:hi] = True
    for n, p in model.named_parameters():
        o = where[id(p)]
        assert bool(mask[o:o + p.numel()].all()) == (p.ndim == 1) and bool(mask[o:o + p.numel()].any()) == (p.ndim == 1), n
    # units are the forward stages: a block needs two ranges (its two norms are not adjacent), the head unit one
    stages = []
    for stage in model.param_stages():
        lo = min(where[id(p)] for p in stage)
        hi = max(where[id(p)] + pad(p.numel()) for p in stage)
        stages.append((lo, hi))
    per_unit = split_no_decay(stages, rs)
    assert [len(x) for x in per_unit] == [0] + [2] * cfg.n_layers + [1]
    assert all(lo % 8 == 0 and hi % 8 == 0 for x in per_unit for lo, hi in x)
