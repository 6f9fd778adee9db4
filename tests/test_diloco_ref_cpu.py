"""The DiLoCo replay (``_diloco_ref``) on the CPU: its schedule and outer step reproduce the upstream golden histories
exactly, and its averaged pseudo-gradient is the bits of the reduction it models. The GPU tests hold the flat path to
this replay, so it is tied here to upstream semantics rather than to our kernels."""

import json
import os

import numpy as np
import pytest
import torch

import _q8_emulation as E
from _diloco_ref import outer_ref, pseudo_grad_bits, schedule

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "diloco")
CASES = [(0, 0.0), (0, 0.5), (0, 1.0), (1, 0.0), (1, 0.5), (1, 1.0)]  # fixture index = position (test_diloco_golden)


def test_schedule_semantics():
    # one fragment, window 4, delay 0: prepare and apply at the end of every window
    assert schedule(4, 1, 0, 8) == [(None, None)] * 3 + [(0, 0)] + [(None, None)] * 3 + [(0, 0)]
    # two fragments, window 3, delay 1: prepared one step early, fragments alternate from the committed count
    assert schedule(6, 2, 1, 6, start=1) == [(None, None), (1, None), (None, 1), (None, None), (0, None), (None, 0)]
    # a vetoed sync retries the same fragment in the next window
    assert [p for _, p in schedule(4, 2, 0, 8, commits=[True, False, True, True])] == [None, 0, None, 1, None, 1, None, 0]
    with pytest.raises(AssertionError):
        schedule(4, 2, 2, 4)  # the delay must leave the window a step


@pytest.mark.parametrize("index", range(len(CASES)))
def test_replay_matches_reference_history(index):
    """The mocked-update scenario of ``test_diloco_golden`` (constant gradient 2, inner lr 1, outer plain SGD lr 2, two
    1x1 fragments, sync_every 6, two committed steps before training) replayed with ``schedule`` + ``outer_ref``."""
    delay, alpha = CASES[index]
    with open(os.path.join(FIXTURES, f"mocked_updates_{index}.json")) as f:
        expected = json.load(f)[0][0]  # both replicas hold the same history
    names = ["layers.0.weight", "layers.1.weight"]
    w = torch.ones(2, dtype=torch.float64)
    orig, mom, snap = w.clone(), torch.zeros(2, dtype=torch.float64), w.clone()
    history, glob = {0: w.clone()}, {0: orig.clone()}
    for i, (prepared, performed) in enumerate(schedule(6, 2, delay, 15, start=2), start=1):
        w -= 1.0 * 2.0
        if prepared is not None:
            snap[prepared] = w[prepared]
        if performed is not None:
            f = performed
            ref = outer_ref(orig[f:f + 1], w[f:f + 1], mom[f:f + 1], orig[f:f + 1] - snap[f:f + 1], 2.0, 0.0, False, alpha)
            orig[f], w[f] = ref.orig[0], ref.param[0]
            glob[i] = orig.clone()
        history[i] = w.clone()
    for section, got in (("history", history), ("global_parameter_history", glob)):
        assert {int(k) for k in expected[section]} <= set(got), section
        for step, params in expected[section].items():
            for j, name in enumerate(names):
                assert got[int(step)][j].item() == params[name][0][0], (section, step, name, got[int(step)].tolist())


def test_outer_ref_bound_admits_fp32_and_rejects_one_ulp_more():
    """The fp32 evaluation of the kernel's formula sits inside the bound; the same value one bf16 ulp off in a single
    element does not, so the bound is tight enough to catch a wrong alpha or a dropped momentum term."""
    from _fp64 import assert_close_elementwise

    g = torch.Generator().manual_seed(0)
    n = 4096
    orig = torch.randn(n, generator=g).to(torch.bfloat16)
    local = (orig.float() + 0.1 * torch.randn(n, generator=g)).to(torch.bfloat16)
    grad = (0.05 * torch.randn(n, generator=g)).to(torch.bfloat16)
    mom = 0.05 * torch.randn(n, generator=g)
    lr, mu, alpha = 0.7, 0.9, 0.3
    b = mu * mom + grad.float()
    o = orig.float() - lr * (grad.float() + mu * b)
    p = (o + alpha * (local.float() - o)).to(torch.bfloat16)
    ref = outer_ref(orig, local, mom, grad, lr, mu, True, alpha)
    assert_close_elementwise(o.to(torch.bfloat16), ref.orig, ulps=1, abs_slack=ref.orig_slack, what="ref orig")
    assert_close_elementwise(p, ref.param, ulps=1, abs_slack=ref.param_slack, what="ref param")
    assert_close_elementwise(b, ref.mom, ulps=0, abs_slack=ref.mom_slack, what="ref mom")
    bad = p.clone()
    bad.view(torch.int16)[1234] += 2
    with pytest.raises(AssertionError, match="worst element"):
        assert_close_elementwise(bad, ref.param, ulps=1, abs_slack=ref.param_slack, what="ref param, one element off")
    other = outer_ref(orig, local, mom, grad, lr, mu, True, 1 - alpha)
    with pytest.raises(AssertionError, match="worst element"):
        assert_close_elementwise(p, other.param, ulps=1, abs_slack=other.param_slack, what="ref param, 1 - alpha")
    from _fp64 import _WORST

    _WORST.clear()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_pseudo_grad_bits_unquantised(dtype):
    """``torch.sub`` rounds ``original - local`` to the dtype; the replicas' differences are summed in rank order in
    fp32, a non-contributing replica adds zeros, and the sum is scaled by 1/participants and rounded once."""
    g = torch.Generator().manual_seed(1)
    n = 37
    origs = [torch.randn(n, generator=g).to(dtype) for _ in range(3)]
    locals_ = [(o.float() + 0.01 * torch.randn(n, generator=g)).to(dtype) for o in origs]
    got = pseudo_grad_bits(origs, locals_, dtype, False, [True, False, True], 2)
    assert got.dtype == dtype and got.shape == (n,)
    d = [(o.float() - l.float()).to(dtype).float() for o, l in zip(origs, locals_)]
    want = (((d[0] + 0.0) + d[2]) * np.float32(0.5)).to(dtype)  # fp32 sum, one multiply, one rounding
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    # the average is 1/participants, not 1/world: with a replica out the two differ
    third = pseudo_grad_bits(origs, locals_, dtype, False, [True, False, True], 3)
    assert not torch.equal(third, got)
    # a subnormal fp32 partial sum is flushed, as the kernels are built with fast math
    tiny = torch.tensor([2.0 ** -130] * 8, dtype=torch.float32)
    z = torch.zeros(8, dtype=torch.float32)
    assert torch.equal(pseudo_grad_bits([tiny, tiny], [z, z], torch.float32, False, [True, True], 2),
                       torch.zeros(8, dtype=torch.float32))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_pseudo_grad_bits_quantised(dtype):
    """The fused Q8G delta: ``original - local`` in fp32, quantised per 512-element group, reduced and dequantised;
    a non-contributing replica quantises nothing (zero scales)."""
    g = torch.Generator().manual_seed(2)
    n = 1100  # three groups, the last one partial
    origs = [torch.randn(n, generator=g).to(dtype) for _ in range(2)]
    locals_ = [(o.float() + 0.05 * torch.randn(n, generator=g)).to(dtype) for o in origs]
    got = pseudo_grad_bits(origs, locals_, dtype, True, [True, True], 2)
    want, _, _ = E.allreduce_scratch([E.pseudo_grad(o, l) for o, l in zip(origs, locals_)], 0.5, [True, True])
    assert torch.equal(got, E.cast(want, dtype))
    # quantisation noise is visible against the exact average, but within one fp8 step of each group's scale
    exact = sum((o.double() - l.double()) for o, l in zip(origs, locals_)) / 2
    assert not torch.equal(got.double(), exact)
    assert float((got.double() - exact).abs().max()) <= float(exact.abs().max()) / 8
    alone = pseudo_grad_bits(origs, locals_, dtype, True, [True, False], 1)
    mine = E.cast(E.allreduce_scratch([E.pseudo_grad(origs[0], locals_[0]), torch.zeros(n)], 1.0, [True, False])[0], dtype)
    assert torch.equal(alone, mine)
