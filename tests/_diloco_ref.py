"""A replay of (Streaming) DiLoCo's outer loop, shared by the CPU tests that tie it to the upstream golden histories and the
GPU tests that hold the flat path (``_StreamingDiLoCoFragment._try_flat_mode``) to it sync by sync.

* :func:`schedule`: which fragment each inner step prepares and which it applies, from the semantics alone. A replica
  runs ``sync_every / n_fragments`` inner steps per window; the window's fragment is the committed outer step count
  modulo ``n_fragments`` (every replica agrees on it); the pseudo-gradient is taken ``delay`` steps before the window
  ends and applied at its end.
* :func:`pseudo_grad_bits`: the averaged pseudo-gradient ``original - local`` bit for bit, through the Q8G emulation
  (``_q8_emulation``) or through the rounding of ``torch.sub`` and the fused all-reduce model (``_collectives_ref``).
* :func:`outer_ref`: the outer step in float64 (torch SGD with momentum ``mu``, optional Nesterov, on the last global
  weights, then ``lerp`` towards the local weights by ``alpha``), with the per-element bound the fused kernel
  (``diloco_outer``) must meet.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

import _collectives_ref as C
import _q8_emulation as E
from _fp64 import FTZ, U, _f32

_DT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}


def schedule(sync_every: int, n_fragments: int, delay: int, steps: int, start: int = 0,
             commits: Optional[Sequence[bool]] = None) -> List[Tuple[Optional[int], Optional[int]]]:
    """For inner steps 1..``steps``: ``(prepared, performed)`` fragment ids (``None`` when the step does neither), both
    taken after the step. ``start`` is the committed outer step count before the first inner step; ``commits[k]`` is
    the verdict of the k-th sync (all commit by default): a vetoed sync leaves the count, so the next window retries
    the same fragment."""
    assert sync_every % n_fragments == 0 and 0 <= delay < sync_every // n_fragments
    window = sync_every // n_fragments
    out: List[Tuple[Optional[int], Optional[int]]] = []
    committed, syncs = start, 0
    for i in range(1, steps + 1):
        pos = (i - 1) % window + 1  # inner steps taken in this window
        frag = committed % n_fragments
        prepared = frag if pos == window - delay else None
        performed = None
        if pos == window:
            performed = frag
            if commits is None or commits[syncs]:
                committed += 1
            syncs += 1
        out.append((prepared, performed))
    return out


def pseudo_grad_bits(origs: Sequence[torch.Tensor], locals_: Sequence[torch.Tensor], dtype: torch.dtype, quantize: bool,
                     contribute: Sequence[bool], participants: int) -> torch.Tensor:
    """The averaged pseudo-gradient every replica holds after ``Manager.allreduce_delta(grad, original, local)``.

    ``origs[r]``/``locals_[r]`` are replica r's last global and live weights (``dtype``, one flat tensor each);
    ``contribute[r]`` is its ``is_participating()``; the average divides by ``participants`` (``num_participants()``).
    Quantised: ``original - local`` in fp32 inside the Q8G scratch pipeline. Not: ``torch.sub`` rounds the difference to
    ``dtype`` and the fused all-reduce sums in rank order, scales by ``1 / participants`` and rounds once."""
    scale = 1.0 / max(participants, 1)
    if quantize:
        want, _, _ = E.allreduce_scratch([E.pseudo_grad(o, l) for o, l in zip(origs, locals_)], scale, list(contribute))
        return E.cast(want, dtype)
    dt = _DT[dtype]
    bits = []
    for o, l, c in zip(origs, locals_, contribute):
        d = (o.detach().cpu().float() - l.detach().cpu().float()).to(dtype)  # fp32 difference of dtype values, rounded once
        bits.append(d.view(torch.int32 if dtype == torch.float32 else torch.int16).numpy().view(C.BITS[dt]) if c else None)
    out = C.allreduce(bits, dt, C.SUM, scale)
    return torch.from_numpy(out.view(np.int32 if dt == "f32" else np.int16).copy()).view(dtype)


@dataclass
class OuterRef:
    """float64 results of one outer step and the elementwise slack each output of the fused kernel may use."""

    orig: torch.Tensor
    param: torch.Tensor
    mom: torch.Tensor
    orig_slack: torch.Tensor
    param_slack: torch.Tensor
    mom_slack: Optional[torch.Tensor]  # None: without momentum the buffer must not change at all


def outer_ref(orig: torch.Tensor, local: torch.Tensor, mom: torch.Tensor, grad: torch.Tensor, lr: float, mu: float,
              nesterov: bool, alpha: float) -> OuterRef:
    """Torch-SGD semantics on the last global weights ``orig`` with the averaged pseudo-gradient ``grad`` and the fp32
    momentum ``mom``, then ``param = o + alpha (local - o)``. Inputs are the tensors the kernel saw, in their own dtypes;
    the check is ``ulps=1`` of the output dtype plus the slack (``assert_close_elementwise``)."""
    lr_, mu_, al = _f32(lr), _f32(mu), _f32(alpha)
    gd, bd, od, ld = (t.detach().double() for t in (grad, mom, orig, local))
    b = mu_ * bd + gd if mu else bd
    step = (gd + mu_ * b if nesterov else b) if mu else gd
    o = od - lr_ * step
    lw = o + al * (ld - o)
    # b = mu b + g: two roundings of its terms
    b_sl = 2 * U * (mu_ * bd.abs() + gd.abs()) + FTZ if mu else None
    # step carries <= 2 U of |g| + mu |b| (+ mu |b| for Nesterov); lr * step and o - that: 2 U more of their terms,
    # rounded to the dtype once (1 ulp)
    s_abs = gd.abs() + mu_ * b.abs() * (2 if nesterov else 1)
    o_sl = 4 * U * (lr_ * s_abs + od.abs())
    # param = o + alpha (l - o) from the fp32 o: (1 - alpha) of o's error, 3 U of alpha |l - o|, 1 U of |result|
    l_sl = abs(1 - al) * o_sl + 3 * U * al * (ld - o).abs() + U * lw.abs()
    return OuterRef(o, lw, b, o_sl + FTZ, l_sl + FTZ, b_sl)
