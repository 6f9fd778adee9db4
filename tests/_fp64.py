"""The element-by-element fp64 checker the kernel tests share, and the one-step fp64 AdamW reference with its derived
slack.

Every check is per element: ``|got - ref| <= ulps * ulp_out(ref) + abs_slack``. ``ulp_out`` is the spacing of the output
dtype at ``|ref|``; ``abs_slack`` is an elementwise bound, derived next to each reference, on an error the kernel is
allowed to make. A whole-tensor norm passes while one vector, one tail or one CTA's rows are wrong, so it is never the
check. A module that uses the checker imports ``_report_margins`` too: it prints every check's worst element against its
bound at the end of the module, so the headroom is visible on success.
"""

import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24  # fp32 unit roundoff; an fp32 ulp at x is <= 2U|x|
FTZ = 2.0 ** -126  # smallest normal fp32/bf16: results below it are flushed to zero under --use_fast_math
_MANT = {torch.bfloat16: 7, torch.float16: 10, torch.float32: 23, torch.float64: 52}
_WORST = {}


def ulp_out(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Spacing of ``dtype`` at ``|ref|`` (float64), down to the dtype's subnormal spacing."""
    a = ref.abs().clamp(min=torch.finfo(dtype).tiny)
    _, e = torch.frexp(a)  # a = m * 2**e with m in [0.5, 1)
    return torch.ldexp(torch.ones_like(a), e - 1 - _MANT[dtype])


def assert_close_elementwise(got, ref, *, ulps, abs_slack=None, what):
    """Assert ``|got - ref| <= ulps * ulp_out(ref) + abs_slack`` for every element (``ref`` float64).

    A non-finite ``ref`` must be matched exactly; a non-finite ``got`` where ``ref`` is finite fails. The worst element
    (largest error over its bound) is reported on failure, and kept for the per-check summary printed at the end of
    the module so the headroom is visible on success too."""
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    ref = ref.to(torch.float64)
    g = got.to(ref.device).to(torch.float64)
    fin = torch.isfinite(ref)
    bound = ulps * ulp_out(torch.where(fin, ref, 0.0), got.dtype)
    if abs_slack is not None:
        bound = bound + abs_slack
    err = torch.where(fin, (g - ref).abs(), torch.where(g == ref, 0.0, math.inf))
    ratio = torch.where(err == 0, 0.0, err / bound).nan_to_num(nan=math.inf).flatten()
    w = int(ratio.argmax())
    r = float(ratio[w])
    idx = tuple(int(i) for i in np.unravel_index(w, tuple(ref.shape))) if ref.dim() else ()
    msg = (f"{what}: worst element {idx}: got {g.flatten()[w].item():.9g}, ref {ref.flatten()[w].item():.9g}, "
           f"|err| {err.flatten()[w].item():.3g}, bound {bound.flatten()[w].item():.3g}, err/bound {r:.3g}")
    if r >= _WORST.get(what, (-1.0, ""))[0]:
        _WORST[what] = (r, msg)
    assert r <= 1.0, msg


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    for what in sorted(_WORST):
        print(f"[margin] {_WORST[what][1]}")
    _WORST.clear()


def _f32(x: float) -> float:
    return float(np.float32(x))


def _adamw_ref(p32, m, v, g, lr, b1, b2, eps, wd, t, gscale, m_new, v_new):
    """One fp64 AdamW step from the kernel's state before it, with fp32-rounded hyper-parameters (what the kernel
    receives); the master's update is computed from the kernel's new m and v, so their rounding does not enter it.
    ``wd`` may be a tensor (0 where an element takes no decay). The bias corrections are 1 - b^t of the fp32 betas the
    moving averages use, each rounded once to fp32."""
    lr, b1, b2, eps, gscale = map(_f32, (lr, b1, b2, eps, gscale))
    wd = wd.double() if torch.is_tensor(wd) else _f32(wd)
    bc1, bc2 = _f32(1.0 - b1 ** t), _f32(1.0 - b2 ** t)
    gr = g.double() * gscale
    md = b1 * m.double() + (1 - b1) * gr
    vd = b2 * v.double() + (1 - b2) * gr * gr
    upd = (lr / bc1) * m_new.double() / (v_new.double().sqrt() / math.sqrt(bc2) + eps)
    wdec = p32.double() * (1 - lr * wd)
    # m: g * gscale, two products and a sum: 4 U of the terms; v: all terms >= 0, 5 roundings -> 5 U relative
    m_sl = 4 * U * (b1 * m.double().abs() + (1 - b1) * gr.abs())
    v_sl = 5 * U * vd
    # master: w * decay (decay from lr * wd and 1 - that: 3 U) minus the update, whose approximate sqrtf (4 ulp), rsqrtf
    # (2 ulp), + eps, __fdividef (2 ulp), lr / bc1 (2 ulp) and the products keep it within 32 U; 1 U for the difference
    w_sl = 4 * U * wdec.abs() + 32 * U * upd.abs()
    return wdec - upd, w_sl, md, m_sl, vd, v_sl
