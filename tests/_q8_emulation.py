"""Bit-exact CPU emulation of the Q8G fp8 wire format and of every kernel pipeline built on it (``csrc/kernels/quant.cu``),
shared by the quantised-collective tests the way ``_zero1_replicas`` is shared by the FT-ZeRO-1 tests.

Q8G cuts a flat message into groups of 512 elements; the group count is padded to a multiple of ``world``. A buffer holds
``float scales[ng]`` at byte 0 and ``uint8 payload[ng * 512]`` at ``round_up(4 * ng, 16)``. Per group, in fp32:

    amax = max(fmaxf over |x|, which ignores NaN, AMAX_FLOOR)
    s    = amax * fl(1/448)                 (NaN when amax is inf: the whole group dequantises to NaN)
    m    = 448 / amax                       (correctly rounded; 0 when amax is inf)
    code = e4m3 RNE with saturation to +-448 of fl(x * m)
    x'   = fl(code * s)

A reduction adds dequantised values in fp32, one rank after another starting at the reducing rank and wrapping around,
each step a separately rounded multiply and add, then multiplies by ``post_scale``. The kernels are built with fast math,
so every fp32 operation flushes subnormal inputs and results to signed zero (FTZ); the emulation does the same.

``Variant`` switches on deliberate deviations from the kernels (summation order, m, FMA, post_scale placement, FTZ); the
CPU self-tests show each one changes bytes, so the GPU tests that compare against ``EXACT`` can tell them apart.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

GROUP = 512
FP8_MAX = 448.0
AMAX_FLOOR = 2.0 ** -116
TINY = 2.0 ** -126  # smallest normal fp32
F32 = torch.float32
INV448 = (torch.tensor(1.0, dtype=F32) / torch.tensor(FP8_MAX, dtype=F32)).item()  # fl(1/448), as the compiler folds it


@dataclass(frozen=True)
class Variant:
    """Deviations from the kernels' arithmetic; ``EXACT`` has none."""

    order_from_zero: bool = False  # phase-B sum starts at rank 0 instead of the reducing rank
    m_from_s: bool = False  # m = 1/s instead of 448/amax
    fma: bool = False  # acc = fma(code, s, acc) instead of a separate multiply and add
    post_before_sum: bool = False  # post_scale applied to every term instead of to the sum
    no_ftz: bool = False  # keep subnormals


EXACT = Variant()


# ------------------------------------------------------------------------------------------------ fp32 arithmetic
def ftz(x: torch.Tensor, v: Variant = EXACT) -> torch.Tensor:
    """Subnormal fp32 values become zero of the same sign."""
    if v.no_ftz:
        return x
    return torch.where(x.abs() < TINY, x * 0.0, x)


def _mul(a, b, v: Variant = EXACT):
    return ftz(ftz(a, v) * ftz(b, v), v)


def _add(a, b, v: Variant = EXACT):
    return ftz(ftz(a, v) + ftz(b, v), v)


def _fma(a, b, c, v: Variant = EXACT):
    # code (4 significant bits) times s (24) is exact in fp64; the fp64 sum is rounded twice, which differs from one
    # rounding only on ties that random data does not hit
    return ftz((ftz(a, v).double() * ftz(b, v).double() + ftz(c, v).double()).float(), v)


def load(x: torch.Tensor) -> torch.Tensor:
    """Flat fp32 values of an fp32/bf16/fp16 tensor (exact), on the CPU."""
    return x.detach().reshape(-1).to("cpu", F32)


def pseudo_grad(a: torch.Tensor, b: Optional[torch.Tensor], v: Variant = EXACT) -> torch.Tensor:
    """What the kernels quantise: ``a`` or fl(a - b)."""
    a = load(a)
    return a if b is None else ftz(ftz(a, v) - ftz(load(b), v), v)


def cast(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """fp32 -> output dtype, round to nearest even (overflow to inf)."""
    return x if dtype == F32 else x.to(dtype)


# ------------------------------------------------------------------------------------------------ layout
def ngroups(nelem: int, world: int = 1) -> int:
    w = max(1, world)
    return ((nelem + GROUP - 1) // GROUP + w - 1) // w * w


def payload_off(ng: int) -> int:
    return (4 * ng + 15) // 16 * 16


def buffer_bytes(nelem: int, world: int = 1) -> int:
    ng = ngroups(nelem, world)
    return payload_off(ng) + ng * GROUP


def slice_buffer_bytes(nelem: int, world: int) -> int:
    sl = ngroups(nelem, world) // world
    return (payload_off(sl) + sl * GROUP + 255) // 256 * 256


def groups_of(x: torch.Tensor, ng: int) -> torch.Tensor:
    """Flat fp32 values zero-padded to ``[ng, 512]``."""
    out = torch.zeros(ng * GROUP, dtype=F32)
    out[: x.numel()] = x[: ng * GROUP]
    return out.view(ng, GROUP)


class Q8:
    """A Q8G message: fp32 scales ``[ng]`` and uint8 e4m3 codes ``[ng, 512]``."""

    def __init__(self, scales: torch.Tensor, codes: torch.Tensor) -> None:
        self.scales, self.codes = scales, codes

    @property
    def ng(self) -> int:
        return self.scales.numel()

    def __getitem__(self, idx) -> "Q8":
        return Q8(self.scales[idx], self.codes[idx])

    @staticmethod
    def cat(parts: Sequence["Q8"]) -> "Q8":
        return Q8(torch.cat([p.scales for p in parts]), torch.cat([p.codes for p in parts]))

    @staticmethod
    def zeros(ng: int) -> "Q8":
        """What a memset buffer holds: scale 0, code 0."""
        return Q8(torch.zeros(ng, dtype=F32), torch.zeros(ng, GROUP, dtype=torch.uint8))

    def to_bytes(self) -> torch.Tensor:
        """The buffer as the kernels lay it out (alignment padding zero)."""
        poff = payload_off(self.ng)
        out = torch.zeros(poff + self.ng * GROUP, dtype=torch.uint8)
        out[: 4 * self.ng] = self.scales.contiguous().view(torch.uint8)
        out[poff:] = self.codes.reshape(-1)
        return out

    @staticmethod
    def from_bytes(buf: torch.Tensor, ng: int) -> "Q8":
        buf = buf.detach().to("cpu").reshape(-1)
        poff = payload_off(ng)
        return Q8(buf[: 4 * ng].clone().view(F32), buf[poff: poff + ng * GROUP].clone().view(ng, GROUP))


# ------------------------------------------------------------------------------------------------ e4m3
def e4m3_codes(y: torch.Tensor) -> torch.Tensor:
    """fp32 -> e4m3 bytes as ``cvt.rn.satfinite.e4m3x2.f32``: round to nearest even, finite values and inf saturate to
    +-448, NaN stays NaN. torch's cast rounds the same way but does not saturate, hence the clamp."""
    return y.clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def e4m3_decode(codes: torch.Tensor) -> torch.Tensor:
    return codes.view(torch.float8_e4m3fn).to(F32)


def group_quant(x: torch.Tensor, v: Variant = EXACT) -> Q8:
    """Quantise ``[ng, 512]`` fp32 values."""
    x = ftz(x, v)
    amax = torch.where(torch.isnan(x), torch.zeros_like(x), x.abs()).amax(dim=1)  # fmaxf ignores NaN
    amax = amax.clamp_min(AMAX_FLOOR)
    finite = amax < float("inf")
    s = torch.where(finite, _mul(amax, torch.tensor(INV448, dtype=F32), v), torch.tensor(float("nan")))
    if v.m_from_s:
        m = torch.where(finite, 1.0 / s, torch.zeros_like(s))
    else:
        m = torch.tensor(FP8_MAX, dtype=F32) / amax
    return Q8(s, e4m3_codes(_mul(x, m[:, None], v)))


def dequant(q: Q8, v: Variant = EXACT) -> torch.Tensor:
    """``[ng, 512]`` fp32 values ``fl(code * s)``."""
    return _mul(e4m3_decode(q.codes), q.scales[:, None], v)


def quantize(x: torch.Tensor, ng: int, v: Variant = EXACT) -> Q8:
    """``q8_quantize_kernel``: ``ng`` groups of the flat fp32 values ``x`` (zeros past its end)."""
    return group_quant(groups_of(x, ng), v)


def reduce(srcs: Sequence[Q8], first: torch.Tensor, post_scale: float, start_zero: bool = False,
           v: Variant = EXACT) -> torch.Tensor:
    """fp32 sum over ranks of ``srcs`` (Q8 messages of equal group count), group g starting at rank ``first[g]`` and
    wrapping around, times ``post_scale``. ``start_zero``: the accumulator starts at +0 (``q8_reduce_kernel``) instead
    of at the first term (so a -0 first term stays -0)."""
    W = len(srcs)
    ng = srcs[0].ng
    post = torch.tensor(post_scale, dtype=F32)
    codes = torch.stack([e4m3_decode(s.codes) for s in srcs])  # [W, ng, 512]
    scales = torch.stack([s.scales for s in srcs])  # [W, ng]
    if v.order_from_zero:
        first = torch.zeros_like(first)
    cols = torch.arange(ng)
    acc = None if not start_zero else torch.zeros(ng, GROUP, dtype=F32)
    for k in range(W):
        p = (first + k) % W
        c, s = codes[p, cols], scales[p, cols][:, None]
        if v.post_before_sum:
            s = _mul(s, post, v)
        if acc is None:
            acc = _mul(c, s, v)
        elif v.fma:
            acc = _fma(c, s, acc, v)
        else:
            acc = _add(acc, _mul(c, s, v), v)
    return acc if v.post_before_sum else _mul(acc, post, v)


def owners(ng: int, world: int) -> torch.Tensor:
    """Rank that reduces each group of a message quantised for ``world`` ranks (contiguous runs of ng/world)."""
    return torch.arange(ng) // (ng // world)


def equal_q8(got: Q8, want: Q8) -> bool:
    """Scales bit for bit and codes byte for byte, NaN matching NaN whatever its sign and payload."""
    gs, ws = got.scales.view(torch.int32), want.scales.view(torch.int32)
    sn, wn = torch.isnan(got.scales), torch.isnan(want.scales)
    gc, wc = got.codes, want.codes
    cn, wcn = (gc & 0x7F) == 0x7F, (wc & 0x7F) == 0x7F
    return (torch.equal(sn, wn) and torch.equal(gs[~sn], ws[~wn]) and torch.equal(cn, wcn)
            and torch.equal(gc[~cn], wc[~wcn]))


def equal_bits(got: torch.Tensor, want: torch.Tensor) -> bool:
    """Same dtype, same bits, NaN matching NaN."""
    got, want = got.detach().to("cpu").reshape(-1), want.detach().to("cpu").reshape(-1)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    gn, wn = torch.isnan(got), torch.isnan(want)
    it = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[got.element_size()]
    return torch.equal(gn, wn) and torch.equal(got[~gn].view(it), want[~wn].view(it))


def first_mismatch(got: torch.Tensor, want: torch.Tensor) -> str:
    got, want = got.detach().to("cpu").reshape(-1).float(), want.detach().to("cpu").reshape(-1).float()
    bad = ~((got == want) | (torch.isnan(got) & torch.isnan(want)))
    if not bad.any():
        return "equal values (bits differ: signed zero?)"
    i = int(bad.nonzero()[0])
    return f"{int(bad.sum())} mismatches, first at {i} (group {i // GROUP}): got {got[i].item()!r} want {want[i].item()!r}"


def message(n: int, world: int, seed: int, dtype: torch.dtype = F32) -> List[torch.Tensor]:
    """Per-rank test inputs (CPU, ``dtype``): normal values whose magnitude changes from group to group over twelve
    decades, with one group at 2^-120 (below the amax floor, where dequantised small codes are subnormal) so that every
    ``Variant`` shows on them."""
    g = torch.Generator().manual_seed(seed)
    ng = (n + GROUP - 1) // GROUP
    out = []
    for _ in range(world):
        mag = torch.pow(10.0, torch.empty(ng).uniform_(-6, 6, generator=g))
        if ng > 2:
            mag[ng // 2] = 2.0 ** -120
        x = torch.randn(ng, GROUP, generator=g) * mag[:, None]
        out.append(x.reshape(-1)[:n].to(dtype))
    return out


# ------------------------------------------------------------------------------------------------ entry points
def allreduce_launch(xs: Sequence[torch.Tensor], post_scale: float, contribute: Sequence[bool],
                     v: Variant = EXACT) -> Tuple[torch.Tensor, Q8, List[Q8]]:
    """One ``q8_allreduce_kernel`` launch (mode 0) over the flat fp32 inputs ``xs`` (one per rank, already ``a - b``).
    Returns the fp32 result (before the output cast, ``numel`` elements), the reduced Q8G message every rank's segment
    holds afterwards, and what each rank quantised in phase A (a non-contributing rank quantises zeros)."""
    W, n = len(xs), xs[0].numel()
    ng = ngroups(n, W)
    mine = [quantize(x if c else torch.zeros(n, dtype=F32), ng, v) for x, c in zip(xs, contribute)]
    red = group_quant(reduce(mine, owners(ng, W), post_scale, v=v), v)
    return dequant(red, v).reshape(-1)[:n], red, mine


def staging_chunk(staging_usable: int, world: int) -> int:
    """Elements per ``q8_allreduce_`` launch: the largest multiple of 512 * world whose Q8G buffer fits in staging, minus
    one such unit (``SymmetricComm.q8_allreduce_``)."""
    unit = GROUP * world
    return (staging_usable * 512 // 516) // unit * unit - unit


def allreduce(xs: Sequence[torch.Tensor], post_scale: float, contribute: Optional[Sequence[bool]] = None,
              per: Optional[int] = None, v: Variant = EXACT) -> Tuple[torch.Tensor, Q8]:
    """``SymmetricComm.q8_allreduce_`` without a scratch segment: one launch per ``per`` elements. Returns the fp32
    result and the reduced Q8G message of the last launch (what the staging buffers hold afterwards)."""
    W, n = len(xs), xs[0].numel()
    contribute = [True] * W if contribute is None else contribute
    per = n if per is None else per
    outs, red = [], None
    for lo in range(0, n, per):
        o, red, _ = allreduce_launch([x[lo: lo + per] for x in xs], post_scale, contribute, v)
        outs.append(o)
    return torch.cat(outs), red


def allreduce_scratch(xs: Sequence[torch.Tensor], post_scale: float, contribute: Optional[Sequence[bool]] = None,
                      v: Variant = EXACT) -> Tuple[torch.Tensor, List[Q8], List[Q8]]:
    """The ``*_q8`` scratch-segment pipeline (quantise, slice-reduce, gather-dequantise). Returns the fp32 result, what
    every rank's scratch holds at offset 0 (its quantised input, or the zeros of the memset of a non-contributing
    rank) and each rank's reduced slice (at ``round_up(buffer_bytes, 256)``)."""
    W, n = len(xs), xs[0].numel()
    contribute = [True] * W if contribute is None else contribute
    ng = ngroups(n, W)
    sl = ng // W
    mine = [quantize(x, ng, v) if c else Q8.zeros(ng) for x, c in zip(xs, contribute)]
    red = group_quant(reduce(mine, owners(ng, W), post_scale, v=v), v)
    return dequant(red, v).reshape(-1)[:n], mine, [red[r * sl:(r + 1) * sl] for r in range(W)]


def reduce_scatter(ins: Sequence[torch.Tensor], slice_elems: int, post_scale: float,
                   contribute: Optional[Sequence[bool]] = None, v: Variant = EXACT) -> List[torch.Tensor]:
    """``q8_reduce_scatter_`` (kernel mode 1): rank-slice s of every input is quantised on its own grid of
    ceil(slice_elems / 512) groups; rank r gets the fp32 sum of slice r (from rank r, wrapping) times ``post_scale``,
    ``valid = clamp(n - r * slice_elems, 0, slice_elems)`` elements. Returns fp32 results per rank."""
    W, n = len(ins), ins[0].numel()
    contribute = [True] * W if contribute is None else contribute
    gs = (slice_elems + GROUP - 1) // GROUP
    outs = []
    for r in range(W):
        lo = r * slice_elems
        parts = [quantize(x[lo: min(n, lo + slice_elems)] if c else torch.zeros(0, dtype=F32), gs, v)
                 for x, c in zip(ins, contribute)]
        acc = reduce(parts, torch.full((gs,), r), post_scale, v=v)
        outs.append(acc.reshape(-1)[: max(0, min(slice_elems, n - lo))])
    return outs


def slice_plan(numels: Sequence[int], world: int, slice_elems: Optional[Sequence[int]] = None) -> List[Tuple[int, int]]:
    """(slice_elems, groups) per tensor of ``collectives._SlicePlan``."""
    out = []
    for i, n in enumerate(numels):
        se = slice_elems[i] if slice_elems is not None else ((n + world - 1) // world + 7) // 8 * 8
        out.append((se, (se + GROUP - 1) // GROUP))
    return out


def _plan_reduce(xs: Sequence[torch.Tensor], se: int, g: int, post: float, v: Variant) -> List[Q8]:
    """Every rank's reduced, requantised slice of one tensor of the generic path (``q8_reduce`` over what the
    all-to-all delivered: slice r of every peer, summed from rank r on an accumulator that starts at +0)."""
    W, n = len(xs), xs[0].numel()
    reds = []
    for r in range(W):
        parts = [quantize(x[r * se: min(n, (r + 1) * se)], g, v) for x in xs]
        reds.append(group_quant(reduce(parts, torch.full((g,), r), post, start_zero=True, v=v), v))
    return reds


def allreduce_quantized(tensors: Sequence[Sequence[torch.Tensor]], avg: bool, v: Variant = EXACT) -> List[torch.Tensor]:
    """``collectives.allreduce_quantized`` over a generic process group. ``tensors[r]`` is rank r's list; returns the
    fp32 result per tensor (the same on every rank): slices quantised, reduced and requantised by their rank, then
    gathered and dequantised."""
    W = len(tensors)
    post = 1.0 / W if avg else 1.0
    outs = []
    for i, (se, g) in enumerate(slice_plan([t.numel() for t in tensors[0]], W)):
        xs = [load(tensors[r][i]) for r in range(W)]
        n = xs[0].numel()
        red = _plan_reduce(xs, se, g, post, v)
        outs.append(torch.cat([dequant(q, v).reshape(-1)[: max(0, min(se, n - r * se))] for r, q in enumerate(red)]))
    return outs


def reduce_scatter_quantized(inputs: Sequence[Sequence[torch.Tensor]], avg: bool, es: int,
                             v: Variant = EXACT) -> List[torch.Tensor]:
    """``collectives.reduce_scatter_quantized`` over a generic process group: per rank, the concatenated fp32 row-slices
    of every row-padded input (``es`` is the element size, which decides the path)."""
    W = len(inputs)
    post = 1.0 / W if avg else 1.0
    padded = []
    for r in range(W):
        ps = []
        for t in inputs[r]:
            rows = t.shape[0] if t.dim() else 1
            prow = (rows + W - 1) // W * W
            p = torch.zeros(prow, max(1, t.numel() // max(rows, 1)), dtype=F32)
            p[:rows] = load(t).view(rows, -1)
            ps.append(p.reshape(-1))
        padded.append(ps)
    slices = [p.numel() // W for p in padded[0]]
    if any((s * es) % 16 for s in slices):
        full = allreduce_quantized(padded, avg, v)
        return [torch.cat([f[r * s:(r + 1) * s] for f, s in zip(full, slices)]) for r in range(W)]
    outs = [[] for _ in range(W)]
    for i, (se, g) in enumerate(slice_plan([p.numel() for p in padded[0]], W, slices)):
        red = _plan_reduce([padded[r][i] for r in range(W)], se, g, post, v)
        for r in range(W):
            outs[r].append(dequant(red[r], v).reshape(-1)[:se])
    return [torch.cat(o) for o in outs]
