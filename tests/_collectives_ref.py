"""A numpy model of what the data-plane reduction kernels compute (``allreduce.cu``, ``reduce_scatter_kernel`` in
``collectives.cu``), and the bit-level check of a kernel's output against it.

Arrays hold raw bits: ``uint32`` for fp32, ``uint16`` for bf16 and fp16. The model:

* every input is promoted to fp32 exactly and the ranks are accumulated in rank order with ``+``, ``fmaxf`` or
  ``fminf``; a rank that does not contribute adds +0.0 at its own position in that order, for every op (it stages
  zeros), so a MAX over negative values with a quiet rank gives 0;
* the library is built with ``--use_fast_math``: fp32 add, mul, max and min flush subnormal operands and results to
  zero of the same sign. bf16 subnormals therefore vanish; fp16 subnormals are normal in fp32 and survive;
* ``fmaxf``/``fminf``: a NaN loses against a number;
* the result is multiplied by the fp32 scale and rounded once, to nearest even, to the dtype (fp16 overflow is ±inf).

The check is bit for bit, except that any NaN matches any NaN and, under MAX/MIN, a zero may carry either sign.
"""

from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

SUM, MAX, MIN = 0, 1, 2
DTYPES = ("f32", "bf16", "f16")
BITS = {"f32": np.uint32, "bf16": np.uint16, "f16": np.uint16}
TINY = np.float32(np.finfo(np.float32).tiny)  # 2^-126, the smallest normal fp32

# values the kernels go wrong on: ±inf, NaN, ±0, subnormals of the dtype (and of fp32), the fp16 range limit
SPECIALS = {
    "f32": np.array([0x7F800000, 0xFF800000, 0x7FC00000, 0x00000000, 0x80000000, 0x00000001, 0x007FFFFF,
                     0x80400000, 0x00800000, 0x80800001], dtype=np.uint32),
    "bf16": np.array([0x7F80, 0xFF80, 0x7FC0, 0x0000, 0x8000, 0x0001, 0x007F, 0x8040, 0x0080], dtype=np.uint16),
    "f16": np.array([0x7C00, 0xFC00, 0x7E00, 0x0000, 0x8000, 0x0001, 0x03FF, 0x8200, 0x7BFF, 0xFBFF,
                     np.float16(60000).view(np.uint16), np.float16(-32768).view(np.uint16)], dtype=np.uint16),
}


def to_f32(bits: np.ndarray, dt: str) -> np.ndarray:
    """Exact promotion of raw ``dt`` bits to fp32 values."""
    if dt == "f32":
        return bits.astype(np.uint32).view(np.float32)
    if dt == "bf16":
        return (bits.astype(np.uint32) << 16).view(np.float32)
    return bits.astype(np.uint16).view(np.float16).astype(np.float32)


def round_to(x: np.ndarray, dt: str) -> np.ndarray:
    """fp32 values -> raw ``dt`` bits, rounded to nearest even (overflow to ±inf)."""
    x = np.asarray(x, dtype=np.float32)
    if dt == "f32":
        return x.view(np.uint32).copy()
    if dt == "f16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).view(np.uint16)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), ((u >> 16) | 0x40).astype(np.uint16), r)


def ftz(x: np.ndarray) -> np.ndarray:
    """fp32 subnormals -> zero of the same sign."""
    return np.where(np.abs(x) < TINY, np.copysign(np.float32(0), x), x).astype(np.float32)


def _red(a: np.ndarray, b: np.ndarray, op: int) -> np.ndarray:
    a, b = ftz(a), ftz(b)
    with np.errstate(invalid="ignore", over="ignore"):
        r = a + b if op == SUM else (np.fmax(a, b) if op == MAX else np.fmin(a, b))
    return ftz(r.astype(np.float32))


def _scale(x: np.ndarray, scale: float) -> np.ndarray:
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        return ftz(ftz(x) * np.float32(scale))


def allreduce(inputs: Sequence[Optional[np.ndarray]], dt: str, op: int, scale: float) -> np.ndarray:
    """Result bits of a reduction over W >= 2 ranks; ``None`` marks a rank that does not contribute."""
    n = next((len(x) for x in inputs if x is not None), 0)
    acc = None
    for x in inputs:
        v = to_f32(x, dt) if x is not None else np.zeros(n, dtype=np.float32)
        acc = v if acc is None else _red(acc, v, op)
    return round_to(_scale(acc, scale), dt)


def scale_copy(x: np.ndarray, dt: str, scale: float, contribute: bool) -> np.ndarray:
    """World 1 (``scale_copy_kernel``): ``x * scale``, or zeros for a rank that does not contribute."""
    if not contribute:
        return np.zeros(len(x), dtype=BITS[dt])
    return round_to(_scale(to_f32(x, dt), scale), dt)


def mismatch(got: np.ndarray, want: np.ndarray, dt: str, op: int) -> Optional[str]:
    """None when ``got`` matches ``want`` (raw bits), else a description of the first element that does not."""
    got, want = np.asarray(got, dtype=BITS[dt]), np.asarray(want, dtype=BITS[dt])
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    g, w = to_f32(got, dt), to_f32(want, dt)
    ok = (got == want) | (np.isnan(g) & np.isnan(w))
    if op in (MAX, MIN):
        ok |= (g == 0) & (w == 0)
    bad = np.flatnonzero(~ok)
    if bad.size == 0:
        return None
    i = int(bad[0])
    return (f"{bad.size} of {got.size} elements differ; first at {i}: got {g[i]!r} ({int(got[i]):#x}), "
            f"want {w[i]!r} ({int(want[i]):#x})")


def values(rng: np.random.Generator, n: int, dt: str, specials: bool = True) -> np.ndarray:
    """Raw bits of ``n`` test values: every 16-byte vector gets a magnitude class (1, 1e3, 1e-3 or 0), and with
    ``specials`` about one element in 32 is replaced by a value of :data:`SPECIALS`."""
    per = 16 // np.dtype(BITS[dt]).itemsize
    nvec = -(-n // per)
    mag = np.repeat(rng.choice(np.array([1.0, 1e3, 1e-3, 0.0]), nvec), per)[:n]
    bits = round_to((rng.standard_normal(n) * mag).astype(np.float32), dt)
    if specials and n:
        k = max(1, n // 32)
        bits[rng.integers(0, n, k)] = rng.choice(SPECIALS[dt], k)
    return bits
