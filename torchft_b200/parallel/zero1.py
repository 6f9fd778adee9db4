"""FT-ZeRO-1: optimizer state partitioned across REPLICA GROUPS, without giving up fault tolerance.

The reference keeps the full optimizer on every replica and all-reduces every gradient
(upstream torchft/manager.py:466-478, upstream torchft/optim.py:52-55). Here the
cross-replica collective and the optimizer are one pipeline of three hand-written sm_90a kernels
(``csrc/kernels/zero1.cu``):

* backward:  ``reduce_scatter`` per unit (one transformer block = one unit), overlapped with backward;
  rank ``r`` reduces slice ``r`` of the unit out of every peer's HBM and also pushes the result to its
  ``k-1`` buddies (ranks ``r+1 .. r+k-1``) -- every slice of optimizer state lives on ``k`` replicas;
* commit:    ONE kernel ANDs "my step was clean" over the quorum through the signal pads and writes a
  device gate word -- no host synchronisation, no RPC; the Manager reads the verdict lazily;
* update:    gated AdamW on the held slices; the primary holder stores the new bf16 weights straight
  into every replica's parameter buffer (the all-gather is the update's epilogue) while the next
  forward already runs, unit by unit.

Fault tolerance. Ownership is a pure function of (unit, quorum rank, world, k) -- see
:class:`ShardLayout` -- so every replica derives it from the quorum alone. On every quorum change
each rank publishes which element ranges of (master, m, v) it holds and at which update count; a
rank whose new slices it does not hold yet pulls them over NVLink (``heal_copy`` kernel, peer
memory) from any replica that does. A slice is lost only if all ``k`` holders disappear within one
quorum transition; it is then re-seeded from the (fully replicated) bf16 weights with zero moments
and reported. The first commit phase after a quorum change re-broadcasts the weights from the
master copies, so a failure in the middle of an all-gather can never leave replicas with
different weights for more than one (discarded or slightly stale) step.
"""

from __future__ import annotations

import contextlib
import json
import logging
import math
import os
import threading
from dataclasses import dataclass
from typing import Any, Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import torch

logger = logging.getLogger(__name__)

Range = Tuple[int, int]

__all__ = ["ShardLayout", "Zero1Optimizer", "merge_ranges", "subtract_ranges", "intersect_ranges", "plan_pulls",
           "plan_reshard", "reshard_pages", "reshard_page_steps", "RankPlan", "plan_quorum", "backed_ranges", "pool_pages", "page_ranges",
           "clip_threshold", "accum_offsets", "accum_elements", "accum_mode", "newest_complete_step", "ckpt_read_plan",
           "lr_schedule_table", "split_no_decay", "schedule_digest", "check_moment_agreement", "moment_type", "sr_bits", "bf16_sr",
           "sr_bits_ema", "bf16_sr_ema", "ema_decay_value", "ema_coefficient", "ema_step", "ema_record", "check_ema_agreement",
           "split_ema_reads", "z1_digest", "audit_every_value", "audit_stride", "decode_audit_report", "audit_findings",
           "audit_seed_source", "token_mean_factor", "token_mean_commit"]

PAGE_SHIFT = 16  # compact state: 64 Ki-element pages (256 KiB per fp32 array)
CONVERT_CHUNK = 1 << 24  # restore into the other moment type: elements converted per device temporary
GNORM_UNITS = 4096  # gradient clipping: capacity of the z1_gnorm segment in units (one fp64 partial per unit)
TOKEN_SLOTS = 2  # global token mean: published slots per rank, used alternately by consecutive commits
MAX_NO_DECAY = 4  # weight-decay exemptions per unit and update launch (kMaxNoDecay of csrc/kernels/api.h)
SR_SEED = 0x27D4EB2F  # bf16 moments: the fixed seed of the rounding bits (sr_bits of csrc/kernels/zero1.cu)
SR_SEED_EMA = 0x165667B1  # bf16 EMA of the weights: the seed of its rounding bits (sr_bits_ema of zero1.cu)


def clip_threshold(max_grad_norm: Optional[float]) -> Optional[float]:
    """The clipping threshold :class:`Zero1Optimizer` uses: ``max_grad_norm``, or env ``TORCHFT_B200_Z1_MAX_GRAD_NORM``
    when it is ``None`` (unset or empty: no clipping). ``inf`` computes the norm and vetoes non-finite steps but never
    scales; zero, negative and NaN thresholds raise ``ValueError``."""
    if max_grad_norm is None:
        env = os.environ.get("TORCHFT_B200_Z1_MAX_GRAD_NORM", "").strip()
        if not env:
            return None
        max_grad_norm = float(env)
    max_grad_norm = float(max_grad_norm)
    if not max_grad_norm > 0:
        raise ValueError(f"max_grad_norm must be > 0 (inf: compute the norm without scaling), got {max_grad_norm}")
    return max_grad_norm


# --------------------------------------------------------------------------- global token mean
def token_mean_factor(divisor: int, n: int) -> float:
    """The global token mean's factor ``f = fp32(divisor / max(N, 1))``, from integers as the commit kernel computes it:
    ``divisor = P * M * c`` is what the reduced gradient is already divided by, ``N`` the quorum's valid targets. Exactly
    1.0 when no target is ignored (``N = P * M * c``); ``divisor`` itself when there is none (every gradient is then 0)."""
    import numpy as np

    return float(np.float32(int(divisor) / max(int(n), 1)))  # int / int is the correctly rounded fp64 quotient


def token_mean_commit(published: Sequence[Tuple[int, float, int]], rows: int, divisor: int,
                      max_norm: Optional[float] = None, norm: Optional[float] = None, own: int = 0,
                      own_mean: Optional[Tuple[int, float]] = None) -> Dict[str, Any]:
    """What the commit kernel of the rank at position ``own`` computes from the quorum's published ``(n, loss, rows)``
    in rank order (a rank that does not contribute publishes ``n = 0, loss = 0``), given its own ``rows`` and
    ``divisor``: ``N`` (exact), ``f`` (:func:`token_mean_factor`), ``veto`` (some rank's rows differ from ``rows``), the
    reported ``loss`` (fp32 of ``L / max(N, 1)`` with ``L`` the fp64 sum in rank order; vetoed: ``own_mean``, the rank's
    own ``(n, loss)``, which a non-contributing rank knows though it published 0s; default: its published pair) and
    ``coef``, the coefficient the update multiplies the reduced gradient by. With clipping (``max_norm``, and ``norm``
    the fp32 norm of the reduced gradient) also ``norm``, which becomes ``fp32(norm * f)``, and ``coef = f * min(1,
    max_norm / (norm + 1e-6))`` with torch's fp32 rounding. Bit for bit what the kernel writes, on every rank alike."""
    import numpy as np

    f32 = np.float32
    n_total = sum(int(n) for n, _, _ in published)
    total = 0.0
    for _, loss, _ in published:
        total += float(loss)  # fp64, rank order
    veto = any(int(r) != int(rows) for _, _, r in published)
    f = token_mean_factor(divisor, n_total)
    out: Dict[str, Any] = {"N": n_total, "f": f, "veto": veto, "coef": f}
    if norm is not None:
        assert max_norm is not None
        g = f32(f32(norm) * f32(f))
        clip = min(f32(1.0), f32(f32(1.0) / f32(g + f32(1e-6))) * f32(max_norm))
        out["norm"], out["coef"] = float(g), float(f32(f32(f) * clip))
        veto = veto or not math.isfinite(float(g))
        out["veto"] = veto
    n_own, l_own = (int(published[own][0]), float(published[own][1])) if own_mean is None else own_mean
    out["loss"] = float(f32(l_own / max(n_own, 1))) if veto else float(f32(total / max(n_total, 1)))
    return out


# --------------------------------------------------------------------------- learning-rate schedule, decay exemptions
def lr_schedule_table(lr: float, lr_lambda: Callable[[int], float], lr_steps: int) -> Any:
    """The fp32 rates of committed updates ``1 .. lr_steps`` as a numpy array: entry ``i`` is
    ``fp32(lr * lr_lambda(i))``, evaluated in Python double -- what ``LambdaLR(opt, lr_lambda)`` sets after ``i``
    scheduler steps. Raises ``ValueError`` for ``lr_steps < 1`` and for a rate that is negative or not finite."""
    import numpy as np

    if int(lr_steps) != lr_steps or lr_steps < 1:
        raise ValueError(f"a learning-rate schedule needs lr_steps >= 1, got {lr_steps}")
    rates = [float(lr) * float(lr_lambda(i)) for i in range(int(lr_steps))]
    bad = next((i for i, x in enumerate(rates) if not (math.isfinite(x) and x >= 0)), None)
    if bad is not None:
        raise ValueError(f"the learning rate of update {bad + 1} is {rates[bad]}: it must be finite and >= 0")
    return np.asarray(rates, dtype=np.float32)


def split_no_decay(units: Sequence[Range], ranges: Sequence[Range], cap: int = MAX_NO_DECAY) -> List[List[Range]]:
    """Flat element ranges exempt from weight decay, as unit-relative ranges per unit (``units`` in their own order).
    Ranges that touch inside one unit are merged. Raises ``ValueError`` for a range that is not 8-element aligned, that
    is not inside one unit, or for more than ``cap`` ranges in one unit."""
    out: List[List[Range]] = [[] for _ in units]
    for lo, hi in sorted((int(a), int(b)) for a, b in ranges):
        if lo % 8 or hi % 8 or lo >= hi:
            raise ValueError(f"weight-decay exemption [{lo}, {hi}) must be a non-empty range of multiples of 8 elements")
        u = next((i for i, (a, b) in enumerate(units) if a <= lo < b), None)
        if u is None or hi > units[u][1]:
            raise ValueError(f"weight-decay exemption [{lo}, {hi}) is not inside one unit")
        out[u].append((lo, hi))
    for u, rs in enumerate(out):
        base = units[u][0]
        out[u] = [(lo - base, hi - base) for lo, hi in merge_ranges(rs)]
        if len(out[u]) > cap:
            raise ValueError(f"unit {u} {tuple(units[u])} has {len(out[u])} weight-decay exemptions, at most {cap} fit "
                             f"one update launch")
    return out


def schedule_digest(table: Any, no_decay: Sequence[Range]) -> str:
    """A digest of the learning-rate table's fp32 bytes (``None``: constant rate) and the merged exempt ranges, which
    every replica of a quorum must share."""
    import hashlib

    h = hashlib.sha256(b"none" if table is None else table.tobytes())
    h.update(json.dumps(merge_ranges(no_decay)).encode())
    return h.hexdigest()


# --------------------------------------------------------------------------- bf16 moments
def moment_type(moment_dtype: Optional[torch.dtype]) -> torch.dtype:
    """The dtype :class:`Zero1Optimizer` keeps ``m`` and ``v`` in: ``moment_dtype``, or env ``TORCHFT_B200_Z1_MOMENTS``
    (``fp32`` or ``bf16``; unset or empty: fp32) when it is ``None``. Anything else raises ``ValueError``."""
    if moment_dtype is None:
        env = os.environ.get("TORCHFT_B200_Z1_MOMENTS", "").strip().lower()
        moment_dtype = {"": torch.float32, "fp32": torch.float32, "bf16": torch.bfloat16}.get(env)
        if moment_dtype is None:
            raise ValueError(f"TORCHFT_B200_Z1_MOMENTS must be fp32 or bf16, got {env!r}")
    if moment_dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"moment_dtype must be torch.float32 or torch.bfloat16, got {moment_dtype}")
    return moment_dtype


def sr_bits(e: Any, t: Any, seed: int = SR_SEED) -> Any:
    """The 32 rounding bits of global element ``e`` at committed update ``t`` (numpy ``uint32``, broadcast over both):
    murmur3's 32-bit finaliser over ``lo32(e) * 0x9E3779B1 + hi32(e) * 0x85EBCA77 + t * 0xC2B2AE3D + seed`` (mod
    2**32). The low half rounds ``m``, the high half ``v``. A pure function: no state, and no dependence on rank, world,
    grid, paging or thread, so every holder of an element draws the same bits at the same update."""
    import numpy as np

    e = np.asarray(e, dtype=np.uint64)
    t = (np.asarray(t, dtype=np.int64) & 0xFFFFFFFF).astype(np.uint32)
    lo, hi = (e & np.uint64(0xFFFFFFFF)).astype(np.uint32), (e >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        x = lo * np.uint32(0x9E3779B1) + hi * np.uint32(0x85EBCA77) + t * np.uint32(0xC2B2AE3D) + np.uint32(seed)
        x = x ^ (x >> np.uint32(16))
        x = x * np.uint32(0x85EBCA6B)
        x = x ^ (x >> np.uint32(13))
        x = x * np.uint32(0xC2B2AE35)
        x = x ^ (x >> np.uint32(16))
    return x


def sr_bits_ema(e: Any, t: Any) -> Any:
    """The rounding bits of a bf16 EMA of the weights: :func:`sr_bits` with the seed ``SR_SEED_EMA``, of which the low
    half rounds element ``e``'s EMA at update ``t``. The other seed keeps them apart from the bits of ``e``'s moments."""
    return sr_bits(e, t, SR_SEED_EMA)


def bf16_sr(x: Any, e: Any, t: Any, which: int, r: Any = None) -> Any:
    """fp32 ``x`` rounded stochastically to bf16, as numpy ``uint16`` bit patterns: the 16 rounding bits ``r`` (default:
    the low half of ``sr_bits(e, t)`` for ``which = 0``, the moment ``m``, and the high half for ``which = 1``, ``v``)
    are added to ``x``'s fp32 bits and the upper 16 bits are kept. The add is on the magnitude, so ``x`` rounds away from
    zero with probability equal to the discarded fraction -- unbiased for both signs -- and a value bf16 represents
    exactly is returned unchanged for every ``r``. Inf and NaN are not added to; a NaN keeps a mantissa bit. This is the
    specification of the update kernel's rounding: ``bf16_sr`` of ``zero1.cu`` returns the same bits."""
    import numpy as np

    if which not in (0, 1):
        raise ValueError(f"which is 0 (m) or 1 (v), got {which}")
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    if r is None:
        bits = sr_bits(e, t)
        r = (bits >> np.uint32(16)) if which else (bits & np.uint32(0xFFFF))
    r = np.asarray(r, dtype=np.uint32)
    special = (u & np.uint32(0x7F800000)) == np.uint32(0x7F800000)
    nan = np.where((u & np.uint32(0x007FFFFF)) != 0, np.uint32(0x40), np.uint32(0))
    with np.errstate(over="ignore"):
        out = np.where(special, (u >> np.uint32(16)) | nan, (u + r) >> np.uint32(16))
    return out.astype(np.uint16)


def bf16_sr_ema(x: Any, e: Any, t: Any) -> Any:
    """fp32 ``x`` rounded to bf16 as the update kernel rounds a bf16 EMA of element ``e`` at update ``t``:
    :func:`bf16_sr` with the low half of ``sr_bits_ema(e, t)``."""
    import numpy as np

    return bf16_sr(x, e, t, 0, r=sr_bits_ema(e, t) & np.uint32(0xFFFF))


# --------------------------------------------------------------------------- EMA of the weights
def ema_decay_value(ema_decay: Optional[float]) -> Optional[float]:
    """The decay of the EMA :class:`Zero1Optimizer` keeps: ``ema_decay``, or env ``TORCHFT_B200_Z1_EMA_DECAY`` when it
    is ``None`` (unset or empty: no EMA). A decay outside ``(0, 1)``, or one whose ``fp32(1 - decay)`` is 0 or 1,
    raises ``ValueError``."""
    import numpy as np

    if ema_decay is None:
        env = os.environ.get("TORCHFT_B200_Z1_EMA_DECAY", "").strip()
        if not env:
            return None
        ema_decay = float(env)
    d = float(ema_decay)
    if not (0.0 < d < 1.0 and 0.0 < float(np.float32(1.0 - d)) < 1.0):
        raise ValueError(f"ema_decay must be in (0, 1) with fp32(1 - ema_decay) in (0, 1), got {ema_decay}")
    return d


def ema_coefficient(decay: float) -> float:
    """``c = fp32(1 - decay)``, rounded once on the host: the update kernel's step is ``ema + c * (w' - ema)``."""
    import numpy as np

    return float(np.float32(1.0 - float(decay)))


def ema_step(ema: Any, w: Any, c: float) -> Any:
    """The update kernel's EMA step in numpy float32, bit for bit: ``ema + c * (w - ema)``, each of the three operations
    rounded to fp32 on its own (the kernel spells them ``__fsub_rn`` / ``__fmul_rn`` / ``__fadd_rn``). A bf16 EMA stores
    ``bf16_sr_ema(ema_step(...), e, t)``."""
    import numpy as np

    ema, w = np.asarray(ema, dtype=np.float32), np.asarray(w, dtype=np.float32)
    return ema + np.float32(c) * (w - ema)


def ema_record(c: Optional[float]) -> Optional[str]:
    """What a rank publishes of its EMA in its ``z1/{rank}`` record: ``c`` as the hex of its fp32 value (``None``: no
    EMA, no key)."""
    import numpy as np

    return None if c is None else float(np.float32(c)).hex()


def check_ema_agreement(records: Dict[int, Dict[str, Any]]) -> None:
    """``RuntimeError`` when the published ``z1/{rank}`` records of a quorum disagree on the EMA of the weights
    (``ema``: its coefficient; absent: no EMA). Holders with different decays would drift apart without a sign, and a
    holder without an EMA could not serve one to a peer that keeps it; every rank reads the same records and raises
    alike, before anything is freed or pulled."""
    kinds = {r: p.get("ema") for r, p in records.items()}
    if len(set(kinds.values())) > 1:
        raise RuntimeError(f"zero1: the replicas of this quorum disagree on the EMA of the weights (coefficient per "
                           f"rank, None = no EMA: {kinds})")


def split_ema_reads(reads: Sequence[Tuple[Any, int, int, int]]) -> Tuple[List[Tuple[Any, int, int, int]], List[Range]]:
    """The EMA part of a checkpoint read plan (``(header, offset, lo, hi)`` from :func:`ckpt_read_plan`): the reads
    whose file has an ``ema`` section, and the merged ranges whose file has none, which are seeded from the master
    weights read with them."""
    have = [r for r in reads if "ema" in r[0]]
    seed = merge_ranges([(lo, hi) for h, _, lo, hi in reads if "ema" not in h])
    return have, seed


# --------------------------------------------------------------------------- replica audit
AUDIT_SEEDS = {"weights": 0x5851F42D4C957F2D, "master": 0x14057B7EF767814F, "m": 0x2545F4914F6CDD1D,
               "v": 0x27BB2EE687B0B0FD, "ema": 0x369DEA0F31A53F85}  # seed_A of z1_digest per array
AUDIT_ARRAYS = ("master", "m", "v", "ema")  # the state arrays in slot order (the EMA only when kept)
AUDIT_GOLDEN = 0x9E3779B97F4A7C15


def _fmix64(x: Any) -> Any:
    import numpy as np

    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xFF51AFD7ED558CCD)
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xC4CEB9FE1A85EC53)
        return x ^ (x >> np.uint64(33))


def z1_digest(data: Any, word0: int, seed: int) -> int:
    """The audit digest of a range of one partitioned array: ``data`` is the byte image of the range (any numpy array,
    read as its bytes, a multiple of 8 bytes) and ``word0`` the GLOBAL index of its first 8-byte word (word ``i`` is bytes
    ``[8 i, 8 i + 8)`` of the flat vector's image). The result is ``sum fmix64(w ^ (i * 0x9E3779B97F4A7C15 + seed))``
    over the little-endian words ``w`` at global index ``i``, mod 2**64, with murmur3's 64-bit finaliser ``fmix64``.
    This is the specification of ``z1_digest_kernel`` (``csrc/kernels/audit.cu``), which returns the same bits:

    * It does not depend on grid, order or thread: wraparound integer addition is associative and commutative.
    * Flat and paged state give the same digest: the index is global, and a page is a multiple of 8 elements, so no
      word straddles a page.
    * Any change confined to one word changes the digest, since ``fmix64`` (and the xor with a fixed value) is a
      bijection. Changes of two or more words collide with probability about 2**-64.
    * Every quantity is an exact integer, so the device reproduces it bit for bit."""
    import numpy as np

    w = np.ascontiguousarray(data).view(np.uint8).view("<u8").astype(np.uint64)
    i = np.arange(int(word0), int(word0) + w.size, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = _fmix64(w ^ (i * np.uint64(AUDIT_GOLDEN) + np.uint64(seed)))
    return int(x.sum(dtype=np.uint64)) if x.size else 0


def audit_every_value(audit_every: Optional[int]) -> int:
    """The audit period :class:`Zero1Optimizer` uses: ``audit_every``, or env ``TORCHFT_B200_Z1_AUDIT_EVERY`` when it is
    ``None`` (unset or empty: 0, no audit). Negative values raise ``ValueError``."""
    if audit_every is None:
        env = os.environ.get("TORCHFT_B200_Z1_AUDIT_EVERY", "").strip()
        audit_every = int(env) if env else 0
    if int(audit_every) != audit_every or audit_every < 0:
        raise ValueError(f"audit_every must be an integer >= 0 (0: no audit), got {audit_every}")
    return int(audit_every)


def audit_stride(replication: int) -> int:
    """Slots per unit in the ``z1_audit`` segment: the weights digest, then one per (held slice ``j < k``, array)."""
    return 1 + min(int(replication), 8) * len(AUDIT_ARRAYS)


def decode_audit_report(raw: bytes, nunits: int, stride: int, narrays: int, k: int) -> Dict[str, Any]:
    """The compare kernel's host-mapped report as ``{seq, mismatches, world, t, weights, state}``: ``t[r]`` is rank
    ``r``'s update count, ``weights[r][u]`` its weights digest of unit ``u`` and ``state[r][u][j][a]`` its digest of
    array ``a`` (``AUDIT_ARRAYS`` order) of its ``j``-th held slice, slice ``r - j``."""
    import numpy as np

    w = np.frombuffer(raw, dtype="<u8")
    seq, mismatches, world, n = (int(x) for x in w[:4])
    rep: Dict[str, Any] = {"seq": seq, "mismatches": mismatches, "world": world, "t": [], "weights": [], "state": []}
    if world == 0:
        return rep
    assert n == nunits * stride + 1, "the report was written for another slot layout"
    slots = w[4:4 + world * n].reshape(world, n)
    for r in range(world):
        rep["t"].append(int(slots[r, -1]))
        rep["weights"].append([int(slots[r, u * stride]) for u in range(nunits)])
        rep["state"].append([[[int(slots[r, u * stride + 1 + j * narrays + a]) for a in range(narrays)] for j in range(k)]
                             for u in range(nunits)])
    return rep


def _outside_majority(digests: Dict[int, Any]) -> List[int]:
    """The ranks whose digest is not that of a strict majority (all of them when there is none)."""
    counts: Dict[Any, int] = {}
    for d in digests.values():
        counts[d] = counts.get(d, 0) + 1
    top = max(counts, key=lambda d: counts[d])
    if 2 * counts[top] <= len(digests):
        return sorted(digests)
    return sorted(r for r, d in digests.items() if d != top)


def audit_seed_source(published: Dict[int, Dict[str, Any]]) -> int:
    """The rank whose bf16 weights the holders of a slice that a diverged audit condemned re-seed it from: the lowest
    rank of the new quorum at its highest update count. Every rank reads the same published records, so every rank picks
    the same one; a joiner (behind, and about to be healed) is never picked."""
    tmax = max(int(p["t"]) for p in published.values())
    return min(r for r, p in published.items() if int(p["t"]) == tmax)


def audit_findings(report: Dict[str, Any], layout: ShardLayout, world: int) -> Tuple[List[Dict[str, Any]], Dict[int, List[Range]]]:
    """What a decoded audit report (:func:`decode_audit_report`) of a quorum of ``world`` ranks says: the findings, one
    per group whose digests disagree, as ``{unit, array, slice, ranks, t}`` (``slice`` is ``None`` for the weights), and
    per rank the ranges it must stop claiming. Only ranks at the quorum's highest update count are compared.

    For each (unit, slice, array) whose holders disagree, the holders outside a strict majority drop the slice; with no
    strict majority (e.g. ``k = 2``) every holder drops it, and the next re-shard re-seeds it. Weights mismatches drop
    nothing: the first update of the next quorum re-broadcasts every unit from the master weights.

    A rank whose row is all zeros (its next audit's memset ran before this rank's compare read it, which a rank whose
    error is already latched can do) is compared as a holder whose digests match nobody, not left out: so a report with
    zeroed rows makes every other rank drop at least what the complete report would, never less."""
    t = report["t"]
    drops: Dict[int, List[Range]] = {r: [] for r in range(world)}
    findings: List[Dict[str, Any]] = []
    if not t:
        return findings, drops
    tmax = max(t)
    zeroed = {r for r in range(world) if not any(report["weights"][r])}  # a unit's digest is 0 with probability 2**-64
    part = [r for r in range(world) if t[r] == tmax or r in zeroed]

    def digest(x: int, r: int) -> Any:
        return ("zeroed", r) if r in zeroed else x

    k = layout.k(world)
    narrays = len(report["state"][0][0][0]) if k > 1 else 0
    for u in range(len(layout.units)):
        w = {r: digest(report["weights"][r][u], r) for r in part}
        if len(set(w.values())) > 1:
            findings.append({"unit": u, "array": "weights", "slice": None, "ranks": _outside_majority(w), "t": tmax})
        if k < 2:
            continue
        for s in range(world):
            lo, hi = layout.slice_bounds(u, world, s)
            holders = [h for h in layout.holders(u, world, s) if h in part]
            for a in range(narrays):
                d = {h: digest(report["state"][h][u][(h - s) % world][a], h) for h in holders}
                if len(set(d.values())) > 1:
                    out = _outside_majority(d)
                    findings.append({"unit": u, "array": AUDIT_ARRAYS[a], "slice": s, "ranks": out, "t": tmax})
                    for h in out:
                        if hi > lo:
                            drops[h].append((lo, hi))
    return findings, {r: merge_ranges(x) for r, x in drops.items()}


# --------------------------------------------------------------------------- interval arithmetic
def merge_ranges(rs: Sequence[Range]) -> List[Range]:
    """Sorted, coalesced, non-empty half-open ranges."""
    out: List[Range] = []
    for lo, hi in sorted((int(a), int(b)) for a, b in rs if b > a):
        if out and lo <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], hi))
        else:
            out.append((lo, hi))
    return out


def intersect_ranges(a: Sequence[Range], b: Sequence[Range]) -> List[Range]:
    a, b = merge_ranges(a), merge_ranges(b)
    out: List[Range] = []
    i = j = 0
    while i < len(a) and j < len(b):
        lo, hi = max(a[i][0], b[j][0]), min(a[i][1], b[j][1])
        if lo < hi:
            out.append((lo, hi))
        if a[i][1] < b[j][1]:
            i += 1
        else:
            j += 1
    return out


def subtract_ranges(a: Sequence[Range], b: Sequence[Range]) -> List[Range]:
    """``a`` minus ``b``."""
    out: List[Range] = []
    b = merge_ranges(b)
    for lo, hi in merge_ranges(a):
        cur = lo
        for blo, bhi in b:
            if bhi <= cur or blo >= hi:
                continue
            if blo > cur:
                out.append((cur, blo))
            cur = max(cur, bhi)
            if cur >= hi:
                break
        if cur < hi:
            out.append((cur, hi))
    return out


def total(rs: Sequence[Range]) -> int:
    return sum(hi - lo for lo, hi in rs)


# --------------------------------------------------------------------------- ownership
@dataclass(frozen=True)
class ShardLayout:
    """Which element ranges of the flat parameter vector a quorum rank holds optimizer state for.

    ``units`` are contiguous element ranges (multiples of 8 elements) tiling the flat buffer. Unit
    ``u`` is cut into ``world`` slices of ``ceil(nvec / world)`` 16-byte vectors (the arithmetic of
    ``Geo`` in ``zero1.cu``); slice ``s`` has primary holder ``s`` and buddies ``s+1 .. s+k-1``.
    """

    units: Tuple[Range, ...]
    replication: int = 2

    def slice_bounds(self, unit: int, world: int, s: int) -> Range:
        lo, hi = self.units[unit]
        nvec = (hi - lo) // 8
        per = (nvec + world - 1) // world
        a, b = min(s * per, nvec), min((s + 1) * per, nvec)
        return lo + a * 8, lo + b * 8

    def k(self, world: int) -> int:
        return max(1, min(self.replication, world))

    def primary(self, rank: int, world: int) -> List[Range]:
        return merge_ranges([self.slice_bounds(u, world, rank) for u in range(len(self.units))])

    def held(self, rank: int, world: int) -> List[Range]:
        """Ranges whose (master, m, v) this rank keeps up to date: its primary slices and the slices it backs up."""
        out: List[Range] = []
        for u in range(len(self.units)):
            for j in range(self.k(world)):
                out.append(self.slice_bounds(u, world, (rank - j) % world))
        return merge_ranges(out)

    def holders(self, unit: int, world: int, s: int) -> List[int]:
        return [(s + j) % world for j in range(self.k(world))]


def check_moment_agreement(records: Dict[int, Dict[str, Any]]) -> None:
    """``RuntimeError`` when the published ``z1/{rank}`` records of a quorum name different moment types (``moments``;
    absent: fp32). Holders of one slice would round the same moments differently and drift apart without a sign, and a
    pull would copy the wrong number of bytes; every rank reads the same records and raises alike, before anything is
    freed or pulled."""
    kinds = {r: p.get("moments", "fp32") for r, p in records.items()}
    if len(set(kinds.values())) > 1:
        raise RuntimeError(f"zero1: the replicas of this quorum disagree on the type of the optimizer moments "
                           f"(per rank: {kinds})")


def plan_pulls(need: Sequence[Range], holdings: Dict[int, Sequence[Range]], me: int) -> Tuple[List[Tuple[int, int, int]], List[Range]]:
    """Cover ``need`` from peers' ``holdings``: ``[(src_rank, lo, hi), ...]`` plus the ranges nobody holds.

    Sources are tried in the order ``me+1, me+2, ...`` so concurrent pullers spread over different peers.
    """
    pulls: List[Tuple[int, int, int]] = []
    left = merge_ranges(need)
    ranks = sorted(r for r in holdings if r != me)
    if ranks:
        start = next((i for i, r in enumerate(ranks) if r > me), 0)
        ranks = ranks[start:] + ranks[:start]
    for r in ranks:
        if not left:
            break
        got = intersect_ranges(left, holdings[r])
        for lo, hi in got:
            pulls.append((r, lo, hi))
        left = subtract_ranges(left, got)
    return pulls, left


# --------------------------------------------------------------------------- durable checkpoints
def newest_complete_step(headers: Sequence[Dict[str, Any]], numel: int) -> Optional[int]:
    """The newest update count ``T`` whose checkpoint files together cover ``[0, numel)`` (``None``: there is none).
    ``headers[i]`` has ``T`` and the written ``ranges`` (``[lo, hi, offset]``). Files of one ``T`` may come from quorums
    of different sizes: holders at the same update count hold the same bits. An update count whose files name
    different moment types (``moments``; absent: fp32) does not count."""
    by_t: Dict[int, List[Range]] = {}
    kinds: Dict[int, set] = {}
    for h in headers:
        by_t.setdefault(int(h["T"]), []).extend((int(lo), int(hi)) for lo, hi, _ in h["ranges"])
        kinds.setdefault(int(h["T"]), set()).add(h.get("moments", "fp32"))
    for t in sorted(by_t, reverse=True):
        # one quorum writes one moment type; an update count with files of both is not one quorum's and is passed over
        if merge_ranges(by_t[t]) == [(0, numel)] and len(kinds[t]) == 1:
            return t
    return None


def ckpt_read_plan(need: Sequence[Range], files: Sequence[Tuple[Any, Sequence[Tuple[int, int, int]]]]
                   ) -> List[Tuple[Any, int, int, int]]:
    """Cover ``need`` from checkpoint files of one update count: ``[(file, offset, lo, hi), ...]`` reads elements
    ``[lo, hi)`` of the flat vector from element ``offset`` of ``file``'s arrays. ``files[i] = (file, ranges)`` with the
    written ``ranges`` as ``(lo, hi, offset)``; earlier files are preferred. Raises ``ValueError`` when the files do not
    cover ``need``."""
    reads: List[Tuple[Any, int, int, int]] = []
    left = merge_ranges(need)
    for f, ranges in files:
        if not left:
            break
        for lo, hi, off in ranges:
            for a, b in intersect_ranges(left, [(lo, hi)]):
                reads.append((f, int(off) + a - int(lo), a, b))
        left = subtract_ranges(left, [(lo, hi) for lo, hi, _ in ranges])
    if left:
        raise ValueError(f"the checkpoint files do not cover {left}")
    return reads


# --------------------------------------------------------------------------- compact (paged) state
def page_ranges(rs: Sequence[Range], shift: int) -> List[Range]:
    """Page indices (as merged half-open ranges) that element ranges ``rs`` touch, for pages of ``2**shift`` elements."""
    return merge_ranges([(lo >> shift, ((hi - 1) >> shift) + 1) for lo, hi in rs if hi > lo])


def backed_ranges(rs: Sequence[Range], pages: Sequence[Range], shift: int) -> List[Range]:
    """The parts of element ranges ``rs`` that lie in ``pages`` (page-index ranges of ``2**shift`` elements)."""
    return intersect_ranges(rs, [(lo << shift, hi << shift) for lo, hi in pages])


def reshard_page_steps(old_pages: Sequence[Range], new_pages: Sequence[Range], source_pages: Sequence[Range]
                       ) -> Tuple[List[Range], List[Range], List[Range]]:
    """The page sets of one rank's compact re-shard, in the order it applies them: ``(free_first, allocate,
    free_last)``. ``free_first`` are the old pages that are neither kept nor read by a peer, ``allocate`` the new pages
    it did not have, and ``free_last`` the old pages kept only for peers, which go once every peer has pulled."""
    free_first = subtract_ranges(old_pages, merge_ranges(list(new_pages) + list(source_pages)))
    allocate = subtract_ranges(new_pages, old_pages)
    free_last = intersect_ranges(subtract_ranges(source_pages, new_pages), old_pages)
    return free_first, allocate, free_last


def plan_reshard(layout: ShardLayout, peers: Dict[int, Tuple[int, Sequence[Range]]], world: int
                 ) -> Tuple[int, Dict[int, Tuple[List[Range], List[Tuple[int, int, int]], List[Range]]]]:
    """Every rank's re-shard for a new quorum, from what each rank published (``peers[r] = (t, holdings)``): the
    update count ``tmax`` the quorum agrees on and ``{rank: (need, pulls, lost)}``. Only holdings at ``tmax`` count;
    a rank that missed an update holds nothing. This is what each rank of :class:`Zero1Optimizer` plans for itself, so
    any rank can tell which of its ranges its peers are about to read."""
    tmax = max(int(t) for t, _ in peers.values())
    valid = {r: list(h) for r, (t, h) in peers.items() if int(t) == tmax}
    plans = {}
    for r in range(world):
        need = subtract_ranges(layout.held(r, world), valid.get(r, []))
        pulls, lost = plan_pulls(need, {q: h for q, h in valid.items() if q != r}, r)
        plans[r] = (need, pulls, lost)
    return tmax, plans


def reshard_pages(layout: ShardLayout, plans: Dict[int, Tuple[List[Range], List[Tuple[int, int, int]], List[Range]]],
                  old_pages: Dict[int, Sequence[Range]], world: int, shift: int) -> Dict[int, Tuple[List[Range], List[Range], int]]:
    """Per rank ``(new_pages, source_pages, peak)`` of a compact re-shard: the pages it holds afterwards, the pages of
    its old state that peers pull from, and the most pages it has allocated at once when it frees every page that is
    neither kept nor a source before it allocates, and frees the sources only after every peer has pulled."""
    sources: Dict[int, List[Range]] = {r: [] for r in range(world)}
    for _, pulls, _ in plans.values():
        for src, lo, hi in pulls:
            sources[src].append((lo, hi))
    out = {}
    for r in range(world):
        new = page_ranges(layout.held(r, world), shift)
        src = page_ranges(sources[r], shift)
        out[r] = (new, src, total(merge_ranges(new + intersect_ranges(old_pages.get(r, []), src))))
    return out


@dataclass
class RankPlan:
    """One rank's part of a quorum change (:func:`plan_quorum`), in the order the re-shard applies it."""

    tmax: int                                # the update count the quorum agrees on
    need: List[Range]                        # held in the new layout and not current here
    pulls: List[Tuple[int, int, int]]        # ``(source rank, lo, hi)``: the parts of ``need`` a peer at ``tmax`` has
    reads: List[Tuple[Any, int, int, int]]   # ``(file, offset, lo, hi)``: what no peer has, from a checkpoint at tmax
    lost: List[Range]                        # what nobody has: re-seeded from the bf16 weights
    counted: bool                            # whether ``lost`` is a loss (at t = 0 the seed IS the state)
    hold: List[Range]                        # the ranges the rank claims afterwards
    hold_mid: List[Range]                    # ... while the re-shard runs (paged: after ``free_first``)
    free_first: List[Range] = ()             # paged: old pages neither kept nor read by a peer
    allocate: List[Range] = ()               # paged: new pages it did not have
    free_last: List[Range] = ()              # paged: old pages kept only for peers, freed once every peer has pulled
    peak: int = 0                            # paged: the most pages it has allocated at once


def _ckpt_reads(lost: Sequence[Range], rank: int, ckpt: Dict[int, Any]) -> List[Tuple[Any, int, int, int]]:
    if not lost:
        return []
    for q in sorted(ckpt, key=lambda q: (q != rank, q)):  # its own restore first
        try:
            return ckpt_read_plan(lost, ckpt[q])
        except ValueError:
            continue
    return []


def plan_quorum(layout: ShardLayout, world: int, published: Dict[int, Dict[str, Any]], shift: Optional[int] = None,
                ckpt: Optional[Dict[int, Any]] = None) -> Dict[int, RankPlan]:
    """Every rank's re-shard for a new quorum of ``world``, from what each rank published: ``published[r]`` has its
    update count ``t``, its holdings ``hold`` and, for paged state (``shift`` = log2 of the page size), its page table
    as ``pages`` runs ``(page, slot, count)``. Only holdings at the highest ``t`` count; a rank that missed an update
    holds nothing. ``ckpt[r]`` are the files at that update count of the checkpoint rank ``r`` restored from, as
    ``(file, ranges)`` for :func:`ckpt_read_plan`: a rank reads what no peer has from its own, else from the first one
    that covers it. Every rank of :class:`Zero1Optimizer` plans every rank, so it knows which of its ranges its peers
    are about to read.

    Full-size state keeps every range it held at the highest ``t`` (also those outside the new layout: peers may pull
    them later). Paged state holds exactly its new slices; while its re-shard runs it claims only the held ranges its
    kept pages still back, so a re-shard that dies before its barrier leaves no claim on a page it gave back."""
    tmax, base = plan_reshard(layout, {r: (p["t"], [tuple(x) for x in p["hold"]]) for r, p in published.items()}, world)
    if shift is not None:
        old = {r: merge_ranges([(pg, pg + n) for pg, _, n in p["pages"]]) for r, p in published.items()}
        pages = reshard_pages(layout, base, old, world, shift)
    plans: Dict[int, RankPlan] = {}
    for r, (need, pulls, lost) in base.items():
        hold = [tuple(x) for x in published[r]["hold"]]
        mine = hold if int(published[r]["t"]) == tmax else []
        reads = _ckpt_reads(lost, r, ckpt or {})
        p = plans[r] = RankPlan(tmax, need, pulls, reads, [] if reads else lost, tmax > 0,
                                layout.held(r, world) if shift is not None else merge_ranges(mine + need), hold)
        if shift is not None:
            new, src, p.peak = pages[r]
            p.free_first, p.allocate, p.free_last = reshard_page_steps(old[r], new, src)
            p.hold_mid = backed_ranges(hold, subtract_ranges(old[r], p.free_first), shift)
    return plans


def pool_pages(layout: ShardLayout, min_world: int, page: int = 1 << PAGE_SHIFT, max_world: int = 8) -> int:
    """Pages per state array that let every rank hold its slices at every world in ``[min_world, max_world]`` and ride
    through every single-member loss or join between those worlds (the re-shard peak), for steady-state holders
    that are all up to date."""
    shift = page.bit_length() - 1
    assert page == 1 << shift and page % 8 == 0, "a page is a power of two and a multiple of 8 elements"
    if not 1 <= min_world <= max_world:
        raise ValueError(f"min_world must be in [1, {max_world}]")

    def held_pages(world: int) -> List[List[Range]]:
        return [page_ranges(layout.held(r, world), shift) for r in range(world)]

    best = max(total(p) for w in range(min_world, max_world + 1) for p in held_pages(w))
    for w in range(min_world, max_world + 1):
        old = [{"t": 1, "hold": layout.held(r, w), "pages": [(lo, 0, hi - lo) for lo, hi in pg]}
               for r, pg in enumerate(held_pages(w))]
        transitions = []
        if w - 1 >= min_world:  # member ``d`` is lost
            transitions += [[old[r] for r in range(w) if r != d] for d in range(w)]
        if w + 1 <= max_world:  # a member with no state joins at quorum rank ``j``
            transitions += [old[:j] + [{"t": 0, "hold": [], "pages": []}] + old[j:] for j in range(w + 1)]
        for members in transitions:
            plans = plan_quorum(layout, len(members), dict(enumerate(members)), shift)
            best = max(best, max(p.peak for p in plans.values()))
    return best


# --------------------------------------------------------------------------- gradient accumulation
def accum_offsets(layout: ShardLayout, rank: int, world: int) -> Tuple[List[int], int]:
    """Where each unit's primary slice of quorum rank ``rank`` lives in its fp32 accumulator: per-unit offsets in
    elements, in unit order, and the elements the accumulator needs. The slices are packed back to back; each is a
    multiple of 8 elements, so every offset is 32-byte aligned."""
    offsets, n = [], 0
    for u in range(len(layout.units)):
        offsets.append(n)
        lo, hi = layout.slice_bounds(u, world, rank)
        n += hi - lo
    return offsets, n


def accum_elements(layout: ShardLayout, min_world: int, max_world: int = 8) -> int:
    """Accumulator elements that hold any rank's primary slices at every world in ``[min_world, max_world]``."""
    if not 1 <= min_world <= max_world:
        raise ValueError(f"min_world must be in [1, {max_world}]")
    return max(accum_offsets(layout, r, w)[1] for w in range(min_world, max_world + 1) for r in range(w))


def accum_mode(micro: int, steps: int) -> int:
    """``acc_mode`` of the reduce launch for micro-batch ``micro`` of ``steps``: 0 without accumulation (``steps`` = 1),
    1 for the first micro-batch (stores), 2 for the middle ones (add), 3 for the last (reduces to bf16)."""
    if steps < 1 or not 0 <= micro < steps:
        raise ValueError(f"micro-batch {micro} is not in [0, {steps})")
    if steps == 1:
        return 0
    return 1 if micro == 0 else (3 if micro == steps - 1 else 2)


# --------------------------------------------------------------------------- the optimizer
class Zero1Optimizer:
    """AdamW with fp32 master and fp32 or bf16 m/v partitioned over the replicas of the current quorum (see module doc).

    All five flat buffers live in NVLink-symmetric segments of the process group: ``param`` and ``grad``
    (bf16; written/read by peers every step) and ``master``/``m``/``v`` (fp32; read by peers only when
    ownership moves). By default the state arrays are full-size and addressed by GLOBAL element index -- only the
    held ranges are kept up to date -- which makes re-sharding a plain ranged copy.

    With ``compact=True`` the state arrays are pools of fixed-size pages instead, and a page table maps each page of
    the flat vector that this rank holds to a pool slot: a rank stores only about ``k/W`` of the state. The pool is
    sized for every world in ``[min_world, 8]`` including the re-shard peaks between them (:func:`pool_pages`); a quorum
    below ``min_world`` or a plan that does not fit raises instead of dropping state. A compact re-shard completes
    inside ``configure`` (it frees and reuses pages, so it synchronises with its peers before it returns).

    With ``max_grad_norm`` the global L2 norm of the reduced bf16 gradient is computed on the device inside the same
    three kernels (no extra launch, no host sync): the reduce-scatter sums the squares of the slice it produces, the
    commit kernel adds every rank's partials in rank order -- so every replica gets the same bits -- and the update
    scales the gradient by ``min(1, max_grad_norm / (norm + 1e-6))``. A step whose norm is not finite is vetoed on
    every replica (counted in ``nonfinite_steps``): no state changes and ``t`` does not advance. ``grad_norm`` is the
    device scalar of the last commit, ``last_grad_norm`` the host value of the last resolved step.

    With ``global_token_mean`` the step applies the gradient of the mean loss over every valid target of the quorum
    instead of the mean of the replicas' (and micro-batches') own means. Before each commit the caller hands
    :meth:`publish_tokens` this rank's count of valid targets ``n``, its loss sum ``L`` (losses normalised by the row
    count ``c = B * S`` of a micro-batch, so ``L = sum_m loss_m * c``) and its shape. The commit kernel publishes them in
    the small ``z1_tokmean`` segment, sums the quorum's counts ``N`` and losses in rank order and folds
    ``f = fp32(P * M * c / max(N, 1))`` into the coefficient the update multiplies the reduced gradient by (with clipping
    the norm is ``f`` times the reduced gradient's and the coefficient ``f`` times the clip coefficient). With no ignored
    target ``f`` is exactly 1 and the step is bit-identical to one without the mode. Ranks whose ``M * B * S`` differ
    veto the step on every rank (counted in ``row_mismatch_steps``). :meth:`token_mean_loss` gives ``L / N`` of the last
    commit, the same bits on every rank of a committed step.

    With ``grad_accum_steps = M > 1`` one step reduces ``M`` micro-batches: :meth:`reduce_scatter` takes the micro-batch
    index, micro-batches ``0 .. M-2`` add their fp32 reduced slice into an accumulator that covers only this rank's
    primary slices (an ordinary device tensor of about ``4 * numel / min_world`` bytes, :meth:`accum_bytes`), and the
    last one adds its own, scales by the caller's ``scale`` and rounds to bf16 once. The first micro-batch of a step
    overwrites the accumulator, so nothing of an aborted step survives into the next. A step in which some unit was
    not reduced ``M`` times is vetoed (:meth:`enqueue`).

    Durable checkpoints (:meth:`save` / :meth:`restore`, format in ``checkpointing/sharded.py``): every replica writes
    the bf16 weights and (master, m, v) over its primary slices at one committed update count ``T``, so the files of
    one quorum tile the flat vector. The snapshot is a device-to-host copy on its own stream, unit by unit behind that
    unit's update; the next update of a unit waits for its copy, and a re-shard waits on the host for the whole
    snapshot, so forward and backward of the next step run under the copy. :meth:`restore` reads the weights, sets
    ``t = T`` and claims no state; the next re-shard reads the ranges that no live holder at ``T`` has from the files,
    instead of re-seeding them. Without a save nothing is allocated and :meth:`update` launches and waits as before.

    Args:
        pg: a ``ProcessGroupB200`` (symmetric segments must be allocated before its first ``configure``)
        numel: elements of the flat parameter vector (multiple of 8)
        units: element ranges in FORWARD order that tile ``[0, numel)`` (one per transformer block)
        replication: holders per slice (``k``); ``min(k, world)`` is used
        compact: paged state (``None``: env ``TORCHFT_B200_Z1_COMPACT=1`` turns it on)
        min_world: compact: the smallest quorum the pool must hold the state for
        state_pages: compact: pool size in pages, overriding :func:`pool_pages`
        page_shift: compact: pages of ``2**page_shift`` elements
        max_grad_norm: clip the global gradient norm to this (``inf``: only veto non-finite steps; ``None``: env
            ``TORCHFT_B200_Z1_MAX_GRAD_NORM``, unset = no clipping)
        grad_accum_steps: micro-batches per step (``M``); the accumulator is sized for every world in
            ``[min_world, 8]``
        lr_lambda: learning-rate schedule: committed update ``t`` (1-based, the device's count) uses
            ``fp32(lr * lr_lambda(min(t, lr_steps) - 1))``, what ``LambdaLR`` gives when stepped after every committed
            step. The rates are tabulated once here (``lr`` is then the base rate, read once); ``None``: the constant
            ``param_groups[0]["lr"]``, read at every :meth:`update`.
        lr_steps: entries of the table; later updates keep the last rate
        no_decay: flat element ranges (multiples of 8, each inside one unit, at most ``MAX_NO_DECAY`` per unit) whose
            elements get no weight decay
        moment_dtype: ``torch.float32`` (default) or ``torch.bfloat16`` for ``m`` and ``v`` (``None``: env
            ``TORCHFT_B200_Z1_MOMENTS=bf16``). bf16 moments take 8 instead of 12 bytes of state per element; the update
            computes in fp32 and rounds them stochastically (:func:`bf16_sr`) with bits that depend only on the element
            index and the committed update count, so the holders of a slice stay bit-identical. ``master`` stays fp32.
            Every replica of a quorum must use the same type. A checkpoint of the other type is converted on restore.
        ema_decay: keep an exponential moving average of the fp32 master weights with this decay ``d`` in ``(0, 1)``
            (``None``: env ``TORCHFT_B200_Z1_EMA_DECAY``, unset = no EMA). It is partitioned state like ``m`` and ``v``
            and of their type (bf16: rounded stochastically with bits of its own): the holders of a slice advance it in
            the update kernel after every committed update, ``ema + fp32(1 - d) * (w' - ema)``; re-shards, heals and
            checkpoints carry it; it is seeded from the weights wherever the master weights are. :meth:`ema_weights`
            swaps it into ``param`` for evaluation. Every replica of a quorum must use the same decay.
        audit_every: every ``N``-th :meth:`update` since the last quorum change, audit replica consistency on the device
            (``None``: env ``TORCHFT_B200_Z1_AUDIT_EVERY``, unset = 0, no audit). Behind the last unit's update, on the
            commit stream, a kernel digests this rank's bf16 weights of every unit and each held slice of every state
            array (:func:`z1_digest`) into its ``z1_audit`` slots; behind a handshake, a one-CTA kernel compares every
            rank's slots: the weights of all ranks at the quorum's update count, and the state of each slice's holders.
            A disagreement latches an error (``kErrDiverged``) that fails the next commit on every rank; at the next
            quorum the holders outside a strict majority of a diverged slice stop claiming it (:func:`audit_findings`),
            so it is pulled from the majority or re-seeded, and the weights are re-broadcast from the masters. With
            ``k = 1`` only the weights are compared; at world 1 nothing is audited. ``audits``, ``divergences`` and
            ``last_audit`` (the decoded report, :meth:`audit_report`) tell what it found. Every replica of a quorum must
            use the same period.
        global_token_mean: average over every valid target of the quorum (see above); every replica of a quorum must
            use it alike (the ``z1_tokmean`` segment is allocated only with it)
    """

    def __init__(self, pg: Any, numel: int, units: Optional[Sequence[Range]] = None, lr: float = 3e-4,
                 betas: Tuple[float, float] = (0.9, 0.95), eps: float = 1e-8, weight_decay: float = 0.1,
                 replication: int = 2, blocks: Optional[int] = None, compact: Optional[bool] = None, min_world: int = 1,
                 state_pages: Optional[int] = None, page_shift: int = PAGE_SHIFT,
                 max_grad_norm: Optional[float] = None, grad_accum_steps: int = 1,
                 lr_lambda: Optional[Callable[[int], float]] = None, lr_steps: int = 0,
                 no_decay: Sequence[Range] = (), moment_dtype: Optional[torch.dtype] = None,
                 ema_decay: Optional[float] = None, audit_every: Optional[int] = None,
                 global_token_mean: bool = False) -> None:
        from torchft_b200.ops import _native

        self.moment_dtype = moment_type(moment_dtype)
        self._msize = 2 if self.moment_dtype == torch.bfloat16 else 4  # bytes per element of m and of v
        self.ema_decay = ema_decay_value(ema_decay)
        self._ema_c = None if self.ema_decay is None else ema_coefficient(self.ema_decay)
        self.ema: Optional[torch.Tensor] = None  # EMA of the weights, of the moment type, indexed like master
        self._ema_active = False                 # inside ema_weights(): param holds bf16(EMA)
        self.max_grad_norm = clip_threshold(max_grad_norm)
        self.audit_every = audit_every_value(audit_every)
        self.audits = 0                  # audits enqueued
        self.divergences = 0             # audits whose report showed replicas or holders that disagree
        self.last_audit: Optional[Dict[str, Any]] = None  # the last decoded report (audit_report)
        self._audit_report: Any = None   # host-mapped words the compare kernel writes (allocated at the first audit)
        self._audit_event: Optional[torch.cuda.Event] = None  # the last audit's compare has run
        self._audit_seq = 0              # sequence number of the last audit enqueued
        self._audit_seen = 0             # ... and of the last report a re-shard acted on
        self._audit_quorums: Dict[int, Tuple[int, int]] = {}  # audit seq -> (rank, world) it ran at
        self._audit_table: Optional[Tuple[Tuple[int, int], torch.Tensor, int, int]] = None  # digest table of (rank, world)
        self._audit_dropped: List[Range] = []  # ranges the last re-shard stopped claiming after a diverged audit
        self._updates_since_config = 0   # update() calls since the last quorum change: the same count on every rank
        # learning-rate schedule: fp32 rate of committed update i + 1 at index i (host copy and device table)
        self._lr_host = lr_schedule_table(lr, lr_lambda, lr_steps) if lr_lambda is not None else None
        self.no_decay: List[Range] = [(int(a), int(b)) for a, b in no_decay]  # split by unit in set_units
        self._nd_units: Optional[List[List[Range]]] = None  # ... unit-relative ranges per unit
        if int(grad_accum_steps) != grad_accum_steps or grad_accum_steps < 1:
            raise ValueError(f"grad_accum_steps must be an integer >= 1, got {grad_accum_steps}")
        self.grad_accum_steps = int(grad_accum_steps)
        self._acc: Optional[torch.Tensor] = None      # accumulation: fp32 primary slices of this rank, packed
        self._acc_offsets: List[int] = []             # ... element offset of each unit's slice in it
        self._acc_for: Optional[Tuple[int, int]] = None  # ... the (rank, world) the offsets were computed for
        assert numel % 8 == 0
        self._K = _native.load()
        self.pg = pg
        self.comm = pg.comm
        self.device = pg.comm.device
        self.numel = numel
        self._replication = int(replication)
        self.layout: ShardLayout = ShardLayout(((0, numel),), self._replication)
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]
        self._lr_tab: Optional[torch.Tensor] = None
        if self._lr_host is not None:
            # a synchronous copy: the table is on the device before any update can be enqueued on any stream
            self._lr_tab = torch.from_numpy(self._lr_host).to(self.device)
            torch.cuda.current_stream(self.device).synchronize()
        # the big kernels are sync-free, so their grids are free parameters: the reduce-scatter is NVLink-latency bound
        # and shares the SMs with backward; the update is HBM-bound and likes many short CTAs (cf. the AdamW cap sweep)
        self._rs_blocks = 128
        self._upd_blocks = blocks or self._K.NUM_SMS * 16
        if compact is None:
            compact = os.environ.get("TORCHFT_B200_Z1_COMPACT", "0") == "1"
        self.compact = bool(compact)
        self.min_world = int(min_world)
        self.param = pg.alloc_symmetric("z1_param", numel * 2).view(torch.bfloat16)
        self.grad = pg.alloc_symmetric("z1_grad", numel * 2).view(torch.bfloat16)
        self.grad_norm: Optional[torch.Tensor] = None  # clipping: device fp32 norm of the last commit
        self.last_grad_norm: Optional[float] = None    # clipping: host norm of the last resolved step
        self.nonfinite_steps = 0                       # clipping: steps vetoed because the norm was inf / nan
        if self.audit_every:
            # one u64 slot per (unit, weights | held slice x array), and the update count; peers read them in the compare
            self._audit_stride = audit_stride(self._replication)
            self._audit_slots = pg.alloc_symmetric("z1_audit", (GNORM_UNITS * self._audit_stride + 1) * 8)
        if self.max_grad_norm is not None:
            # symmetric segments are zero-filled at allocation, so the FlatParams.ALIGN padding of z1_grad, which no
            # wgrad GEMM writes, adds nothing to the norm. One fp64 partial per unit; peers read them in the commit.
            self._gnorm = pg.alloc_symmetric("z1_gnorm", GNORM_UNITS * 8).view(torch.float64)[:GNORM_UNITS]
            self._clip = torch.zeros(2, dtype=torch.float32, device=self.device)  # [norm, coef] of the last commit
            self.grad_norm = self._clip[0]
            self._resolved_norm: Optional[float] = None
        self.global_token_mean = bool(global_token_mean)
        self.row_mismatch_steps = 0      # token mean: steps vetoed because the ranks' M * B * S differed
        self._tok_pending: Optional[Tuple[torch.Tensor, torch.Tensor, int, int, bool]] = None  # publish_tokens()
        self._tok_commits = 0            # commits since the last quorum change: their parity picks the slot
        self._resolved_reason: Optional[int] = None
        if self.global_token_mean:
            # two slots per rank (zero1_commit_kernel explains why two are enough); [N] and [L / N, f] of the last commit
            self._tok_slots = pg.alloc_symmetric("z1_tokmean", TOKEN_SLOTS * self._K.ZERO1_TOKSLOT_BYTES)
            self._tok_count = torch.zeros(1, dtype=torch.int64, device=self.device)
            self._tok_out = torch.zeros(2, dtype=torch.float32, device=self.device)
            if self.max_grad_norm is None:
                self._clip = torch.zeros(2, dtype=torch.float32, device=self.device)  # [unused, f]: the coefficient
        # element e of the flat vector lives at pool index (table[e >> shift] << shift) | (e & mask) of paged state; full-size
        # state has no table and keeps it at e (see _pieces)
        self._table: Optional[torch.Tensor] = None
        self._table_host: Any = None
        if not self.compact:
            self.master = pg.alloc_symmetric("z1_master", numel * 4).view(torch.float32)
            self.m = pg.alloc_symmetric("z1_m", numel * self._msize).view(self.moment_dtype)
            self.v = pg.alloc_symmetric("z1_v", numel * self._msize).view(self.moment_dtype)
            if self.ema_decay is not None:
                self.ema = pg.alloc_symmetric("z1_ema", numel * self._msize).view(self.moment_dtype)
        else:
            self.master = torch.empty(0, dtype=torch.float32, device=self.device)  # set_units allocates
            self.m = self.v = torch.empty(0, dtype=self.moment_dtype, device=self.device)
            if self.ema_decay is not None:
                self.ema = self.m
            if not 1 <= self.min_world <= 8:
                raise ValueError("min_world must be in [1, 8]")
            self._page_shift = int(page_shift)
            self._page = 1 << self._page_shift
            if self._page < 8:
                raise ValueError("a page holds at least 8 elements")
            self._state_pages = state_pages
            self.capacity = 0  # pool pages per state array, fixed by set_units (they decide the re-shard peak)
        # gate[0]: verdict of the last commit, gate[1]: applied updates (AdamW's t), both written on the device
        self.gate = torch.zeros(2, dtype=torch.int32, device=self.device)
        self.t = 0                       # host mirror of gate[1] (advanced when a verdict is resolved)
        # identical seed on every replica => everything valid at t = 0 (compact: seeded on the pages held at the first quorum)
        self._holdings: List[Range] = [] if self.compact else [(0, numel)]
        self._lock = threading.Lock()
        self._reshard_stream = torch.cuda.Stream(device=self.device)
        self._reshard_event: Optional[torch.cuda.Event] = None
        self._refresh_pending = False
        self._commit_layout: Optional[Tuple[int, int]] = None
        self._commit_stream: torch.cuda.Stream = torch.cuda.current_stream(self.device)
        self._commit_event: Optional[torch.cuda.Event] = None
        self.lost_elements = 0           # state elements that had to be re-seeded because no holder survived
        self.pulled_bytes = 0
        self._micro_seen: List[int] = [0] * len(self.layout.units)  # accumulation: micro-batches reduced per unit
        self._configured = False         # a quorum has been configured (restore must come before)
        self._ckpt: Any = None           # durable checkpoints: ShardedWriter (staging buffer, writer thread)
        self._snap_stream: Optional[torch.cuda.Stream] = None
        self._snap_events: Optional[List[torch.cuda.Event]] = None  # per unit: its snapshot copy has been enqueued
        self._snap_done: Optional[torch.cuda.Event] = None          # ... and the whole snapshot
        self._disk: Optional[Tuple[int, str, List[Any]]] = None  # restore: (T, directory, files) for the next re-shard
        self.disk_read_elements = 0      # state elements re-shards read from a restored checkpoint's files
        if units is not None:
            self.set_units(units)
        elif self.no_decay:
            self._nd_units = split_no_decay(self.layout.units, self.no_decay)
        pg.add_configure_hook(self._on_configured)

    def set_units(self, units: Sequence[Range], no_decay: Optional[Sequence[Range]] = None) -> None:
        """Fix the unit ranges (forward order, tiling ``[0, numel)``); call before the first quorum. ``no_decay``
        replaces the constructor's weight-decay exemptions (flat element ranges); each must lie inside one unit."""
        assert all(lo % 8 == 0 and hi % 8 == 0 for lo, hi in units)
        assert merge_ranges(units) == [(0, self.numel)] and total(units) == self.numel, "units must tile the flat buffer exactly"
        if self.max_grad_norm is not None and len(units) > GNORM_UNITS:
            raise ValueError(f"gradient clipping supports at most {GNORM_UNITS} units, got {len(units)}")
        if self.audit_every and len(units) > GNORM_UNITS:
            raise ValueError(f"the replica audit supports at most {GNORM_UNITS} units, got {len(units)}")
        if self.compact and self.capacity:
            raise RuntimeError("compact state: the units are fixed once the page pools are allocated")
        units = tuple((int(a), int(b)) for a, b in units)
        nd = self.no_decay if no_decay is None else [(int(a), int(b)) for a, b in no_decay]
        self._nd_units = split_no_decay(units, nd)  # raises before anything changes
        self.no_decay = nd
        self.layout = ShardLayout(units, self._replication)
        self._micro_seen = [0] * len(self.layout.units)
        if self.compact:
            self._alloc_pools()
        if self.grad_accum_steps > 1:
            self._alloc_accum()

    def _alloc_accum(self) -> None:
        """One fp32 accumulator for this rank's primary slices, large enough for every world in ``[min_world, 8]``.
        Only this rank reads it, so it is an ordinary device tensor, not a symmetric segment."""
        self._acc = None  # a re-allocation for new units frees the old one first
        self._acc = torch.empty(accum_elements(self.layout, self.min_world), dtype=torch.float32, device=self.device)
        self._acc_for = None

    def _accum_for(self, rank: int, world: int) -> None:
        """Point the accumulator offsets at this quorum's slice geometry; raises when the slices do not fit."""
        if self._acc is None:
            self._alloc_accum()
        need = max(accum_offsets(self.layout, r, world)[1] for r in range(world))
        if need > self._acc.numel():
            # the same numbers on every rank: all of them raise alike
            raise RuntimeError(f"zero1: gradient accumulation at a quorum of {world} needs {4 * need} accumulator bytes "
                               f"per rank, {self.accum_bytes()} are allocated (sized for min_world={self.min_world})")
        self._acc_offsets = accum_offsets(self.layout, rank, world)[0]
        self._acc_for = (rank, world)

    def accum_bytes(self) -> int:
        """Device bytes of the gradient-accumulation buffer (0 without accumulation)."""
        return 0 if self._acc is None else 4 * self._acc.numel()

    def _alloc_pools(self) -> None:
        import numpy as np

        cap = self._state_pages
        if cap is None:
            cap = pool_pages(self.layout, self.min_world, self._page)
        self.capacity = int(cap)
        n = self.capacity * self._page
        if n >= self.numel:
            logger.warning("zero1: compact state pools of %d pages are not smaller than full-size state (min_world=%d "
                           "means a rank may have to hold everything): no memory is saved", self.capacity, self.min_world)
        self.master = self.pg.alloc_symmetric("z1_master", n * 4).view(torch.float32)[:n]
        self.m = self.pg.alloc_symmetric("z1_m", n * self._msize).view(self.moment_dtype)[:n]
        self.v = self.pg.alloc_symmetric("z1_v", n * self._msize).view(self.moment_dtype)[:n]
        if self.ema_decay is not None:
            self.ema = self.pg.alloc_symmetric("z1_ema", n * self._msize).view(self.moment_dtype)[:n]
        npages = (self.numel + self._page - 1) >> self._page_shift
        self._table_host = np.full(npages, -1, dtype=np.int32)  # page of the flat vector -> pool slot (-1: not held)
        self._table = torch.full((npages,), -1, dtype=torch.int32, device=self.device)
        self._free: List[int] = list(range(self.capacity - 1, -1, -1))  # pop() hands out the lowest slot

    # ------------------------------------------------------------------ init / heal
    @torch.no_grad()
    def seed_master(self) -> None:
        """Call once after the bf16 weights were initialised (same seed on every replica): seeds what this rank holds,
        i.e. all of full-size state. Compact state holds nothing yet and is seeded from the weights at the first
        quorum, when the rank's slices are known."""
        self._seed(self._holdings)

    def state_dict(self) -> Dict[str, Any]:
        """What a healing replica needs from ANY peer: the replicated bf16 weights and the update count.
        Its slices of (master, m, v) arrive through the re-shard pull from their holders."""
        return {"param": self.param, "t": self.t}

    def load_state_dict(self, sd: Dict[str, Any]) -> None:
        with torch.no_grad():
            if sd["param"].data_ptr() != self.param.data_ptr():
                self.param.copy_(sd["param"])
        self._set_t(int(sd["t"]))

    def _set_t(self, t: int) -> None:
        self.t = t
        with torch.cuda.stream(self._reshard_stream):
            self.gate[1:2].fill_(t)

    # ------------------------------------------------------------------ re-shard on quorum change
    def _on_configured(self, store: Any, rank: int, world: int, epoch: int) -> None:
        """Runs inside ``ProcessGroupB200.configure`` (quorum thread) with the quorum-scoped store. Every rank publishes
        ``{t, hold, pages?, disk?}``, plans every rank's re-shard (:func:`plan_quorum`) and applies its own: pulls
        (one copy launch), checkpoint reads and re-seeds on the re-shard stream, which the next commit waits for.
        Full-size state returns without waiting for them. Paged state frees the pages that are neither kept nor a
        source first and allocates its new ones, and after its pulls it meets its peers at a store barrier before it
        frees the pages it kept for them, so its re-shard completes here."""
        from torchft_b200.checkpointing.p2p_transport import device_copy

        with self._lock:
            if self._snap_done is not None:
                # a snapshot copy may still read the state that pulls, seeds, page reuse and heal are about to rewrite
                self._snap_done.synchronize()
            names = ("z1_param", "z1_grad", "z1_master", "z1_m", "z1_v") + (("z1_gnorm",) if self.max_grad_norm is not None else ()) \
                + (("z1_ema",) if self.ema is not None else ()) + (("z1_audit",) if self.audit_every else ()) \
                + (("z1_tokmean",) if self.global_token_mean else ())
            missing = [n for n in names if not self.comm.is_symmetric(n)]
            if missing:
                # the kernels dereference peer pointers: every replica must construct its Zero1Optimizer before its first
                # quorum (segments allocated later only become symmetric at the NEXT quorum change)
                raise RuntimeError(f"FT-ZeRO-1 segments {missing} are not mapped on every replica of this quorum")
            self._tok_commits = 0  # every rank of the new quorum starts its slot parity here
            if self.grad_accum_steps > 1:
                self._accum_for(rank, world)
            self._apply_audit()  # before publishing: the ranges a diverged audit condemned are not claimed
            me = {"t": self.t, "hold": self._holdings}
            if self.audit_every:
                me["audit"] = self.audit_every  # no audit publishes no key
            sched = self._schedule_digest()
            if sched is not None:
                me["sched"] = sched
            if self._msize == 2:
                me["moments"] = "bf16"  # fp32 moments publish no key: their record stays as it was
            if self._ema_c is not None:
                me["ema"] = ema_record(self._ema_c)  # likewise without an EMA
            if self._disk is not None:
                me["disk"] = [self._disk[0], self._disk[1]]  # every rank may read what no live holder has from it
            if self.compact:
                if world < self.min_world:
                    raise RuntimeError(f"zero1: a quorum of {world} is below min_world={self.min_world}; the compact "
                                       f"state pools ({self.capacity} pages) are not sized for it")
                me["pages"] = self._page_runs()
            store.set(f"z1/{rank}", json.dumps(me))
            peers: Dict[int, Dict[str, Any]] = {rank: me}
            for r in range(world):
                if r != rank:
                    peers[r] = json.loads(bytes(store.get(f"z1/{r}")).decode())
            digests = {r: p.get("sched") for r, p in peers.items()}
            if len(set(digests.values())) > 1:
                # holders of one slice would apply different rates or decays to the same bits and drift apart without a
                # sign; every rank reads the same records and raises alike, before anything is freed or pulled
                raise RuntimeError(f"zero1: the replicas of this quorum disagree on the learning-rate schedule or the "
                                   f"weight-decay exemptions (digest per rank: {digests})")
            check_moment_agreement(peers)
            check_ema_agreement(peers)
            periods = {r: p.get("audit", 0) for r, p in peers.items()}
            if len(set(periods.values())) > 1:
                # the audit's handshake would pair with another kernel of a peer that does not audit at the same step
                raise RuntimeError(f"zero1: the replicas of this quorum disagree on audit_every (per rank: {periods})")
            ckpt = self._ckpt_files(rank, peers)
            plans = plan_quorum(self.layout, world, peers, self._page_shift if self.compact else None, ckpt)
            plan = plans[rank]
            if plan.lost and ckpt:
                logger.warning("zero1: no checkpoint of update %d covers this rank's lost ranges %s", plan.tmax, plan.lost)
            s = self._reshard_stream
            s.wait_stream(self._commit_stream)  # no update of the old quorum may still touch state that is about to move
            if self.compact:
                peak = max(p.peak for p in plans.values())
                if peak > self.capacity:
                    # every rank sees the same plans and raises alike, before anything is freed
                    raise RuntimeError(f"zero1: re-sharding to a quorum of {world} needs {peak} state pages on one rank, "
                                       f"the pools hold {self.capacity} (raise min_world's range or state_pages)")
                self._free_pages(plan.free_first)
                # from here on a failure (a peer dying before the barrier) leaves this rank at its old t: it must not
                # claim ranges whose pages it gave back, or a later quorum would pull (or keep) state that is gone
                self._holdings = plan.hold_mid
                self._alloc_pages(plan.allocate)
                with torch.cuda.stream(s):
                    self._table.copy_(torch.from_numpy(self._table_host))
            with torch.cuda.stream(s):
                if plan.pulls:
                    tables = {src: self._peer_table(peers[src].get("pages")) for src, _, _ in plan.pulls}
                    entries: List[Tuple[int, int, int]] = []
                    for name, local in self._state_arrays(prefix="z1_"):
                        ptrs = self.comm.peer_pointers(name)
                        for src, lo, hi in plan.pulls:
                            for a, b, at in self._pieces(tables[src], lo, hi):
                                for c, d, mine in self._pieces(self._table_host, a, b):
                                    sz = local.element_size()
                                    entries.append((ptrs[src] + (at + c - a) * sz, local.data_ptr() + mine * sz, (d - c) * sz))
                    device_copy(entries, s, chunk_bytes=1 << 20)
                if plan.reads:
                    self._read_state(plan.reads)  # nobody live holds these at T: the restored checkpoint does
                seed_src = audit_seed_source(peers)
                same_w = intersect_ranges(plan.lost, self._audit_dropped) if rank != seed_src else []
                if same_w:
                    # the holders of a diverged slice may hold different weights: every holder seeds it from the same
                    # rank's copy, so their masters agree. That rank is at tmax, so no heal writes its param, and its
                    # own updates wait for this quorum's first commit, which waits for this re-shard.
                    src = self.comm.peer_pointers("z1_param")[seed_src]
                    device_copy([(src + 2 * lo, self.param.data_ptr() + 2 * lo, 2 * (hi - lo)) for lo, hi in same_w], s)
                self._seed(plan.lost)  # nobody holds these: re-seed from the replicated bf16 weights
            if self.compact:
                s.synchronize()
                self.comm._store_barrier(store, "z1/pulled", world)  # every peer has finished reading our source pages
                self._free_pages(plan.free_last)
                with torch.cuda.stream(s):
                    self._table.copy_(torch.from_numpy(self._table_host))
            with torch.cuda.stream(s):
                if self.t != plan.tmax:
                    self.gate[1:2].fill_(plan.tmax)
                self._reshard_event = s.record_event()
            if plan.lost and plan.counted:
                self.lost_elements += total(plan.lost)
                logger.warning("zero1: %d state elements had no surviving holder and were re-seeded from the weights "
                               "(moments reset)", total(plan.lost))
            self.pulled_bytes += self._state_item() * total([(lo, hi) for _, lo, hi in plan.pulls])
            self.t = plan.tmax
            self._holdings = plan.hold
            self._refresh_pending = world > 1
            self._updates_since_config = 0
            self._audit_dropped = []
            if self.audit_every and world > 1:
                self._audit_setup(rank, world)
            self._configured, self._disk = True, None

    def _state_arrays(self, prefix: str = "") -> List[Tuple[str, torch.Tensor]]:
        """``(name, array)`` of the partitioned state: master, m, v and, when kept, the EMA."""
        arrays = [("master", self.master), ("m", self.m), ("v", self.v)] + ([("ema", self.ema)] if self.ema is not None else [])
        return [(prefix + n, a) for n, a in arrays]

    def _state_item(self) -> int:
        """Bytes of the partitioned state per element: 12 with fp32 moments, 8 with bf16, plus 4 or 2 with an EMA."""
        return sum(a.element_size() for _, a in self._state_arrays())

    def _schedule_digest(self) -> Optional[str]:
        """What this rank publishes of its schedule and exemptions (``None`` without either: the record stays as it was)."""
        if self._lr_host is None and not self.no_decay:
            return None
        return schedule_digest(self._lr_host, self.no_decay)

    def _ckpt_files(self, rank: int, peers: Dict[int, Dict[str, Any]]) -> Dict[int, Any]:
        """The checkpoint files at the quorum's update count that ranks restored from, for :func:`plan_quorum`: this
        rank's own restore, or else the directory every restored peer published (a live rank may now hold slices that
        only restored ranks held)."""
        from torchft_b200.checkpointing.sharded import scan

        tmax = max(int(p["t"]) for p in peers.values())
        if self._disk is not None and self._disk[0] == tmax:
            return {rank: self._disk[2]}
        scanned: Dict[str, Any] = {}
        out = {}
        for r, p in peers.items():
            d = p.get("disk")
            if d and int(d[0]) == tmax:
                if d[1] not in scanned:
                    scanned[d[1]] = [(h, [tuple(int(x) for x in rg) for rg in h["ranges"]]) for h in scan(d[1])
                                     if int(h["T"]) == tmax]
                out[r] = scanned[d[1]]
        return out

    # ------------------------------------------------------------------ compact (paged) state
    def _page_runs(self) -> List[Tuple[int, int, int]]:
        """The page table as ``(page, slot, count)`` runs of consecutive pages in consecutive slots."""
        runs: List[List[int]] = []
        for pg in map(int, (self._table_host >= 0).nonzero()[0]):
            slot = int(self._table_host[pg])
            if runs and runs[-1][0] + runs[-1][2] == pg and runs[-1][1] + runs[-1][2] == slot:
                runs[-1][2] += 1
            else:
                runs.append([pg, slot, 1])
        return [tuple(r) for r in runs]

    def _peer_table(self, runs: Optional[Sequence[Sequence[int]]]) -> Any:
        """A page table from published ``(page, slot, count)`` runs (``None``: full-size state, no table)."""
        import numpy as np

        if runs is None:
            return None
        t = np.full(len(self._table_host), -1, dtype=np.int64)
        for pg, slot, n in runs:
            t[pg:pg + n] = np.arange(slot, slot + n)
        return t

    def _pieces(self, table: Any, lo: int, hi: int) -> List[Tuple[int, int, int]]:
        """``[lo, hi)`` cut at page boundaries as ``(elem_lo, elem_hi, pool_index)``, pieces in consecutive slots merged.
        Without a ``table`` (full-size state) element ``e`` is at index ``e``: one piece."""
        if table is None:
            return [(lo, hi, lo)] if hi > lo else []
        out: List[Tuple[int, int, int]] = []
        sh, mask = self._page_shift, self._page - 1
        e = lo
        while e < hi:
            end = min(hi, ((e >> sh) + 1) << sh)
            slot = int(table[e >> sh])
            assert slot >= 0, f"zero1: element {e} is not mapped to a pool page"
            at = (slot << sh) | (e & mask)
            if out and out[-1][1] == e and out[-1][2] + (e - out[-1][0]) == at:
                out[-1] = (out[-1][0], end, out[-1][2])
            else:
                out.append((e, end, at))
            e = end
        return out

    def _free_pages(self, pages: Sequence[Range]) -> None:
        for plo, phi in pages:
            for pg in range(plo, phi):
                slot = int(self._table_host[pg])
                if slot >= 0:
                    self._free.append(slot)
                    self._table_host[pg] = -1
        self._free.sort(reverse=True)

    def _alloc_pages(self, pages: Sequence[Range]) -> None:
        for plo, phi in pages:
            for pg in range(plo, phi):
                if self._table_host[pg] < 0:
                    self._table_host[pg] = self._free.pop()

    @torch.no_grad()
    def _seed(self, ranges: Sequence[Range]) -> None:
        """``master = float(param)``, ``m = v = 0`` and ``ema = master`` on ``ranges`` (current stream). bf16(master) is
        ``param`` exactly, so a bf16 EMA starts equal to the master weights too."""
        for lo, hi in ranges:
            for a, b, at in self._pieces(self._table_host, lo, hi):
                self.master[at:at + b - a].copy_(self.param[a:b])
                self.m[at:at + b - a].zero_()
                self.v[at:at + b - a].zero_()
                if self.ema is not None:
                    self.ema[at:at + b - a].copy_(self.param[a:b])

    # ------------------------------------------------------------------ per-step pipeline
    def unit_of(self, lo: int, hi: int) -> int:
        return self.layout.units.index((lo, hi))

    def reduce_scatter(self, unit: int, scale: float, contribute: bool, micro: int = 0) -> Any:
        """Reduce unit ``unit`` of the gradient buffer across the quorum (comm stream, overlaps backward). With
        gradient accumulation, ``micro`` is the micro-batch index; ``scale`` applies on the last micro-batch only."""
        lo, hi = self.layout.units[unit]
        mode = accum_mode(micro, self.grad_accum_steps)
        clip = self.max_grad_norm is not None
        if self.comm.world == 1 and not clip and not mode:
            if scale != 1.0 or not contribute:
                self.grad[lo:hi].mul_(scale if contribute else 0.0)
            return None
        # with accumulation the kernel runs at world 1 too (in place, no handshake): the scale belongs after the sum
        # over micro-batches, which it adds into (modes 1, 2) or out of (mode 3) this rank's accumulator
        acc = 0
        if mode:
            rank, world = self.comm.rank, self.comm.world
            if self._acc_for != (rank, world):
                self._accum_for(rank, world)
            acc = self._acc.data_ptr() + 4 * self._acc_offsets[unit]
        gn = self._gnorm.data_ptr() + 8 * unit if clip and mode in (0, 3) else 0
        after = self._commit_event if clip else None
        k = self.layout.replication

        def launch(s: torch.cuda.Stream) -> None:
            if after is not None:
                # the last commit kernel read the partials this step overwrites (see zero1_commit_kernel)
                s.wait_event(after)
            self.comm.zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, scale, contribute, k, self._rs_blocks, s,
                                            gnorm=gn, acc=acc, acc_mode=mode)

        work = self.pg._launch(launch, None)
        if mode:
            # micro-batches must arrive in order from 0; anything else poisons the unit until the next micro-batch 0
            in_order = micro == 0 or self._micro_seen[unit] == micro
            self._micro_seen[unit] = micro + 1 if in_order else -1
        return work

    # -- committer protocol of Manager.commit_on_device ---------------------------------------------------------
    def bind_stream(self, stream: torch.cuda.Stream) -> None:
        """The stream the verdict and update kernels run on (the trainer's optimizer stream)."""
        self._commit_stream = stream

    def publish_tokens(self, n_valid: torch.Tensor, loss_sum: torch.Tensor, rows: int, participants: int,
                       contribute: bool) -> None:
        """Global token mean: what the next :meth:`enqueue` publishes for this rank. ``n_valid`` (device int64 scalar)
        counts the step's targets that are not ignored, ``loss_sum`` (device fp64 scalar) is the sum of their losses,
        ``rows`` is the step's ``M * B * S`` and ``participants`` the ``P`` the reduce-scatters divided by. Both tensors
        are written on the current stream, which the commit stream waits for. A rank that does not ``contribute``
        publishes 0 targets and a loss of 0 (a vetoed step still reports its own mean from the real pair)."""
        if not self.global_token_mean:
            raise RuntimeError("publish_tokens needs Zero1Optimizer(global_token_mean=True)")
        self._tok_pending = (n_valid.reshape(1), loss_sum.reshape(1), int(rows), max(int(participants), 1), bool(contribute))

    def token_mean_loss(self) -> torch.Tensor:
        """Global token mean: ``L / N`` of the last commit as a new device scalar, copied on the current stream behind
        that commit. The same bits on every rank of a committed step; a vetoed step gives this rank's own ``L / n``."""
        if not self.global_token_mean or self._commit_event is None:
            raise RuntimeError("token_mean_loss needs a commit of Zero1Optimizer(global_token_mean=True)")
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(self._commit_event)
        return self._tok_out[0].clone()

    def enqueue(self, host_ok: bool) -> int:
        """Enqueue the verdict kernel behind this step's reduce-scatters (comm stream) and backward (current stream).

        With gradient accumulation a unit that was not reduced for all ``M`` micro-batches (e.g. the Manager stopped
        launching after an error) makes the local verdict negative; the kernel still runs, so the peers learn of it."""
        if self.grad_accum_steps > 1:
            seen, self._micro_seen = self._micro_seen, [0] * len(self.layout.units)
            short = [u for u, n in enumerate(seen) if n != self.grad_accum_steps]
            if short:
                if host_ok:
                    logger.warning("zero1: units %s were not reduced for all %d micro-batches: the step is vetoed",
                                   short, self.grad_accum_steps)
                host_ok = False
        stream = self._commit_stream
        stream.wait_stream(self.pg.comm_stream)
        stream.wait_stream(torch.cuda.current_stream(self.device))
        if self._reshard_event is not None:
            stream.wait_event(self._reshard_event)  # a verdict also tells peers "my pulls are done"
            self._reshard_event = None
        self._commit_layout = (self.comm.rank, self.comm.world)
        clip = {} if self.max_grad_norm is None else dict(gnorm="z1_gnorm", nunits=len(self.layout.units),
                                                           max_norm=self.max_grad_norm, norm=self._clip)
        tok: Dict[str, Any] = {}
        if self.global_token_mean:
            if self._tok_pending is None:
                raise RuntimeError("global_token_mean: publish_tokens must come before every commit")
            (n, loss, rows, participants, contribute), self._tok_pending = self._tok_pending, None
            for x in (n, loss):
                x.record_stream(stream)  # read by the commit kernel on the commit stream
            tok = dict(tokens="z1_tokmean", slot=self._tok_commits % TOKEN_SLOTS, n_valid=n, loss_sum=loss, rows=rows,
                       divisor=participants * rows, contribute=contribute, token_out=self._tok_out,
                       token_count=self._tok_count)
            if not clip:
                tok["norm"] = self._clip  # its second word is the coefficient the update reads
            self._tok_commits += 1
        seq = self.comm.zero1_commit_(self.gate, host_ok, True, stream, **clip, **tok)
        self._commit_event = stream.record_event()
        return seq

    def wait(self, seq: int, timeout: Any = None) -> bool:
        """Block the calling thread until the verdict of ``seq`` is on the host."""
        self._commit_event.synchronize()
        v = self.comm.verdict(seq)
        if v is None:
            raise RuntimeError(f"commit {seq}: the verdict kernel finished without posting a verdict")
        if self.max_grad_norm is not None:
            self._resolved_norm = self.comm.grad_norm(seq)
        if self.global_token_mean:
            self._resolved_reason = self.comm.commit_reason(seq)
        return v

    def update(self, events: Optional[Sequence[torch.cuda.Event]] = None) -> None:
        """Gated AdamW + weight all-gather for every unit, in forward order, on the commit stream; ``events[i]``
        fires when unit ``i``'s weights are current on THIS replica (all peers' pushes have landed)."""
        self._not_in_ema("update")
        stream = self._commit_stream
        k = self.layout.replication
        lr = self.param_groups[0]["lr"]
        hp = (lr, self.betas[0], self.betas[1], self.eps, self.weight_decay)
        # clipping and the token mean: the coefficient the commit kernel wrote
        coef = self._clip.data_ptr() + 4 if self.max_grad_norm is not None or self.global_token_mean else 0
        # with a schedule the kernel reads the rate of the device's update count from the table; lr is unused
        sched = {} if self._lr_tab is None else {"lr_table": self._lr_tab.data_ptr(), "lr_steps": self._lr_tab.numel()}
        nd = self._nd_units if self.no_decay else None
        modes = (1, 0) if self._refresh_pending else (0,)
        self._refresh_pending = False
        snap, self._snap_events = self._snap_events, None
        for i, (lo, hi) in enumerate(self.layout.units):
            if snap is not None:
                stream.wait_event(snap[i])  # the last save's copy of this unit has read it
            state = self._update_state(lo)
            for mode in modes:
                self.comm.zero1_update_("z1_param", lo * 2, self.grad.data_ptr() + lo * 2, nelem=hi - lo, hyper=hp,
                                        gate=self.gate, replication=k, mode=mode, blocks=self._upd_blocks, stream=stream,
                                        coef=coef, no_decay=nd[i] if nd else (), moment_dtype=self.moment_dtype,
                                        **sched, **state)
            if events is not None:
                events[i].record(stream)
        if self.audit_every:
            self._updates_since_config += 1
            if self.comm.world > 1 and self._updates_since_config % self.audit_every == 0:
                self._audit(stream)

    # ------------------------------------------------------------------ replica audit
    def _audit(self, stream: torch.cuda.Stream) -> None:
        """Enqueue one audit on ``stream`` behind the last unit's update and weight handshake: zero the slots, copy the
        update count, digest (one launch), handshake and compare (see DESIGN.md for why this is race-free)."""
        rank, world = self.comm.rank, self.comm.world
        nunits, stride, narrays = len(self.layout.units), self._audit_stride, len(self._state_arrays())
        n = nunits * stride + 1
        assert self._audit_table is not None and self._audit_table[0] == (rank, world), "set up at the quorum change"
        _, table, nentries, chunks = self._audit_table
        sp = int(stream.cuda_stream)
        slots = self._audit_slots.data_ptr()
        self._K.memset_async(slots, 0, 8 * n, sp)
        self._K.memcpy_async(slots + 8 * (n - 1), self.gate.data_ptr() + 4, 4, sp)  # t = gate[1], little-endian
        self._K.z1_digest(table.data_ptr(), nentries, chunks, slots, max(1, min(chunks, self._K.NUM_SMS * 3)), sp)
        self._audit_seq += 1
        self.comm.z1_audit_compare_("z1_audit", self._audit_report, self._audit_seq, nunits, stride,
                                    self.layout.k(world), narrays, stream)
        self._audit_event = stream.record_event()
        self._audit_quorums = {s: q for s, q in self._audit_quorums.items() if s > self._audit_seen}
        self._audit_quorums[self._audit_seq] = (rank, world)
        self.audits += 1

    def _audit_setup(self, rank: int, world: int) -> None:
        """At a quorum change: the host-mapped report (once, for up to 8 ranks) and the digest kernel's rows
        (``audit::DigestEntry``) for this rank at ``(rank, world)``: the weights of every unit, and with ``k > 1`` each
        state array over each held slice. The copy is synchronous, so it is made here and never inside :meth:`update`,
        whose launches must not wait for the device; the arrays and the page table stay where they are."""
        if self._audit_report is None:
            n = len(self.layout.units) * self._audit_stride + 1
            self._audit_report = self._K.MappedWords(self._K.Z1_AUDIT_REPORT_HEADER + 8 * n)
        if self._audit_table is not None and self._audit_table[0] == (rank, world):
            return
        cw = int(self._K.Z1_DIGEST_CHUNK_WORDS)
        rows: List[Tuple[int, ...]] = []
        chunk0 = 0
        k, stride = self.layout.k(world), self._audit_stride
        table = self._table.data_ptr() if self._table is not None else 0

        def add(base: int, es: int, paged: bool, lo: int, hi: int, seed: int, slot: int) -> None:
            nonlocal chunk0
            if hi <= lo:
                return  # an empty slice: its slot stays 0 on every holder
            nwords = (hi - lo) * es // 8
            pbs = self._page_shift + es.bit_length() - 1 if paged else 0
            rows.append((base, table if paged else 0, pbs, lo * es // 8, nwords, seed, slot, chunk0))
            chunk0 += (nwords + cw - 1) // cw

        for u, (lo, hi) in enumerate(self.layout.units):
            add(self.param.data_ptr(), 2, False, lo, hi, AUDIT_SEEDS["weights"], u * stride)
            if k < 2:
                continue
            for j in range(k):
                a, b = self.layout.slice_bounds(u, world, (rank - j) % world)
                for x, (name, arr) in enumerate(self._state_arrays()):
                    add(arr.data_ptr(), arr.element_size(), bool(table), a, b, AUDIT_SEEDS[name],
                        u * stride + 1 + j * len(self._state_arrays()) + x)
        self._audit_table = ((rank, world), torch.tensor(rows, dtype=torch.int64).to(self.device), len(rows), chunk0)

    def audit_report(self) -> Optional[Dict[str, Any]]:
        """The report of the last audit whose compare ran (:func:`decode_audit_report`), after waiting for the last
        audit on the host; ``None`` before the first audit. Also kept as ``last_audit``."""
        if self._audit_event is None:
            return None
        self._audit_event.synchronize()
        seq = int.from_bytes(self._audit_report.read()[:8], "little")
        rank_world = self._audit_quorums.get(seq)
        if rank_world is None:
            return self.last_audit  # no compare of a recorded audit has run
        k = self.layout.k(rank_world[1])
        self.last_audit = decode_audit_report(self._audit_report.read(), len(self.layout.units), self._audit_stride,
                                              len(self._state_arrays()), k)
        self.last_audit["rank"] = rank_world[0]
        return self.last_audit

    def _apply_audit(self) -> None:
        """At a quorum change: act once on a report that shows a divergence. Log each finding and stop claiming the
        ranges :func:`audit_findings` gives this rank, if this rank was at the audited quorum's update count and is
        still there."""
        rep = self.audit_report()
        if rep is None or rep["seq"] <= self._audit_seen:
            return
        self._audit_seen = rep["seq"]
        if not rep["mismatches"]:
            return
        self.divergences += 1
        findings, drops = audit_findings(rep, self.layout, rep["world"])
        for f in findings:
            logger.warning("zero1: audit %d: %s of unit %d%s differs on quorum ranks %s at update %d", rep["seq"],
                           f["array"], f["unit"], "" if f["slice"] is None else f" slice {f['slice']}", f["ranks"], f["t"])
        me = rep["rank"]
        if self.t == max(rep["t"]) == rep["t"][me] and drops[me]:
            logger.warning("zero1: this rank stops claiming %s after the audit", drops[me])
            self._holdings = subtract_ranges(self._holdings, drops[me])
            self._audit_dropped = drops[me]

    def _update_state(self, lo: int) -> Dict[str, int]:
        """The state arguments of ``zero1_update_`` for the unit that starts at element ``lo``. Full-size state passes
        the arrays at ``lo`` and no table, which selects the kernel without page lookups; paged state passes the pools
        and the page table, through which the kernel finds each element."""
        ema = {} if self.ema is None else {"ema_c": self._ema_c}
        if self._table is None:
            # the global element index of the unit's start is what bf16 moments hash for their rounding bits
            if self.ema is not None:
                ema["ema"] = self.ema.data_ptr() + self._msize * lo
            return {"master": self.master.data_ptr() + 4 * lo, "m": self.m.data_ptr() + self._msize * lo,
                    "v": self.v.data_ptr() + self._msize * lo, "state_off": lo, **ema}
        if self.ema is not None:
            ema["ema"] = self.ema.data_ptr()
        ptrs = {"master": self.master.data_ptr(), "m": self.m.data_ptr(), "v": self.v.data_ptr()}
        return {**ptrs, "table": self._table.data_ptr(), "state_off": lo, "page_shift": self._page_shift, **ema}

    def resolved(self, verdict: bool) -> None:
        """The Manager learned the verdict of the last :meth:`commit` (lazily, on the quorum thread)."""
        with self._lock:
            if verdict and self._commit_layout is not None:
                rank, world = self._commit_layout
                self.t += 1
                self._holdings = self.layout.held(rank, world)
            self._commit_layout = None
            if self.max_grad_norm is not None and self._resolved_norm is not None:
                norm, self._resolved_norm = self._resolved_norm, None
                self.last_grad_norm = norm
                if not math.isfinite(norm):
                    self.nonfinite_steps += 1
                    logger.warning("zero1: gradient norm is %s: the step was skipped on every replica (%d so far)",
                                   norm, self.nonfinite_steps)
            reason, self._resolved_reason = self._resolved_reason, None
            if reason and reason & self._K.ZERO1_VETO_ROWS:
                self.row_mismatch_steps += 1
                logger.warning("zero1: the replicas published different row counts M * B * S, so no one token-mean "
                               "factor fits: the step was skipped on every replica (%d so far)", self.row_mismatch_steps)

    # ------------------------------------------------------------------ durable checkpoints
    @torch.no_grad()
    def save(self, directory: str, manager_state: Optional[Dict[str, int]] = None,
             events: Optional[Sequence[torch.cuda.Event]] = None, keep: int = 2) -> int:
        """Snapshot this rank's primary slices (bf16 weights, master, m, v) at the update count ``t`` and write them to
        ``directory`` in the background; returns ``t``. Every replica of the quorum calls it after the same step.

        The last step's verdict must be resolved (``Manager.state_dict()`` does it). ``events[i]`` are the events
        :meth:`update` recorded for unit ``i`` (default: everything enqueued on the commit stream so far);
        ``manager_state`` is ``{"step", "batches_committed"}`` for the header. A save first waits for the previous
        write and re-raises its error; :meth:`wait_checkpoint` waits for this one. ``keep`` newest steps of the files
        this optimizer wrote are kept."""
        self._not_in_ema("save")
        if not self._configured:
            raise RuntimeError("zero1: nothing to checkpoint before the first quorum")
        if self._commit_layout is not None:
            raise RuntimeError("zero1: the last step's verdict is not resolved; settle it first (Manager.state_dict())")
        rank, world = self.comm.rank, self.comm.world
        ranges = intersect_ranges(self.layout.primary(rank, world), self._holdings)
        return self._save(directory, ranges, rank, world, manager_state, events, keep)

    def _save(self, directory: str, ranges: Sequence[Range], rank: int, world: int,
              manager_state: Optional[Dict[str, int]], events: Optional[Sequence[torch.cuda.Event]], keep: int) -> int:
        from torchft_b200.checkpointing.sharded import ShardedWriter, sections

        if self._ckpt is None or self._ckpt.directory != directory or self._ckpt.keep != keep:
            if self._ckpt is not None:
                self._ckpt.wait()
            self._ckpt = ShardedWriter(directory, keep)
        w = self._ckpt
        w.wait()  # the previous write has left the staging buffer; surfaces its error
        written, e = [], 0
        for lo, hi in ranges:
            written.append((lo, hi, e))
            e += hi - lo
        sec = sections(e, self._msize, ema=self.ema is not None)
        stage = w.staging((2 + self._state_item()) * e)  # bf16 weights, fp32 master, m, v (and the EMA) per element
        if self._snap_stream is None:
            self._snap_stream = torch.cuda.Stream(device=self.device)
        s = self._snap_stream
        after = None if events is not None else self._commit_stream.record_event()
        u8 = torch.uint8
        done: List[torch.cuda.Event] = []
        with torch.cuda.stream(s):
            for i, unit in enumerate(self.layout.units):
                s.wait_event(events[i] if events is not None else after)  # unit i's update and weight pushes landed
                for lo, hi, off in written:
                    for a, b in intersect_ranges([(lo, hi)], [unit]):
                        x = off + a - lo
                        stage[2 * x:2 * (x + b - a)].copy_(self.param[a:b].view(u8), non_blocking=True)
                        for name, arr in self._state_arrays():
                            sz = arr.element_size()
                            base = sec[name] + sz * x
                            for c, d, at in self._pieces(self._table_host, a, b):  # maximal runs of consecutive slots
                                stage[base + sz * (c - a):base + sz * (d - a)].copy_(arr[at:at + d - c].view(u8),
                                                                                     non_blocking=True)
                done.append(s.record_event())
        self._snap_events, self._snap_done = done, done[-1]
        ms = manager_state or {"step": self.t, "batches_committed": 0}
        header = {"version": 1, "numel": self.numel, "units": [list(u) for u in self.layout.units], "T": self.t,
                  "step": int(ms["step"]), "batches": int(ms["batches_committed"]), "world": world, "rank": rank,
                  "k": self.layout.k(world), "compact": self.compact, "ranges": [list(r) for r in written],
                  "elements": e, "sections": sec,
                  "hparams": {"lr": self.param_groups[0]["lr"], "betas": list(self.betas), "eps": self.eps,
                              "weight_decay": self.weight_decay, "max_grad_norm": self.max_grad_norm}}
        if self._msize == 2:
            header["moments"] = "bf16"  # a header without the key describes fp32 moments
        if self.ema is not None:
            header["ema"] = {"decay": self.ema_decay}  # ... and one without this key has no EMA section
        w.submit(header, self._snap_done)
        return self.t

    def wait_checkpoint(self) -> None:
        """Block until the last :meth:`save` is on disk; re-raises a failed write."""
        if self._ckpt is not None:
            self._ckpt.wait()

    def snapshot_bytes(self) -> int:
        """Pinned host bytes of the checkpoint staging buffer (0 before the first save)."""
        stage = None if self._ckpt is None else self._ckpt.stage
        return 0 if stage is None else stage.numel()

    @torch.no_grad()
    def restore(self, directory: str) -> Optional[Dict[str, int]]:
        """Before the first quorum: load the newest complete checkpoint in ``directory``. Reads the full bf16 weights,
        sets ``t`` to its update count ``T``, claims no state, and arms the next re-shard to read the ranges no live
        holder at ``T`` has from the files. Returns the header's ``{"step", "batches_committed"}`` for the Manager, or
        ``None`` when no update count is complete. Unreadable files are skipped; files written for another ``numel``
        or other units raise ``ValueError`` before any state changes."""
        from torchft_b200.checkpointing.sharded import check_compatible, scan

        self._not_in_ema("restore")
        if self._configured:
            raise RuntimeError("zero1: restore must be called before the first quorum")
        headers = scan(directory)
        check_compatible(headers, self.numel, self.layout.units)
        T = newest_complete_step(headers, self.numel)
        if T is None:
            return None
        files = [(h, [tuple(int(x) for x in r) for r in h["ranges"]]) for h in headers if int(h["T"]) == T]
        self._read_ranges(ckpt_read_plan([(0, self.numel)], files), ("param",))
        self._set_t(T)
        self._holdings = []  # nothing held is current until the re-shard: the files or live peers at T provide it
        self._disk = (T, directory, files)
        self._reshard_stream.synchronize()  # the weights are in place before the first forward
        first = files[0][0]
        logger.info("zero1: restored the weights of update %d from %d checkpoint file(s) in %s", T, len(files), directory)
        return {"step": int(first["step"]), "batches_committed": int(first["batches"])}

    def _read_state(self, reads: Sequence[Tuple[Any, int, int, int]]) -> None:
        self._read_ranges(reads, ("master", "m", "v"))
        if self.ema is not None:
            have, seed = split_ema_reads(reads)
            self._read_ranges(have, ("ema",))
            if seed:
                logger.warning("zero1: the checkpoint files of %s have no EMA of the weights: it starts from the "
                               "master weights there", seed)
                with torch.cuda.stream(self._reshard_stream):
                    for lo, hi in seed:
                        for a, b, at in self._pieces(self._table_host, lo, hi):
                            self.ema[at:at + b - a].copy_(self.master[at:at + b - a])  # bf16: rounds to nearest
        self.disk_read_elements += total([(lo, hi) for _, _, lo, hi in reads])

    def _read_ranges(self, reads: Sequence[Tuple[Any, int, int, int]], arrays: Sequence[str]) -> None:
        """``arrays`` over the flat ranges of ``reads`` from the files, through pinned bounce buffers, on the re-shard
        stream (compact state: into the pool pages the table maps them to)."""
        from torchft_b200.checkpointing.sharded import RangedReader, file_dtype

        dst = {"param": self.param, **dict(self._state_arrays())}
        rd = RangedReader(self._reshard_stream)
        try:
            for h, off, lo, hi in reads:
                for name in arrays:
                    convert = file_dtype(h, name) != dst[name].dtype
                    for a, b, at in self._pieces(None if name == "param" else self._table_host, lo, hi):
                        if not convert:
                            rd.read(h, name, off + a - lo, dst[name][at:at + b - a])
                            continue
                        # moments (or EMA) saved in the other type: fp32 -> bf16 rounds to nearest, bf16 -> fp32 is exact
                        for c in range(a, b, CONVERT_CHUNK):
                            n = min(CONVERT_CHUNK, b - c)
                            with torch.cuda.stream(self._reshard_stream):
                                tmp = torch.empty(n, dtype=file_dtype(h, name), device=self.device)
                                rd.read(h, name, off + c - lo, tmp)
                                dst[name][at + c - a:at + c - a + n].copy_(tmp)
        finally:
            rd.close()

    # ------------------------------------------------------------------ introspection
    def lr_at(self, t: int) -> float:
        """The fp32 learning rate committed update ``t`` (1-based) applies: the table's entry ``min(max(t, 1),
        lr_steps) - 1`` with a schedule, else ``param_groups[0]["lr"]`` rounded to fp32."""
        import numpy as np

        if self._lr_host is None:
            return float(np.float32(self.param_groups[0]["lr"]))
        return float(self._lr_host[min(max(int(t), 1), len(self._lr_host)) - 1])

    def state_bytes_held(self) -> int:
        return self._state_item() * total(self.layout.held(self.comm.rank, max(self.comm.world, 1)))

    def state_bytes_allocated(self) -> int:
        """Device bytes of the master/m/v arrays and the EMA (compact: the page pools)."""
        return self._state_item() * self.master.numel()

    def held_state(self) -> Dict[Range, Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        """Copies of (master, m, v) over each range this rank holds, keyed by ``(lo, hi)`` (for inspection and tests)."""
        out = {}
        torch.cuda.synchronize(self.device)
        for lo, hi in self._holdings:
            pieces = self._pieces(self._table_host, lo, hi)
            out[(lo, hi)] = tuple(torch.cat([x[at:at + b - a] for a, b, at in pieces]) for x in (self.master, self.m, self.v))
        return out

    def held_ema(self) -> Dict[Range, torch.Tensor]:
        """Copies of the EMA of the weights over each range this rank holds, keyed like :meth:`held_state`."""
        if self.ema is None:
            raise RuntimeError("zero1: this optimizer keeps no EMA of the weights (ema_decay)")
        torch.cuda.synchronize(self.device)
        return {(lo, hi): torch.cat([self.ema[at:at + b - a] for a, b, at in self._pieces(self._table_host, lo, hi)])
                for lo, hi in self._holdings}

    # ------------------------------------------------------------------ evaluating the EMA
    @contextlib.contextmanager
    def ema_weights(self) -> Iterator[None]:
        """Inside the context ``param`` holds bf16(EMA) on every replica; on exit it holds bf16(master) again, bit for
        bit. Every replica of the quorum enters after the same step (the swap pushes each primary slice to everybody).

        Entry enqueues the EMA broadcast (update kernel mode 2) of every unit on the commit stream, behind the last
        update, and makes the current stream wait for it; exit enqueues the refresh (mode 1) behind whatever the current
        stream did inside, and makes the current stream wait for that. Both broadcasts start with a handshake, so no
        replica's push overwrites a peer's ``param`` while that peer is still updating or evaluating it. Inside, :meth:`update`, :meth:`save` and
        :meth:`restore` raise: training steps, checkpoints and the heal payload (:meth:`state_dict`, whose ``param``
        a healing peer copies) must never see the EMA in place of the weights. A heal is served only from the Manager's
        quorum task, which ``start_quorum`` starts at the beginning of a step and ``commit_on_device`` waits for (and
        closes the checkpoint window after) before the step's update is enqueued; no step can start inside the context,
        so no quorum task runs there either."""
        if self.ema is None:
            raise RuntimeError("zero1: this optimizer keeps no EMA of the weights (ema_decay)")
        if not self._configured:
            raise RuntimeError("zero1: there are no EMA weights to swap in before the first quorum")
        self._not_in_ema("ema_weights")
        self._broadcast(2)
        self._ema_active = True
        try:
            yield
        finally:
            self._broadcast(1)
            self._ema_active = False

    def _broadcast(self, mode: int) -> None:
        """Every unit's primary slice of bf16(EMA) (``mode`` 2) or bf16(master) (1) into every replica's ``param``, on
        the commit stream between the current stream's work before and after.

        The pushes land in the peers' ``param``, so they wait behind a handshake: no rank pushes before every peer's
        commit stream has reached the same point, i.e. before every peer has finished its last update (at W = k that
        update ends without a handshake of its own) and whatever its current stream read of ``param`` before it entered
        or left the context (an evaluation)."""
        stream, cur = self._commit_stream, torch.cuda.current_stream(self.device)
        stream.wait_stream(cur)  # what the current stream reads of param (an evaluation) comes first
        if self._snap_done is not None:
            stream.wait_event(self._snap_done)  # the last save has copied param
        self.comm.zero1_barrier_(stream)  # ... on every replica
        hp = (self.param_groups[0]["lr"], self.betas[0], self.betas[1], self.eps, self.weight_decay)  # unused here
        for lo, hi in self.layout.units:
            self.comm.zero1_update_("z1_param", lo * 2, self.grad.data_ptr() + lo * 2, nelem=hi - lo, hyper=hp,
                                    gate=self.gate, replication=self.layout.replication, mode=mode,
                                    blocks=self._upd_blocks, stream=stream, moment_dtype=self.moment_dtype,
                                    **self._update_state(lo))
        cur.wait_stream(stream)

    def _not_in_ema(self, what: str) -> None:
        if self._ema_active:
            raise RuntimeError(f"zero1: {what} inside ema_weights(): param holds the EMA weights, not the training "
                               f"weights")

    def zero_grad(self, set_to_none: bool = False) -> None:  # gradients are overwritten by the wgrad GEMMs
        pass
