"""The FT-ZeRO-1 kernels (``csrc/kernels/zero1.cu``) element by element, at every world size 1..8 and at Llama-3 unit
sizes: a llama3_1b block (60 821 504 elements) for the full matrix, a llama3_8b block (218 112 000) at W = 7 and 8, and
edge units of 8, 56, 8W - 8 and 8(3W + 1) elements, where some slices are empty and the last one is short.

- reduce: every holder's slice equals the rank-order fp32 sum, scaled and rounded once to bf16, bit for bit; every other
  byte of the gradient segment (the rest of the unit, sentinel-filled neighbour units) is unchanged; the clipping partial
  is exact on data whose per-thread fp32 sums are exact and within the per-thread chain bound on random data.
- commit: the global norm within half an fp32 ulp of the fp64 norm of the partials, the coefficient bit for bit.
- update: one fp64 AdamW step from the kernel's own prior state (``_fp64._adamw_ref``), so errors never compound; weights
  on every rank are bf16(master of the primary holder) bit for bit; state outside the held ranges is untouched.

Ranks are pre-signalled ``SymmetricComm.virtual_world`` ranks run one after the other (one concurrent run checks that
real signalling gives the same bits). The step count the update reads is the device word ``gate[1]`` that
``Zero1Optimizer._set_t`` writes. References are computed per slice, in chunks of 2^24 elements. Peak device
memory, counted from the allocations: about 16 GB, for the llama3_8b block at W = 8 with fp32 moments (7.0 GB of gradient
and parameter segments, 5.2 GB of compact state, about 3.5 GB of gradient, masks and chunked references).
"""

from __future__ import annotations

import itertools
import math
from datetime import timedelta

import numpy as np
import pytest
import torch

from _fp64 import FTZ, U, _adamw_ref, _f32, _report_margins, assert_close_elementwise  # noqa: F401
from _zero1_state import BF16, FP32, S16, State, chunks

pytestmark = pytest.mark.gpu

B1B, B8B = 60_821_504, 218_112_000  # llama3_1b and llama3_8b transformer blocks, in elements
PAD = 4096  # elements of each neighbouring unit around the unit under test (sentinel-filled)
LR, B1, EPS, WD = 1e-3, 0.9, 1e-8, 0.1
TS = (1, 2, 10, 100, 1000, 3000, 10 ** 4, 10 ** 6)
LR_STEPS = 50  # t = 1, 2, 10 read the table, later t its last entry
MAX_NORM = 1.0
NSM = 132
CAP = NSM * 32  # grid cap of both kernels
RS_DEFAULT, UPD_DEFAULT = 128, NSM * 16

RAN = set()  # kernel instances launched: ("reduce", W, clip, acc) / ("update", W, paged, clip, moments)
ACC_NAMES = {0: "off", 1: "acc", 2: "acc", 3: "last"}


def _expected_instances():
    red = {("reduce", w, c, a) for w in range(1, 9) for c in (False, True) for a in ("off", "acc", "last")
           if not (c and a == "acc") and not (w == 1 and not c and a == "off")}
    upd = {("update", w, p, c, m) for w in range(1, 9) for p in (False, True) for c in (False, True) for m in ("f32", "bf16")}
    return red | upd


# ----------------------------------------------------------------------------- worlds, geometry, data
_CUR = {}


def _world(W, n):
    """Pre-signalled virtual world of W ranks whose gradient and parameter segments hold a unit of n elements with PAD
    on each side. One world is alive at a time; the previous one is freed."""
    from torchft_b200.parallel.symm_mem import SymmetricComm

    if _CUR.get("key") == (W, n):
        return _CUR["comms"]
    _free()
    nb = (n + 2 * PAD) * 2
    comms = SymmetricComm.virtual_world(W, {"z1_grad": nb, "z1_param": nb, "z1_gnorm": 64}, presignal=True,
                                        timeout=timedelta(seconds=30))
    _CUR.update(key=(W, n), comms=comms)
    return comms


def _free(comms=None):
    own = comms is None
    comms = _CUR.pop("comms", None) if own else comms
    if own:
        _CUR.pop("key", None)
    if comms:
        torch.cuda.synchronize()
        for c in comms:
            c.shutdown()
        for c in comms:
            c.free_segments()
        torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _release_worlds():
    yield
    _free()


def _seg(c, name, n, dtype=BF16):
    return c.segment(name)[: (n + 2 * PAD) * 2].view(dtype)


def _slices(n, W):
    """[lo, hi) of slice s in elements, as the kernels' Geo cuts a unit of n elements into W slices."""
    nvec = n // 8
    sl = -(-nvec // W)
    return [(min(s * sl, nvec) * 8, min((s + 1) * sl, nvec) * 8) for s in range(W)]


def _held(r, W, k):
    return [(r - j) % W for j in range(min(k, W))]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _random_grad(n, seed):
    """bf16 values over 17 binades (no fp32 sum of a few of them underflows), one in 16 of them zero."""
    g = _gen(seed)
    x = torch.randn(n, device="cuda", generator=g)
    x *= torch.exp2(torch.randint(-8, 9, (n,), device="cuda", generator=g).float())
    x *= torch.rand(n, device="cuda", generator=g) >= 1 / 16
    return x.bfloat16()


def _small_grad(n, seed, who, contributors):
    """Values in {0, +-1, +-2, +-4}, each element non-zero for one contributor at most: every sum is a small integer, every
    square and every fp32 per-thread sum of squares exact."""
    g = _gen(seed)
    owner = torch.randint(0, contributors, (n,), device="cuda", generator=g)
    val = torch.tensor([0.0, 1, -1, 2, -2, 4, -4], device="cuda")[torch.randint(0, 7, (n,), device="cuda", generator=g)]
    return torch.where(owner == who, val, 0.0).bfloat16()


# ----------------------------------------------------------------------------- reduce + commit
def _reduce(comms, n, k, grid, clip, M, kind, seed, quiet=None):
    """Reduce-scatter of one unit over M micro-batches on every rank (the quiet rank first: its memset must precede the
    others' reads), then the commit when clipping. Checks everything the module docstring lists for reduce and commit."""
    W = len(comms)
    scale = 2.0 ** -5 if kind == "small" else 1.0 / (W * M)
    grads = [_seg(c, "z1_grad", n) for c in comms]
    for g in grads:
        g.view(torch.int16).fill_(S16)
    sl = _slices(n, W)
    # the first micro-batch must store, not add: the accumulators start as NaN
    accs = [torch.full((max(8, sl[r][1] - sl[r][0]),), float("nan"), device="cuda") for r in range(W)]
    gn = [c.segment("z1_gnorm").view(torch.float64) for c in comms]
    for x in gn:
        x.fill_(float("nan"))
    order = ([quiet] if quiet is not None else []) + [r for r in range(W) if r != quiet]

    def data(m, r):
        if r == quiet:
            return torch.zeros(n, dtype=BF16, device="cuda")
        if kind == "small":
            return _small_grad(n, seed + 1000 * m, r * M + m, W * M)
        return _random_grad(n, seed + 1000 * m + r)

    total = None
    for m in range(M):
        s = None
        for r in range(W):
            d = data(m, r)
            grads[r][PAD:PAD + n].copy_(d)
            s = d.float() if s is None else s + d.float()  # rank order, fp32, round to nearest: the kernel's sum
        total = s if total is None else total + s
        mode = 0 if M == 1 else (1 if m == 0 else (3 if m == M - 1 else 2))
        for r in order:
            comms[r].zero1_reduce_scatter_("z1_grad", PAD * 2, n, scale, r != quiet, k, grid, None,
                                           gnorm=gn[r].data_ptr() if clip and mode in (0, 3) else 0,
                                           acc=accs[r].data_ptr() if M > 1 else 0, acc_mode=mode)
            RAN.add(("reduce", W, bool(clip) and mode in (0, 3), ACC_NAMES[mode]))
        del s
    torch.cuda.synchronize()
    assert all(c.errored() is None for c in comms)
    want = (total * scale).bfloat16()
    del total
    last = {r: data(M - 1, r) for r in range(W)}
    tag = f"W={W} k={k} grid={grid} clip={clip} M={M} {kind} n={n}"
    for r in range(W):
        seg = grads[r].view(torch.int16)
        assert bool((seg[:PAD] == S16).all()) and bool((seg[PAD + n:] == S16).all()), f"neighbour units written ({tag}, rank {r})"
        exp = last[r].clone()
        for s in _held(r, W, k):
            exp[sl[s][0]:sl[s][1]] = want[sl[s][0]:sl[s][1]]
        got = grads[r][PAD:PAD + n]
        if not torch.equal(got.view(torch.int16), exp.view(torch.int16)):
            bad = (got.view(torch.int16) != exp.view(torch.int16)).nonzero()[:4].flatten().tolist()
            raise AssertionError(f"gradient segment of rank {r} differs at elements {bad} ({tag})")
    if not clip:
        return
    G = max(1, min(grid, CAP, (n // 8 + 511) // 512))
    Ur = _unroll(W, M > 1)
    parts = []
    for r in range(W):
        lo, hi = sl[r]
        exact = want[lo:hi].double().square().sum()
        got = gn[r][0]
        if kind == "small":
            assert float(got) == float(exact), f"clip partial of rank {r}: {float(got)!r} != {float(exact)!r} ({tag})"
        else:
            # per thread: 8 fused squares per vector into a fresh sum, then one add per vector into the thread's sum;
            # an element passes through at most 7 + (vectors per thread) fp32 roundings. The fp64 CTA sums add nothing
            # measurable at these lengths (<= 2^13 terms of 2^-53).
            nvpt = -(-((hi - lo) // 8) // (G * 512 * Ur)) * Ur
            chain = 7 + nvpt
            assert_close_elementwise(got.reshape(1), exact.reshape(1), ulps=0,
                                     abs_slack=(chain * U + 2.0 ** -40) * exact.reshape(1),
                                     what=f"reduce clip partial W={W} M={M}")
        parts.append(got)
    norms = [torch.zeros(2, device="cuda") for _ in comms]
    gates = [torch.zeros(2, dtype=torch.int32, device="cuda") for _ in comms]
    for r in range(W):
        comms[r].zero1_commit_(gates[r], True, True, None, gnorm="z1_gnorm", nunits=1, max_norm=MAX_NORM, norm=norms[r])
    torch.cuda.synchronize()
    for r in range(W):
        assert torch.equal(norms[r], norms[0]), f"norm / coef bits of rank {r} ({tag})"
        assert gates[r].tolist() == [1, 1]
    sq = torch.stack(parts).sum()
    # fp64 sum of W non-negative partials (W 2^-53) and an fp64 square root, then one rounding to fp32: half an ulp
    assert_close_elementwise(norms[0][:1], sq.sqrt().reshape(1), ulps=0.5, abs_slack=(W + 2) * 2.0 ** -53 * sq.sqrt().reshape(1),
                             what="commit norm")
    assert torch.equal(norms[0][1], torch.clamp(MAX_NORM / (norms[0][0] + 1e-6), max=1.0)), f"clip coefficient ({tag})"


def _unroll(W, acc):
    """reduce_unroll() of zero1.cu for the P2P path."""
    if not acc:
        return 2 if W >= 8 else 3 if W == 7 else 4 if W >= 3 else 8
    return 8 if W <= 1 else 4 if W <= 4 else 3 if W <= 6 else 2


REDUCE_CONFIGS = [(clip, M) for clip in (False, True) for M in (1, 3)]
GRIDS = (1, 7, RS_DEFAULT, CAP)


@pytest.mark.parametrize("W,k", [(w, k) for w in range(1, 9) for k in (1, 2, 3) if k <= w])
def test_reduce_and_commit_llama3_1b_block(W, k):
    comms = _world(W, B1B)
    for ci, (clip, M) in enumerate(REDUCE_CONFIGS):
        if W == 1 and not clip and M == 1:
            continue  # one rank without clipping or accumulation launches no reduce
        for j in (0, 2):
            grid = GRIDS[(ci + k + j) % 4]
            kind = "small" if j == 0 and clip else "random"
            quiet = W - 1 if (W >= 3 and ci == 3 and j == 2) else None
            _reduce(comms, B1B, k, grid, clip, M, kind, seed=100 * W + 10 * k + ci + j, quiet=quiet)


@pytest.mark.parametrize("W", range(1, 9))
def test_reduce_edge_units(W):
    for n in sorted({8, 56, 8 * W - 8, 8 * (3 * W + 1)} - {0}):
        comms = _world(W, n)
        for ci, (clip, M) in enumerate(REDUCE_CONFIGS):
            if W == 1 and not clip and M == 1:
                continue
            _reduce(comms, n, min(W, 1 + ci % 3), GRIDS[ci % 4], clip, M, "small" if clip else "random", seed=7 * n + ci)


# ----------------------------------------------------------------------------- update
def _init_state(n, sl, W, k, shift, soff, md, seed):
    """Every holder of slice s starts from the same seeded master / m / v."""
    states = [State(n, [sl[s] for s in _held(r, W, k) if sl[s][0] < sl[s][1]], shift, soff, md, seed + r) for r in range(W)]
    for s, (lo, hi) in enumerate(sl):
        for a, b in chunks(lo, hi):
            g = _gen(seed * 31 + s * 7 + a)
            w = torch.randn(b - a, device="cuda", generator=g) * 0.05
            m = torch.randn(b - a, device="cuda", generator=g) * 1e-3
            v = (torch.randn(b - a, device="cuda", generator=g) * 1e-3).square()
            if md == "bf16":
                m, v = m.bfloat16(), v.bfloat16()
            for r in range(W):
                if s in _held(r, W, k):
                    states[r].put(a, b, w, m, v)
    return states


def _nd_ranges(n, sl, shift, soff):
    """Weight-decay exemptions across the first slice boundary, across a page boundary, and at the ends of the unit."""
    out = []
    b = sl[0][1]
    if 0 < b < n:
        out.append((max(0, b - 40), min(n, b + 24)))
    page = 1 << (shift or 8)
    pb = ((soff + n // 3) // page + 1) * page - soff
    if 16 <= pb <= n - 24:
        out.append((pb - 16, pb + 24))
    out.append((0, 8))
    if n >= 16:
        out.append((n - 16, n))
    out = sorted(set(out))
    merged = []
    for lo, hi in out:
        if merged and lo <= merged[-1][1]:
            merged[-1] = (merged[-1][0], max(hi, merged[-1][1]))
        else:
            merged.append((lo, hi))
    return merged[:4]


def _lr_table(seed):
    tab = torch.rand(LR_STEPS, generator=torch.Generator().manual_seed(seed)) * LR
    return tab.cuda()


def _update_case(comms, n, k, shift, md, coef, lr_tab, nd, steps, grid, seed, refresh=False, record=True):
    """Steps ``steps`` = [(t, b2), ...] of the update on every rank from seeded state; each step is checked against one
    fp64 AdamW step from the kernel's state before it. Returns the final (params, states) for bit comparisons."""
    W = len(comms)
    sl = _slices(n, W)
    soff = 0 if shift is None else 8 * 37 + (1 << shift) * 3
    states = _init_state(n, sl, W, k, shift, soff, md, seed)
    grads = [_seg(c, "z1_grad", n) for c in comms]
    params = [_seg(c, "z1_param", n) for c in comms]
    coef_t = torch.tensor([coef if coef is not None else 1.0], device="cuda")
    tag = f"W={W} k={k} n={n} shift={shift} {md} coef={coef} lr_tab={lr_tab is not None} nd={len(nd)} grid={grid}"
    for step, (t, b2) in enumerate(steps):
        g = _random_grad(n, seed * 13 + step)
        for x in grads:
            x[PAD:PAD + n].copy_(g)
        for p in params:
            p.view(torch.int16).fill_(S16)
        before = [[states[s].get(a, b) for a, b in chunks(*sl[s])] for s in range(W)]  # primary holder s of slice s
        gates = [torch.tensor([1, t], dtype=torch.int32, device="cuda") for _ in comms]
        for r, c in enumerate(comms):
            st = states[r]
            c.zero1_update_("z1_param", PAD * 2, grads[r].data_ptr() + PAD * 2, nelem=n, hyper=(LR, B1, b2, EPS, WD),
                            gate=gates[r], replication=k, mode=0, blocks=grid,
                            coef=coef_t.data_ptr() if coef is not None else 0,
                            lr_table=lr_tab.data_ptr() if lr_tab is not None else 0,
                            lr_steps=LR_STEPS if lr_tab is not None else 0, no_decay=nd, **st.args())
            if record:
                RAN.add(("update", W, shift is not None, coef is not None, md))
        torch.cuda.synchronize()
        assert all(c.errored() is None for c in comms)
        lr = float(lr_tab[min(max(t, 1), LR_STEPS) - 1]) if lr_tab is not None else LR
        what = f"{'bf16' if md == 'bf16' else 'f32'} b2={b2}"
        full_master = torch.empty(n, device="cuda")
        for s, (lo, hi) in enumerate(sl):
            for (a, b), (w0, m0, v0) in zip(chunks(lo, hi), before[s]):
                w1, m1, v1 = states[s].get(a, b)
                full_master[a:b] = w1
                for r in range(W):  # every holder stores the primary's bits
                    if r != s and s in _held(r, W, k):
                        for x, y, name in zip((w1, m1, v1), states[r].get(a, b), ("master", "m", "v")):
                            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"holder {r} of slice {s}: {name} ({tag} t={t})"
                gs = coef if coef is not None else 1.0
                wd = torch.full((b - a,), _f32(WD), dtype=torch.float64, device="cuda")
                for x0, x1 in nd:
                    if x0 < b and x1 > a:
                        wd[max(x0, a) - a:min(x1, b) - a] = 0.0
                if md == "f32":
                    w_ref, w_sl, m_ref, m_sl, v_ref, v_sl = _adamw_ref(w0, m0, v0, g[a:b], lr, B1, b2, EPS, wd, t,
                                                                      gs, m1, v1)
                    upd = (w_ref - w0.double() * (1 - _f32(lr) * wd)).abs()
                    assert_close_elementwise(m1, m_ref, ulps=0, abs_slack=m_sl + FTZ, what=f"update m {what}")
                    assert_close_elementwise(v1, v_ref, ulps=0, abs_slack=v_sl + FTZ, what=f"update v {what}")
                    # + 3 U of the update: the fp64 pow of the bias corrections rounds to the reference's fp32 value
                    # except at a near-tie, one ulp away (2 U through 1 / bc1, 1 U through 1 / sqrt(bc2))
                    assert_close_elementwise(w1, w_ref, ulps=1, abs_slack=w_sl + 3 * U * upd + FTZ,
                                             what=f"update master {what}")
                else:
                    _, _, m_ref, m_sl, v_ref, v_sl = _adamw_ref(w0, m0, v0, g[a:b], lr, B1, b2, EPS, wd, t, gs,
                                                               m0, v0)
                    w_ref, w_sl, *_ = _adamw_ref(w0, m0, v0, g[a:b], lr, B1, b2, EPS, wd, t, gs, m_ref, v_ref)
                    upd = (w_ref - w0.double() * (1 - _f32(lr) * wd)).abs()
                    bc1, bc2 = _f32(1 - _f32(B1) ** t), _f32(1 - _f32(b2) ** t)
                    denom = v_ref.sqrt() / math.sqrt(bc2) + _f32(EPS)
                    # the weights use the kernel's fp32 moments, within m_sl / v_sl of the reference: m_sl enters the
                    # update through lr / bc1 / denom, v's 5 U relative through the square root as 2.5 U (3 U)
                    w_sl = w_sl + (3 + 3) * U * upd + (_f32(lr) / bc1) * m_sl / denom
                    assert_close_elementwise(w1, w_ref, ulps=1, abs_slack=w_sl + FTZ, what=f"update master {what}")
                    _assert_bf16_neighbour(m1, m_ref, m_sl + FTZ, f"update m {what} ({tag} t={t})")
                    _assert_bf16_neighbour(v1, v_ref, v_sl + FTZ, f"update v {what} ({tag} t={t})")
                    _assert_zero_gradient_rounding(g[a:b], soff + a, t, b2, m0, v0, m1, v1, f"{tag} t={t}")
        want = full_master.bfloat16()
        for r in range(W):
            p = params[r].view(torch.int16)
            assert bool((p[:PAD] == S16).all()) and bool((p[PAD + n:] == S16).all()), f"neighbour weights written ({tag})"
            assert torch.equal(p[PAD:PAD + n], want.view(torch.int16)), f"weights of rank {r} ({tag} t={t})"
            assert states[r].untouched(), f"state outside the held ranges of rank {r} ({tag})"
    if refresh:
        for p in params:
            p.view(torch.int16).fill_(S16)
        gates = [torch.tensor([0, steps[-1][0]], dtype=torch.int32, device="cuda") for _ in comms]
        for r, c in enumerate(comms):
            st = states[r]
            c.zero1_update_("z1_param", PAD * 2, grads[r].data_ptr() + PAD * 2, nelem=n,
                            hyper=(LR, B1, steps[-1][1], EPS, WD), gate=gates[r], replication=k, mode=1, blocks=grid,
                            **st.args())
        torch.cuda.synchronize()
        for r in range(W):
            assert torch.equal(params[r].view(torch.int16)[PAD:PAD + n], want.view(torch.int16)), f"refresh of rank {r} ({tag})"
    return [p[PAD:PAD + n].clone() for p in params], states


def _assert_zero_gradient_rounding(g, e0, t, b2, m0, v0, m1, v1, what):
    """Where the gradient is zero the kernel's fp32 moments are the single rounded products b1 * m and b2 * v, so the
    stored bits are exactly what ``bf16_sr``, the specification of the device rounding, makes of them."""
    from torchft_b200.parallel.zero1 import bf16_sr

    idx = (g == 0).nonzero().flatten()
    assert idx.numel() > 0 or g.numel() < 64
    if idx.numel() == 0:
        return
    e = (idx + e0).cpu().numpy().astype(np.uint64)
    for name, b, x0, x1, which in (("m", B1, m0, m1, 0), ("v", b2, v0, v1, 1)):
        want = bf16_sr(np.float32(b) * x0[idx].float().cpu().numpy(), e, t, which)
        got = x1[idx].view(torch.int16).cpu().numpy().view(np.uint16)
        assert (got == want).all(), f"{name}: {int((got != want).sum())} of {idx.numel()} zero-gradient elements ({what})"


def _assert_bf16_neighbour(stored, ref, slack, what):
    """``stored`` (bf16) is one of the two bf16 neighbours of a value within ``slack`` of the fp64 ``ref``: the kernel's
    fp32 moment lies in that interval and is rounded stochastically to one of its bf16 neighbours."""
    def towards(x, away):
        bits = x.contiguous().view(torch.int32)
        return ((bits + 0xFFFF if away else bits) & ~0xFFFF).view(torch.float32)

    lo64, hi64 = ref - slack, ref + slack
    # the fp32 bounds are widened by an fp32 ulp so their own rounding cannot cut off a neighbour
    lo_f = (lo64 - 2 * U * lo64.abs()).float()
    hi_f = (hi64 + 2 * U * hi64.abs()).float()
    lo = torch.where(lo_f >= 0, towards(lo_f, False), towards(lo_f, True))  # the largest bf16 <= lo_f
    hi = torch.where(hi_f >= 0, towards(hi_f, True), towards(hi_f, False))  # the smallest bf16 >= hi_f
    s = stored.float()
    ok = (s >= lo) & (s <= hi)
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} stored moments are not a bf16 neighbour of the reference"


def _update_cases(W):
    """Eight cases per world, one per template instance (paging x clipping x moment type); the replication, page size,
    schedule, exemptions, grid and step counts rotate over them so that each appears at every world."""
    cases = []
    for i, (paged, clip, md) in enumerate(itertools.product((False, True), (False, True), ("f32", "bf16"))):
        j = i + W
        k = 1 + j % min(W, 3)
        shift = (16 if j % 2 else 8) if paged else None
        steps = [(TS[j % 8], 0.999), (TS[(j + 3) % 8], 0.95), (TS[(j + 5) % 8], 0.999)]
        cases.append(dict(k=k, shift=shift, md=md, coef=0.37 if clip else None, lr_tab=j % 2 == 1, nd=j % 3 != 0,
                          grid=(1, UPD_DEFAULT, 3, CAP)[j % 4], steps=steps))
    assert {(c["shift"] is not None, c["coef"] is not None, c["md"]) for c in cases} == \
        set(itertools.product((False, True), (False, True), ("f32", "bf16")))
    return cases


@pytest.mark.parametrize("W", range(1, 9))
def test_update_llama3_1b_block(W):
    comms = _world(W, B1B)
    for i, c in enumerate(_update_cases(W)):
        sl = _slices(B1B, W)
        soff = 0 if c["shift"] is None else 8 * 37 + (1 << c["shift"]) * 3
        nd = _nd_ranges(B1B, sl, c["shift"], soff) if c["nd"] else []
        _update_case(comms, B1B, c["k"], c["shift"], c["md"], c["coef"], _lr_table(i) if c["lr_tab"] else None, nd,
                     c["steps"], c["grid"], seed=10 * W + i, refresh=5 <= W <= 7 and i < 2)


@pytest.mark.parametrize("W", range(1, 9))
def test_update_edge_units(W):
    for n in sorted({8, 56, 8 * W - 8, 8 * (3 * W + 1)} - {0}):
        comms = _world(W, n)
        for i, c in enumerate(_update_cases(W)):
            sl = _slices(n, W)
            soff = 0 if c["shift"] is None else 8 * 37 + (1 << c["shift"]) * 3
            nd = _nd_ranges(n, sl, c["shift"], soff) if c["nd"] else []
            _update_case(comms, n, c["k"], c["shift"], c["md"], c["coef"], _lr_table(i) if c["lr_tab"] else None, nd,
                         c["steps"][:1], c["grid"], seed=100 * W + 10 * i + n % 10, refresh=5 <= W <= 7)


@pytest.mark.parametrize("W", [7, 8])
def test_llama3_8b_block(W):
    comms = _world(W, B8B)
    _reduce(comms, B8B, 2, RS_DEFAULT, True, 1, "random", seed=W)
    _reduce(comms, B8B, 2, CAP, False, 3, "random", seed=W + 1)
    sl = _slices(B8B, W)
    md = "bf16" if W == 7 else "f32"
    _update_case(comms, B8B, 2, 16, md, 0.37, _lr_table(W), _nd_ranges(B8B, sl, 16, 8 * 37 + (3 << 16)),
                 [(1000, 0.999), (1, 0.95)], UPD_DEFAULT, seed=W)
    _free()


# ----------------------------------------------------------------------------- grid and ordering
def test_bits_do_not_depend_on_the_grid_or_on_real_signalling():
    from torchft_b200.parallel.symm_mem import SymmetricComm

    W, k, n = 7, 2, B1B
    comms = _world(W, n)
    for grid in (1, 3, RS_DEFAULT):
        _reduce(comms, n, k, grid, True, 1, "random", seed=5)  # bit for bit against the same reference at each grid
    runs = {}
    for grid in (1, 3, UPD_DEFAULT):
        params, states = _update_case(comms, n, k, 16, "bf16", 0.37, None, [], [(10, 0.999)], grid, seed=9, record=False)
        runs[grid] = [params] + [[torch.cat([st.get(lo, hi)[i].view(torch.uint8) for lo, hi in st.held]) for i in range(3)]
                                 for st in states]
    for grid, r in runs.items():
        for a, b in zip(runs[1], r):
            for x, y in zip(a, b):
                assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"grid {grid} differs from grid 1"
    ref_params = runs[1][0]
    _free()

    # the same pipeline with real signalling, every rank on its own stream, concurrently
    nb = (n + 2 * PAD) * 2
    live = SymmetricComm.virtual_world(W, {"z1_grad": nb, "z1_param": nb, "z1_gnorm": 64}, presignal=False,
                                       timeout=timedelta(seconds=60))
    try:
        sl = _slices(n, W)
        soff = 8 * 37 + (3 << 16)
        states = _init_state(n, sl, W, k, 16, soff, "bf16", 9)
        g = _random_grad(n, 9 * 13)
        for c in live:
            _seg(c, "z1_grad", n)[PAD:PAD + n].copy_(g)
            _seg(c, "z1_param", n).view(torch.int16).fill_(S16)
        coef = torch.tensor([0.37], device="cuda")
        gates = [torch.tensor([1, 10], dtype=torch.int32, device="cuda") for _ in live]
        streams = [torch.cuda.Stream() for _ in live]
        torch.cuda.synchronize()
        for r, c in enumerate(live):
            st = states[r]
            with torch.cuda.stream(streams[r]):
                c.zero1_update_("z1_param", PAD * 2, _seg(c, "z1_grad", n).data_ptr() + PAD * 2, nelem=n,
                                hyper=(LR, B1, 0.999, EPS, WD), gate=gates[r], replication=k, mode=0,
                                blocks=UPD_DEFAULT, stream=streams[r], coef=coef.data_ptr(), **st.args())
        torch.cuda.synchronize()
        assert all(c.errored() is None for c in live)
        for r, c in enumerate(live):
            assert torch.equal(_seg(c, "z1_param", n)[PAD:PAD + n].view(torch.int16), ref_params[r].view(torch.int16)), \
                f"rank {r}: concurrent weights differ from the pre-signalled run"
            for i in range(3):
                got = torch.cat([states[r].get(lo, hi)[i].view(torch.uint8) for lo, hi in states[r].held])
                assert torch.equal(got, runs[1][1 + r][i]), f"rank {r}: concurrent state {i} differs"
    finally:
        _free(live)


# ----------------------------------------------------------------------------- world one against the flat optimizer
def test_world_one_update_stores_the_bits_of_the_flat_optimizer():
    """The same state, gradient and t through ``zero1_update`` at W = 1 (flat state, fp32 moments, no extras) and through
    ``FlatAdamW``'s kernel: both take 1 - b^t of the fp32 betas, rounded once, so every stored bit agrees."""
    from torchft_b200.ops import fused

    n = B1B
    comms = _world(1, n)
    c = comms[0]
    grad, param = _seg(c, "z1_grad", n), _seg(c, "z1_param", n)
    st = State(n, [(0, n)], None, 0, "f32", 0)
    for b2 in (0.95, 0.999):
        for t in TS:
            gen = _gen(t)
            w = torch.randn(n, device="cuda", generator=gen) * 0.05
            m = torch.randn(n, device="cuda", generator=gen) * 1e-3
            v = (torch.randn(n, device="cuda", generator=gen) * 1e-3).square()
            g = _random_grad(n, t + 1)
            st.put(0, n, w, m, v)
            grad[PAD:PAD + n].copy_(g)
            gate = torch.tensor([1, t], dtype=torch.int32, device="cuda")
            c.zero1_update_("z1_param", PAD * 2, grad.data_ptr() + PAD * 2, nelem=n, hyper=(LR, B1, b2, EPS, WD),
                            gate=gate, replication=1, mode=0, blocks=UPD_DEFAULT, **st.args())
            opt = fused.FlatAdamW(torch.empty(n, dtype=BF16, device="cuda"), g.clone(), lr=LR, betas=(B1, b2), eps=EPS,
                                  weight_decay=WD)
            opt.master.copy_(w)
            opt.m.copy_(m)
            opt.v.copy_(v)
            opt.t = t - 1
            opt.step()
            torch.cuda.synchronize()
            for name, x, y in (("master", st.master, opt.master), ("m", st.m, opt.m), ("v", st.v, opt.v),
                               ("weights", param[PAD:PAD + n], opt.p)):
                same = x.view(torch.uint8).view(-1, 4 if x.dtype == FP32 else 2) == y.view(torch.uint8).view(-1, 4 if y.dtype == FP32 else 2)
                assert bool(same.all()), f"{name} at t={t} b2={b2}: {int((~same.all(1)).sum())} elements differ"
    _free()


def test_every_kernel_instance_ran():
    """Every instance the launchers pick for W <= 8 without multicast ran above (run the whole module)."""
    missing = sorted(_expected_instances() - RAN, key=str)
    assert not missing, f"never launched: {missing}"
    assert {w for _, w, *_ in RAN} == set(range(1, 9))
