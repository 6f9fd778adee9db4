"""Every fp8 (Q8G) quantised-collective entry point against the bit-exact CPU emulation in ``_q8_emulation``: scale and
payload bytes, output bits, on every rank of the one-GPU virtual world of ``test_collectives_gpu``. Also the contract of
the edge groups: a finite group whose amax is a normal fp32 never dequantises to all zeros or to NaN, and an inf anywhere
in a group (or an fp32 overflow of its sum) makes the whole group NaN, as the unquantised sum is non-finite there."""

from __future__ import annotations

import math
import threading

import pytest
import torch

import _q8_emulation as E
from _collectives import _ok, _run, _world

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
DTYPES = (torch.float32, torch.bfloat16, torch.float16)


def _dev(xs):
    return [x.to(DEV) for x in xs]


def _msg(n, world, seed, dtype, scale=1.0):
    """``E.message`` scaled into the range of ``dtype`` (fp16 overflows past 65504)."""
    return [(x * scale).to(dtype) for x in E.message(n, world, seed)]


def _fp16_safe(dtype):
    return 1e-3 if dtype == torch.float16 else 1.0


def _assert_bits(got, want, what):
    assert E.equal_bits(got, want), f"{what}: {E.first_mismatch(got, want)}"


def _assert_q8(got, want, what):
    if not E.equal_q8(got, want):
        sg = (got.scales.view(torch.int32) != want.scales.view(torch.int32)) & ~(torch.isnan(got.scales) & torch.isnan(want.scales))
        cg = (got.codes != want.codes).any(1)
        raise AssertionError(f"{what}: scales differ in groups {sg.nonzero().view(-1)[:8].tolist()}, "
                             f"codes in groups {cg.nonzero().view(-1)[:8].tolist()} of {want.ng}")


def _staging(c, nbytes):
    return c.segment("core")[c._pad_bytes: c._pad_bytes + nbytes]


# ------------------------------------------------------------------------------------------------ standalone kernels
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", [1, 3, 8])
def test_quantize_dequantize_exact(dtype, world):
    from torchft_b200 import quantization as Q

    for n in (1, 15, 16, 17, 511, 512, 513, 512 * world * 3 - 8, 100_003):
        a, b = _msg(n, 2, n, dtype, _fp16_safe(dtype))
        for sub in (None, b):
            buf = Q.quantize_q8(a.to(DEV), world_size=world, subtract=None if sub is None else sub.to(DEV))
            ng = E.ngroups(n, world)
            assert buf.numel() == E.buffer_bytes(n, world)
            want = E.quantize(E.pseudo_grad(a, sub), ng)
            _assert_q8(E.Q8.from_bytes(buf, ng), want, f"quantize n={n} sub={sub is not None}")
            pad = E.Q8.from_bytes(buf, ng)[(n + E.GROUP - 1) // E.GROUP:]  # groups padded for the world: all zero
            assert torch.equal(pad.codes, torch.zeros_like(pad.codes))
            out = Q.dequantize_q8(buf, n, dtype, world_size=world)
            _assert_bits(out, E.cast(E.dequant(want).reshape(-1)[:n], dtype), f"dequantize n={n}")


@pytest.mark.parametrize("world", [2, 3, 8])
def test_fused_quantize_reduce_dequantize_exact(world):
    """``fused_quantize_into_fp8`` / ``fused_reduce_fp8`` / ``fused_dequantize_from_fp8`` over a list of tensors of
    mixed shapes and dtypes, every rank holding different data; rank r reduces its slice from rank r on."""
    from torch.distributed import ReduceOp

    from torchft_b200 import quantization as Q

    shapes = [((7, 3), torch.float32), ((1000,), torch.bfloat16), ((33, 129), torch.float16), ((2, 2, 512), torch.float32)]
    data = [[_msg(int(torch.tensor(s).prod()), 1, 10 * r + i, dt, _fp16_safe(dt))[0].view(s) for i, (s, dt) in enumerate(shapes)]
            for r in range(world)]
    bufs = [Q.fused_quantize_into_fp8(_dev(d), world) for d in data]
    offs, _ = Q._layout(data[0], world)
    for r in range(world):
        for t, o in zip(data[r], offs):
            ng = E.ngroups(t.numel(), world)
            _assert_q8(E.Q8.from_bytes(bufs[r][o:], ng), E.quantize(E.load(t), ng), f"fused quantize rank {r}")
    final = torch.empty_like(bufs[0])
    ins = _dev(data[0])  # fused_reduce_fp8 builds its device pointer table on the inputs' device
    for op, post in ((ReduceOp.SUM, 1.0), (ReduceOp.AVG, 1.0 / world)):
        for rank in range(world):
            copies = [b.clone() for b in bufs]
            Q.fused_reduce_fp8(ins, copies, world, rank, op)
            for i, (t, o) in enumerate(zip(data[0], offs)):
                ng = E.ngroups(t.numel(), world)
                sl = ng // world
                parts = [E.quantize(E.load(data[p][i]), ng)[rank * sl:(rank + 1) * sl] for p in range(world)]
                red = E.group_quant(E.reduce(parts, torch.full((sl,), rank), post, start_zero=True))
                _assert_q8(E.Q8.from_bytes(copies[rank][o:], ng)[rank * sl:(rank + 1) * sl], red, f"fused reduce rank {rank}")
            Q.copy_rank_slice(data[0], final, copies[rank], world, rank)
        outs = [torch.empty_like(t, device=DEV) for t in data[0]]
        Q.fused_dequantize_from_fp8(outs, final, world)
        for i, (t, o) in enumerate(zip(outs, offs)):
            ng = E.ngroups(t.numel(), world)
            got = E.Q8.from_bytes(final[o:], ng)
            _assert_bits(t, E.cast(E.dequant(got).reshape(-1)[: t.numel()], t.dtype), f"fused dequantize tensor {i}")


def test_standalone_launchers_exact():
    """``q8_quantize`` with more groups than the data needs, ``q8_reduce`` over a sub-range of groups with
    ``first`` != 0, ``q8_dequantize`` of fewer elements than the groups hold."""
    from torchft_b200.ops import _native

    K, sp = _native.load(), _native.stream_ptr()
    W, n, ng = 3, 2000, 9
    xs = _msg(n, W, 5, torch.bfloat16)
    bufs = [torch.zeros(E.payload_off(ng) + ng * E.GROUP, dtype=torch.uint8, device=DEV) for _ in range(W)]
    xd = _dev(xs)
    for x, b in zip(xd, bufs):
        K.q8_quantize(x.data_ptr(), 0, n, ng, _native.dtype_code(x), b.data_ptr(), sp)
    qs = [E.quantize(E.load(x), ng) for x in xs]
    for r in range(W):
        _assert_q8(E.Q8.from_bytes(bufs[r], ng), qs[r], f"quantize rank {r}")
    dst = torch.zeros_like(bufs[0])
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=DEV)
    K.q8_reduce(ptrs.data_ptr(), W, 2, ng, 2, 7, 0.25, dst.data_ptr(), sp)
    red = E.group_quant(E.reduce([q[2:7] for q in qs], torch.full((5,), 2), 0.25, start_zero=True))
    got = E.Q8.from_bytes(dst, ng)
    _assert_q8(got[2:7], red, "reduce")
    assert torch.equal(got.scales[:2], torch.zeros(2)) and torch.equal(got.scales[7:], torch.zeros(2))
    out = torch.zeros(1500, dtype=torch.float16, device=DEV)
    K.q8_dequantize(dst.data_ptr(), ng, out.data_ptr(), 1500, _native.dtype_code(out), sp)
    _assert_bits(out, E.cast(E.dequant(got).reshape(-1)[:1500], torch.float16), "dequantize")


# ------------------------------------------------------------------------------------------------ fused all-reduce
def _fused_case(comms, n, dtype, seed, with_b=True, alias=False, quiet=None, scale=None):
    W = len(comms)
    scale = 1.0 / W if scale is None else scale
    a = _msg(n, W, seed, dtype, _fp16_safe(dtype))
    b = _msg(n, W, seed + 1, dtype, _fp16_safe(dtype)) if with_b else [None] * W
    ad = _dev(a)
    bd = [None if x is None else x.to(DEV) for x in b]
    outs = ad if alias else [torch.empty(n, dtype=dtype, device=DEV) for _ in range(W)]
    contribute = [r != quiet for r in range(W)]
    return a, b, ad, bd, outs, contribute, scale


@pytest.mark.parametrize("world", [2, 3, 5, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_q8_allreduce_exact(world, dtype):
    """Output bits, the reduced Q8G message in every rank's staging buffer, the same result on every rank; with and
    without ``b``, ``out`` aliasing ``a``, one rank not contributing; message sizes around group and slice edges, so the
    grid runs from 4 blocks up to ``_q8_max_blocks``."""
    comms = _world(world)
    sizes = [1, 15, 16, 17, 511, 512, 513, 512 * world * 3 - 8, 512 * world * 3 + 8, 100_003, (1 << 20) + 24]
    for i, n in enumerate(sizes):
        with_b, alias, quiet = i % 2 == 0, i % 3 == 1, (world - 1 if i % 4 == 3 else None)
        a, b, ad, bd, outs, contribute, scale = _fused_case(comms, n, dtype, 100 + i, with_b, alias, quiet)
        _run(comms, lambda r, c, s: c.q8_allreduce_(outs[r], ad[r], bd[r], scale=scale, contribute=contribute[r], stream=s))
        _ok(comms)
        xs = [E.pseudo_grad(x, y) for x, y in zip(a, b)]
        want, red = E.allreduce(xs, scale, contribute)
        case = f"n={n} b={with_b} alias={alias} quiet={quiet}"
        _assert_bits(outs[0], E.cast(want, dtype), case)
        for r, c in enumerate(comms):
            assert E.equal_bits(outs[r], outs[0]), f"rank {r} differs from rank 0: {case}"
            _assert_q8(E.Q8.from_bytes(_staging(c, E.buffer_bytes(n, world)), red.ng), red, f"staging of rank {r}: {case}")


@pytest.mark.parametrize("world", [2, 3])
def test_q8_allreduce_in_several_launches_exact(world):
    """A staging buffer small enough that the message takes three or more launches: each launch has its own group grid
    and slice owners, and the staging buffers keep the reduced message of the last one."""
    comms = _world(world, staging=1 << 20)
    per = E.staging_chunk(comms[0]._staging_usable, world)
    for n, dtype in ((3 * per + 1000, torch.float32), (4 * per, torch.bfloat16)):
        a, b, ad, bd, outs, contribute, scale = _fused_case(comms, n, dtype, 7)
        before = [c.launches for c in comms]
        _run(comms, lambda r, c, s: c.q8_allreduce_(outs[r], ad[r], bd[r], scale=scale, stream=s))
        _ok(comms)
        assert [c.launches - x for c, x in zip(comms, before)] == [math.ceil(n / per)] * world >= [3] * world
        want, red = E.allreduce([E.pseudo_grad(x, y) for x, y in zip(a, b)], scale, per=per)
        _assert_bits(outs[0], E.cast(want, dtype), f"n={n}")
        last = n - (math.ceil(n / per) - 1) * per
        for r, c in enumerate(comms):
            assert E.equal_bits(outs[r], outs[0])
            _assert_q8(E.Q8.from_bytes(_staging(c, E.buffer_bytes(last, world)), red.ng), red, f"staging of rank {r}")


@pytest.mark.parametrize("world", [2, 3, 8])
def test_q8_allreduce_scratch_pipeline_exact(world):
    """The ``*_q8`` scratch segment pipeline: each rank's scratch holds its quantised input (zeros when it does not
    contribute), its reduced slice follows at ``round_up(buffer_bytes, 256)``, and the output bits are the emulation's."""
    nmax = (1 << 20) + 24
    comms = _world(world, segs={"buf": 1 << 20, "frag_q8": E.buffer_bytes(nmax, world) + 256 + E.slice_buffer_bytes(nmax, world)})
    for i, (n, dtype) in enumerate(((nmax, torch.float32), (100_003, torch.bfloat16), (513, torch.float16), (17, torch.float32))):
        quiet = 1 if i % 2 == 1 else None
        a, b, ad, bd, outs, contribute, scale = _fused_case(comms, n, dtype, 30 + i, with_b=i != 2, quiet=quiet)
        before = [c.launches for c in comms]
        _run(comms, lambda r, c, s: c.q8_allreduce_(outs[r], ad[r], bd[r], scale=scale, contribute=contribute[r], stream=s))
        _ok(comms)
        assert [c.launches - x for c, x in zip(comms, before)] == [5] * world
        want, mine, reds = E.allreduce_scratch([E.pseudo_grad(x, y) for x, y in zip(a, b)], scale, contribute)
        case = f"n={n} {dtype} quiet={quiet}"
        _assert_bits(outs[0], E.cast(want, dtype), case)
        ng = E.ngroups(n, world)
        q_bytes = (E.buffer_bytes(n, world) + 255) // 256 * 256
        for r, c in enumerate(comms):
            assert E.equal_bits(outs[r], outs[0])
            seg = c.segment("frag_q8")
            _assert_q8(E.Q8.from_bytes(seg, ng), mine[r], f"scratch of rank {r}: {case}")
            _assert_q8(E.Q8.from_bytes(seg[q_bytes:], ng // world), reds[r], f"reduced slice of rank {r}: {case}")


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_q8_reduce_scatter_exact(world, dtype):
    """Mode 1: every rank-slice on its own group grid, the fp32 sum cast straight to the output. Slices that are not a
    multiple of 512 and inputs shorter than ``world * slice_elems``: a partial last slice, and empty ones."""
    comms = _world(world, staging=16 << 20)
    for i, (se, n) in enumerate(((1000, world * 1000), (1000, world * 1000 - 300), (4104, 4104 * (world - 1) + 8),
                                 (520, 520 * max(1, world - 2)), (8, world * 8), (65536, world * 65536 - 24))):
        quiet = 0 if i == 2 else None
        ins = _msg(n, world, 50 + i, dtype, _fp16_safe(dtype))
        ind = _dev(ins)
        outs = [torch.full((se,), 7.0, dtype=dtype, device=DEV) for _ in range(world)]
        contribute = [r != quiet for r in range(world)]
        _run(comms, lambda r, c, s: c.q8_reduce_scatter_(outs[r], ind[r], se, scale=1.0 / world, contribute=contribute[r], stream=s))
        _ok(comms)
        want = E.reduce_scatter([E.load(x) for x in ins], se, 1.0 / world, contribute)
        gs = (se + E.GROUP - 1) // E.GROUP
        for r, c in enumerate(comms):
            valid = want[r].numel()
            case = f"rank {r} se={se} n={n} valid={valid}"
            _assert_bits(outs[r][:valid], E.cast(want[r], dtype), case)
            assert torch.equal(outs[r][valid:].float().cpu(), torch.full((se - valid,), 7.0)), case  # past the input
            if contribute[r]:  # phase A left this rank's quantised input, slice by slice, in its staging buffer
                mine = E.Q8.cat([E.quantize(E.load(ins[r])[s * se: min(n, (s + 1) * se)], gs) for s in range(world)])
                _assert_q8(E.Q8.from_bytes(_staging(c, E.payload_off(mine.ng) + mine.ng * E.GROUP), mine.ng), mine, case)


# ------------------------------------------------------------------------------------------------ generic path
class _FakePG:
    """One rank of an in-process process group: ``alltoall_base`` and ``allgather`` copy between the ranks' tensors after
    every rank has arrived (``threading.Barrier``), with the device synchronised around the copies."""

    def __init__(self, rank, world, shared):
        self._r, self._w, self._s = rank, world, shared

    def size(self):
        return self._w

    def rank(self):
        return self._r

    def _exchange(self, mine):
        torch.cuda.current_stream().synchronize()
        self._s["slots"][self._r] = mine
        self._s["barrier"].wait()
        yield self._s["slots"]
        torch.cuda.current_stream().synchronize()
        self._s["barrier"].wait()

    def alltoall_base(self, out, inp, out_splits, in_splits, opts):
        for slots in self._exchange(inp):
            for q in range(self._w):
                out.view(self._w, -1)[q].copy_(slots[q].view(self._w, -1)[self._r])
        return self

    def allgather(self, outs, ins, opts):
        for slots in self._exchange(ins[0]):
            for q in range(self._w):
                outs[0][q].copy_(slots[q])
        return self

    def wait(self, timeout=None):
        return True


def _threaded(world, fn):
    shared = {"barrier": threading.Barrier(world, timeout=60), "slots": [None] * world}
    errs = []

    def body(r):
        try:
            fn(r, _FakePG(r, world, shared))
            torch.cuda.synchronize()
        except BaseException as e:  # noqa: BLE001
            errs.append(e)
            shared["barrier"].abort()

    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]


@pytest.mark.parametrize("world", [2, 3, 8])
def test_generic_allreduce_and_reduce_scatter_quantized_exact(world):
    """``collectives.allreduce_quantized`` / ``reduce_scatter_quantized`` over a process group without the fused
    kernels: slices of a ``_SlicePlan`` quantised per rank, reduced from the own rank on, requantised, gathered."""
    from torch.distributed import ReduceOp

    from torchft_b200 import collectives as C

    specs = [((5,), torch.float32), ((1000, 3), torch.bfloat16), ((64, 129), torch.float16), ((513,), torch.float32)]
    data = [[_msg(int(torch.tensor(s).prod()), 1, 70 * r + i, dt, _fp16_safe(dt))[0].view(s) for i, (s, dt) in enumerate(specs)]
            for r in range(world)]
    for avg in (False, True):
        ts = [_dev(d) for d in data]
        _threaded(world, lambda r, pg: C.allreduce_quantized(ts[r], ReduceOp.AVG if avg else ReduceOp.SUM, pg).wait())
        want = E.allreduce_quantized(data, avg)
        for r in range(world):
            for i, (t, w) in enumerate(zip(ts[r], want)):
                _assert_bits(t, E.cast(w, t.dtype).view(t.shape), f"allreduce rank {r} tensor {i} avg={avg}")
    for rs_specs in (((world * 4, 64), (world * 2 + 1, 512), (7, 8)), ((3, 5), (world, 1001))):  # aligned / unaligned slices
        for dtype in (torch.bfloat16, torch.float32):
            inputs = [[_msg(a * b, 1, 90 * r + a, dtype)[0].view(a, b) for a, b in rs_specs] for r in range(world)]
            ind = [_dev(x) for x in inputs]
            outs = [C.allocate_reduce_scatter_output(ind[r], world)[0] for r in range(world)]
            _threaded(world, lambda r, pg: C.reduce_scatter_quantized(outs[r], ind[r], ReduceOp.AVG, pg).wait())
            want = E.reduce_scatter_quantized(inputs, True, torch.tensor([], dtype=dtype).element_size())
            for r in range(world):
                _assert_bits(outs[r], E.cast(want[r], dtype), f"reduce-scatter rank {r} {rs_specs} {dtype}")


# ------------------------------------------------------------------------------------------------ edge groups
def _edge_groups(dtype):
    """(name, ranks, 512 values) of the special groups; ``ranks`` None means every rank."""
    G = E.GROUP
    z = torch.zeros(G)
    one = z.clone()
    one[77] = -3.0
    pow448 = torch.tensor([448.0 * 2.0 ** k * (-1) ** k for k in range(-20, 8)])  # up to 57344: finite in fp16
    powg = z.clone()
    powg[: pow448.numel()] = pow448
    mid = z.clone()  # amax 448 -> m = 1: every value sits exactly between two e4m3 neighbours
    mid[0] = 448.0
    mid[1:9] = torch.tensor([1.0625, 1.1875, -2.125, 0.5 + 1 / 32, 3 * 2.0 ** -10, 2.0 ** -10, 13.0, -232.0])
    big = torch.randn(G, generator=torch.Generator().manual_seed(4)) * 1e37
    big[3] = 3.4e38 if dtype == torch.float32 else 3.38e38  # bf16 rounds 3.4e38 to inf
    tiny_normal = torch.zeros(G)
    tiny_normal[::3] = torch.linspace(2.0 ** -125, 400 * 2.0 ** -126, tiny_normal[::3].numel())
    tiny_inf_m = torch.zeros(G)
    tiny_inf_m[5::7] = torch.linspace(-1e-37, 1e-37, tiny_inf_m[5::7].numel())
    tiny_inf_m[5] = 1.2e-37
    inf = torch.randn(G, generator=torch.Generator().manual_seed(5))
    ninf, nan, naninf = inf.clone(), inf.clone(), inf.clone()
    inf[100] = math.inf
    ninf[200] = -math.inf
    nan[300] = math.nan
    naninf[10], naninf[11] = math.nan, math.inf
    over = torch.full((G,), 1.0)
    over[42] = 3.0e38
    groups = [("zeros", None, z), ("one", [0], one), ("pow448", [0], powg), ("midpoints", [0], mid),
              ("inf", [0], inf), ("-inf", [1], ninf), ("nan", [0], nan), ("nan+inf", [1], naninf)]
    if dtype == torch.float32:
        groups += [("tiny_normal", [0], tiny_normal), ("tiny_inf_m", [1], tiny_inf_m)]
    if dtype != torch.float16:
        groups += [("amax_flt_max", [0], big), ("overflow", None, over)]
    if dtype == torch.bfloat16:
        sub = torch.randn(G, generator=torch.Generator().manual_seed(6)) * 2.0 ** -130  # bf16 subnormals (FTZ: zeros)
        sub[0] = 2.0 ** -120
        groups.append(("bf16_subnormal", [0], sub))
    return groups


@pytest.mark.parametrize("dtype", DTYPES)
def test_edge_groups_exact_and_contract(dtype):
    """Every edge group once in the middle of one message (standalone quantise/dequantise and the fused all-reduce), then
    each alone in the partial tail group of a short message (fused all-reduce)."""
    from torchft_b200 import quantization as Q

    W, G = 3, E.GROUP
    groups = _edge_groups(dtype)
    comms = _world(W)

    def allreduce(ins):
        n = ins[0].numel()
        ad = _dev(ins)
        outs = [torch.empty(n, dtype=dtype, device=DEV) for _ in range(W)]
        _run(comms, lambda r, c, s: c.q8_allreduce_(outs[r], ad[r], None, scale=1.0 / W, stream=s))
        _ok(comms)
        want, _ = E.allreduce([E.load(x) for x in ins], 1.0 / W)
        _assert_bits(outs[0], E.cast(want, dtype), f"edge all-reduce {dtype} n={n}")
        assert all(E.equal_bits(o, outs[0]) for o in outs)
        return outs[0]

    ng = 2 * len(groups) + 1
    xs = _msg(ng * G, W, 3, torch.float32, _fp16_safe(dtype))
    for k, (name, ranks, vals) in enumerate(groups):
        _place(xs, 2 * k + 1, ranks, vals)
    ins = [x.to(dtype) for x in xs]
    buf = Q.quantize_q8(ins[0].to(DEV))
    want_q = E.quantize(E.load(ins[0]), ng)
    _assert_q8(E.Q8.from_bytes(buf, ng), want_q, f"edge quantize {dtype}")
    _assert_bits(Q.dequantize_q8(buf, ng * G, dtype), E.cast(E.dequant(want_q).reshape(-1), dtype), f"edge dequantize {dtype}")
    got = allreduce(ins)
    for k, (name, _, _) in enumerate(groups):
        _check_contract(name, ins, got, 2 * k + 1)
    tail = G - 200
    for name, ranks, vals in groups:
        xs = _msg(2 * G + tail, W, 4, torch.float32, _fp16_safe(dtype))
        _place(xs, 2, ranks, vals[:tail])
        ins = [x.to(dtype) for x in xs]
        _check_contract(name, ins, allreduce(ins), 2)


def _place(xs, g, ranks, vals):
    for r, x in enumerate(xs):
        x[g * E.GROUP: g * E.GROUP + vals.numel()] = vals if ranks is None or r in ranks else 0.0


def _check_contract(name, ins, got, g):
    lo, hi = g * E.GROUP, min(ins[0].numel(), (g + 1) * E.GROUP)
    parts = [E.load(x)[lo:hi] for x in ins]
    ref = sum(p.double() for p in parts)
    out = got[lo:hi].float().cpu()
    has_inf = any(p.isinf().any() for p in parts)
    overflow = bool((ref.abs() > torch.finfo(torch.float32).max).any())
    if has_inf or overflow:
        assert torch.isnan(out).all(), f"{name}: an inf or an fp32 overflow must make the whole group NaN"
        assert not torch.isfinite(ref.float()).all()  # as the unquantised sum is not finite
        return
    if name == "zeros":
        assert E.equal_bits(out, torch.zeros_like(out)), "an all-zero group stays exactly +0"
    nan = torch.stack([p.isnan() for p in parts]).any(0)
    assert torch.equal(torch.isnan(out), nan), f"{name}: NaN only where an input was NaN"
    amax = ref[~nan].abs().max().item() if (~nan).any() else 0.0
    if amax >= 2.0 ** -125:
        assert (out[~nan] != 0).any(), f"{name}: a finite nonzero group became 0"
