"""The NVLink data plane byte for byte: all-reduce (one-shot, two-shot, world-1 scale-copy; zero-copy and staged),
reduce-scatter, the push exchange behind all-gather / broadcast / all-to-all / all-to-all-v, and send/recv, at every
world size, dtype and op, against the numpy model in ``_collectives_ref`` (reductions) or the moved bytes themselves.

Harness rules:

* The ranks run concurrently (``virtual_world(presignal=False)`` driven by ``_run``): pre-signalled worlds do not
  reproduce in-place one-shot or staged two-shot results.
* Every all-reduce plan is forced with ``_force_plan`` and W x blocks stays <= 112, the cap ``virtual_world`` puts on
  ``_max_blocks``, so every CTA of every rank is resident at once: a latched timeout reported by ``_ok`` is then a
  finding, not noise. ``_threads`` varies over 128, 256 and 512.
* ``alltoallv_`` reads its round agreement back on the host, so its ranks are driven from one host thread each, on
  their own streams, in a world with a short timeout.
* Sentinels: every tensor sits at an offset inside a larger buffer (the symmetric segment for zero-copy, an ordinary
  allocation for staged) with random bytes before and after it that differ per rank (equal sentinels would survive an
  AVG or a MAX over themselves). After every collective every byte outside the tensor must be unchanged on every rank.
* Each rank's kernel module is wrapped in a recorder that forwards every call and notes the (kernel, dtype, W, op,
  algo) instance it launches, with the launcher's fall-back from in-place one-shot to two-shot past threads x 8
  vectors per CTA; the last test asserts that every instance ran (run the whole module).
"""

from __future__ import annotations

import threading

import numpy as np
import pytest
import torch

import _collectives_ref as R
from _collectives import DEV, _ok, _run, _world

pytestmark = pytest.mark.gpu

PAD = 64  # sentinel bytes on each side of a tensor (a stray 16-byte store lands inside them)
DTS = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}
CODE = {0: "f32", 1: "bf16", 2: "f16"}
RAW = {"f32": (torch.int32, np.int32), "bf16": (torch.int16, np.int16), "f16": (torch.int16, np.int16),
       "u8": (torch.uint8, np.uint8)}
THREADS = (128, 256, 512)
RAN = set()  # ("ar", dtype, W, op, algo) / ("copy", dtype) / ("rs", dtype, W, op)


class _Recorder:
    """Forwards every call to the kernel module and records the all-reduce / reduce-scatter instance it launches.
    With ``nvls`` set to a list, ``allreduce_nvls`` only appends its element count there and launches nothing."""

    def __init__(self, comm, K):
        self._comm, self._K, self.nvls = comm, K, None

    def __getattr__(self, name):
        return getattr(self._K, name)

    def allreduce(self, *a):
        user_out, n, dt, op, algo, blocks, threads = a[4], a[5], a[6], a[7], a[12], a[13], a[14]
        W = self._comm._world
        if W == 1:
            RAN.add(("copy", CODE[dt]))
        else:
            vecs = -(-n * (4 if dt == 0 else 2) // 16)
            if algo == 0 and user_out == 0 and -(-vecs // blocks) > threads * 8:
                algo = 1  # the in-place one-shot keeps its results in registers: allreduce.cu falls back
            RAN.add(("ar", CODE[dt], W, op, algo))
        return self._K.allreduce(*a)

    def reduce_scatter(self, *a):
        RAN.add(("rs", CODE[a[6]], self._comm._world, a[7]))
        return self._K.reduce_scatter(*a)

    def allreduce_nvls(self, *a):
        if self.nvls is None:
            return self._K.allreduce_nvls(*a)
        self.nvls.append(a[4])


def _comms(world, **kw):
    comms = _world(world, **kw)
    for c in comms:
        c._K = _Recorder(c, c._K)
    return comms


def _free(comms):
    for c in comms:
        c.shutdown()
    for c in comms:
        c.free_segments()


class _Placed:
    """``n`` elements of ``dt`` at byte offset ``PAD + skew`` of the uint8 buffer ``buf``, with random sentinel bytes
    (from ``rng``, so different per rank) in front of it and in the PAD bytes after it."""

    def __init__(self, buf, n, dt, rng, skew=0):
        es = 1 if dt == "u8" else np.dtype(R.BITS[dt]).itemsize
        self.dt, self.nb, self.lo = dt, n * es, PAD + skew
        self.region = buf[: self.lo + self.nb + PAD]
        assert self.region.numel() == self.lo + self.nb + PAD, "buffer too small"
        self.raw = self.region[self.lo: self.lo + self.nb].view(RAW[dt][0])
        self.t = self.raw if dt == "u8" else self.raw.view({"f32": torch.float32, "bf16": torch.bfloat16,
                                                            "f16": torch.float16}[dt])
        self.before = rng.integers(0, 256, self.lo, dtype=np.uint8)
        self.after = rng.integers(0, 256, PAD, dtype=np.uint8)

    def load(self, bits=None):
        self.region[: self.lo].copy_(torch.from_numpy(self.before))
        self.region[self.lo + self.nb:].copy_(torch.from_numpy(self.after))
        if bits is not None:
            self.raw.copy_(torch.from_numpy(np.ascontiguousarray(bits).view(RAW[self.dt][1])))

    def bits(self):
        return self.raw.cpu().numpy().view(np.uint8 if self.dt == "u8" else R.BITS[self.dt])

    def check_sentinels(self, what):
        got = self.region.cpu().numpy()
        for name, want, have in (("before", self.before, got[: self.lo]), ("after", self.after, got[self.lo + self.nb:])):
            bad = np.flatnonzero(want != have)
            assert bad.size == 0, f"{what}: {bad.size} sentinel bytes {name} the tensor changed (first at {bad[0]})"


def _check(places, want, dt, op, what):
    first = places[0].bits()
    for r, p in enumerate(places):
        got = p.bits()
        err = R.mismatch(got, want, dt, op)
        assert err is None, f"{what} rank {r}: {err}"
        assert np.array_equal(got, first), f"{what}: rank {r} differs from rank 0"
        p.check_sentinels(f"{what} rank {r}")
    return first


def _staged_bufs(world, nbytes):
    return [torch.empty(nbytes + 2 * PAD + 16, dtype=torch.uint8, device=DEV) for _ in range(world)]


# ----------------------------------------------------------------------------------------------------------- all-reduce
def _allreduce_lengths(W, N, bmax):
    """(elements, (blocks, threads) or None) at the edges of the decomposition; None lets the test pick the grid."""
    lim = 3 * 128 * 8  # vectors the in-place one-shot holds in registers at 3 CTAs of 128 threads
    return [
        (0, None), (1, None), (N - 1, None), (N, None), (N + 1, None), (5, None),
        (W * N - 1, None), (W * N, None), (W * N + 1, None),
        (2 * N + 1, None), ((W + 1) * N + 3, None),          # slices past the first few are empty
        (W * N * (3 * bmax + 1) + 3, (bmax, 512)),            # a slice that does not divide by the grid
        (lim * N, (3, 128)), (lim * N + 1, (3, 128)), (lim * N + N, (3, 128)),  # register limit, and one vector past
        (4096, None), (70_000, None), (100_003, None), (1 << 19, None),
    ]


@pytest.mark.parametrize("dtype", list(DTS), ids=list(DTS.values()))
@pytest.mark.parametrize("world", range(1, 9))
def test_allreduce_exact(world, dtype):
    W, dt = world, DTS[dtype]
    comms = _comms(W)
    N = 16 // dtype.itemsize
    bmax = comms[0]._max_blocks
    rng = np.random.default_rng(1000 * W + dtype.itemsize)
    lengths = _allreduce_lengths(W, N, bmax)
    nmax = max(n for n, _ in lengths)
    staged = _staged_bufs(W, nmax * dtype.itemsize)
    scales = (1.0, 1.0 / W, 0.5)
    for i, (n, plan) in enumerate(lengths):
        blocks, threads = plan if plan is not None else ((1, 3, bmax)[i % 3], THREADS[(i // 3) % 3])
        ins = [R.values(rng, n, dt) for _ in range(W)]
        zc = [_Placed(c.segment("buf"), n, dt, rng) for c in comms]
        st = [_Placed(b, n, dt, rng) for b in staged]
        for op in (R.SUM, R.MAX, R.MIN):
            k = i + op
            scale = scales[k % 3]
            quiet = [(), (k % W,), tuple(r for r in range(W) if r != k % W)][(k // 3) % 3] if W > 1 else [(), (0,)][k % 2]
            if W == 1:
                want = ins[0] if (scale == 1.0 and not quiet) else R.scale_copy(ins[0], dt, scale, not quiet)
                paths = [("zero-copy", zc, None), ("staged", st, None)]
            else:
                want = R.allreduce([None if r in quiet else x for r, x in enumerate(ins)], dt, op, scale)
                paths = [(f"{where} {'one' if algo == 0 else 'two'}-shot", places, (algo, blocks))
                         for where, places in (("zero-copy", zc), ("staged", st)) for algo in (0, 1)]
            first = None
            for name, places, force in paths:
                for p, x in zip(places, ins):
                    p.load(x)

                def fn(r, c, s, places=places, force=force):
                    c._force_plan, c._threads = force, threads
                    c.allreduce_(places[r].t, op=op, scale=scale, contribute=r not in quiet, stream=s)
                    c._force_plan, c._threads = None, 512

                _run(comms, fn)
                _ok(comms)
                what = f"W={W} {dt} n={n} op={op} scale={scale:g} quiet={quiet} {name} grid={blocks}x{threads}"
                got = _check(places, want, dt, op, what)
                assert first is None or np.array_equal(got, first), f"{what}: differs from the first path"
                first = got
    _free(comms)


@pytest.mark.parametrize("dtype", list(DTS), ids=list(DTS.values()))
@pytest.mark.parametrize("world", [2, 5, 8])
def test_allreduce_staged_message_larger_than_staging(world, dtype):
    """2.5x the usable staging of a 2 MiB staging world: one launch per staging-sized piece, every piece exact."""
    W, dt = world, DTS[dtype]
    comms = _comms(W, staging=2 << 20)
    per = comms[0]._staging_usable // dtype.itemsize
    n = per * 5 // 2
    rng = np.random.default_rng(W)
    ins = [R.values(rng, n, dt) for _ in range(W)]
    places = [_Placed(b, n, dt, rng) for b in _staged_bufs(W, n * dtype.itemsize)]
    for op, scale, quiet, force in ((R.SUM, 1.0 / W, (1,), (1, 8)), (R.MAX, 1.0, (), (0, 8)), (R.MIN, 0.5, (0,), (1, 3))):
        for p, x in zip(places, ins):
            p.load(x)
        before = [c.launches for c in comms]

        def fn(r, c, s):
            c._force_plan = force
            c.allreduce_(places[r].t, op=op, scale=scale, contribute=r not in quiet, stream=s)
            c._force_plan = None

        _run(comms, fn)
        _ok(comms)
        assert [c.launches - b for c, b in zip(comms, before)] == [3] * W
        want = R.allreduce([None if r in quiet else x for r, x in enumerate(ins)], dt, op, scale)
        _check(places, want, dt, op, f"W={W} {dt} n={n} op={op} plan={force}")
    _free(comms)


def test_allreduce_llama3_1b_block_two_shot_zero_copy():
    """One llama3_1b block of bf16 gradients (60 821 504 elements) at W = 8, zero-copy two-shot: normal-range values,
    so the reference is the rank-order fp32 sum on the device, scaled, rounded once."""
    W, n = 8, 60_821_504
    comms = _comms(W, segs={"buf": n * 2 + 4 * PAD})
    g = torch.Generator(device=DEV).manual_seed(8)
    xs = [torch.randn(n, device=DEV, generator=g).bfloat16() for _ in range(W)]
    rng = np.random.default_rng(8)
    places = [_Placed(c.segment("buf"), n, "bf16", rng) for c in comms]
    for p, x in zip(places, xs):
        p.load()
        p.t.copy_(x)
    acc = xs[0].float()
    for x in xs[1:]:
        acc += x.float()
    want = (acc * (1.0 / W)).bfloat16()
    del acc

    def fn(r, c, s):
        c._force_plan = (1, c._max_blocks)
        c.allreduce_(places[r].t, scale=1.0 / W, stream=s)
        c._force_plan = None

    _run(comms, fn)
    _ok(comms)
    for r, p in enumerate(places):
        assert torch.equal(p.t.view(torch.int16), want.view(torch.int16)), f"rank {r}"
        p.check_sentinels(f"rank {r}")
    del xs, want
    _free(comms)


def test_nvls_routing_keeps_tail_lengths_on_the_p2p_kernels():
    """NVLS cannot run in a one-GPU world: a fake multicast entry and a recorder that launches nothing show where
    ``allreduce_`` routes. An aligned message of >= 256 KiB goes to NVLS; one that ends inside a 16-byte vector goes to
    the P2P kernels (multimem stores write whole vectors) and is exact with its sentinels intact."""
    W = 5
    comms = _comms(W)
    calls = []
    rng = np.random.default_rng(5)
    try:
        for c in comms:
            c._mc["buf"] = (0, 1 << 40, c._segments["buf"].nbytes)
            c._K.nvls = calls
        assert comms[0]._nvls_min == 256 << 10
        for n, to_nvls in ((128 << 10, True), ((128 << 10) + 1, False), ((128 << 10) + 13, False)):
            ins = [R.values(rng, n, "bf16") for _ in range(W)]
            places = [_Placed(c.segment("buf"), n, "bf16", rng) for c in comms]
            for p, x in zip(places, ins):
                p.load(x)
            del calls[:]
            _run(comms, lambda r, c, s: c.allreduce_(places[r].t, scale=1.0 / W, stream=s))
            _ok(comms)
            if to_nvls:
                assert calls == [n] * W
                for p, x in zip(places, ins):
                    assert np.array_equal(p.bits(), x)  # nothing was launched
                    p.check_sentinels(f"n={n}")
            else:
                assert calls == []
                _check(places, R.allreduce(ins, "bf16", R.SUM, 1.0 / W), "bf16", R.SUM, f"n={n}")
    finally:
        for c in comms:
            c._mc.pop("buf", None)
            c._K.nvls = None
    _free(comms)


# ------------------------------------------------------------------------------------------------------- reduce-scatter
@pytest.mark.parametrize("dtype", list(DTS), ids=list(DTS.values()))
@pytest.mark.parametrize("world", range(2, 9))
def test_reduce_scatter_exact(world, dtype):
    W, dt, es = world, DTS[dtype], dtype.itemsize
    N = 16 // es
    comms = _comms(W, segs={"buf": 8 << 20})
    small = _comms(W, staging=2 << 20)
    rng = np.random.default_rng(2000 * W + es)
    bmax = comms[0]._max_blocks
    per = (small[0]._staging_usable // (W * es)) // 8 * 8  # elements of one staging round of ``small``
    # (n, grid override or None, world): vector path (n*es % 16 == 0) and scalar path, CTAs with nothing to do,
    # and a staged message of three rounds
    cases = [(1, None, comms), (N - 1, None, comms), (N, None, comms), (N + 1, None, comms), (3 * N, bmax, comms),
             (bmax * N - N, bmax, comms), (8, None, comms), (1001, None, comms), (4104, None, comms),
             (65_536, None, comms), (65_536 + 3, None, comms), (2 * per + N + 1, None, small), (2 * per + 8 * N, None, small)]
    scales = (1.0, 1.0 / W, 0.25)
    for i, (n, grid, cs) in enumerate(cases):
        ins = [R.values(rng, W * n, dt) for _ in range(W)]
        out_bufs = _staged_bufs(W, n * es + 16)
        in_bufs = _staged_bufs(W, W * n * es)
        for op in (R.SUM, R.MAX, R.MIN):
            scale = scales[(i + op) % 3]
            want = [R.allreduce([x[r * n:(r + 1) * n] for x in ins], dt, op, scale) for r in range(W)]
            wheres = ("staged",) if cs is small else ("zero-copy", "staged")
            for where in wheres:
                for skew in (0, es):  # an ``out`` off 16-byte alignment takes the scalar path
                    src = [_Placed(c.segment("buf") if where == "zero-copy" else b, W * n, dt, rng)
                           for c, b in zip(cs, in_bufs)]
                    outs = [_Placed(b, n, dt, rng, skew) for b in out_bufs]
                    for p, x in zip(src, ins):
                        p.load(x)
                    for p in outs:
                        p.load(np.zeros(n, R.BITS[dt]))

                    def fn(r, c, s, src=src, outs=outs):
                        if grid is not None:
                            c._xblocks = lambda nbytes: grid
                        c.reduce_scatter_(outs[r].t, src[r].t, op=op, scale=scale, stream=s)
                        c.__dict__.pop("_xblocks", None)

                    _run(cs, fn)
                    _ok(cs)
                    what = f"W={W} {dt} n={n} op={op} scale={scale:g} {where} skew={skew} grid={grid}"
                    for r in range(W):
                        err = R.mismatch(outs[r].bits(), want[r], dt, op)
                        assert err is None, f"{what} rank {r}: {err}"
                        outs[r].check_sentinels(f"{what} out rank {r}")
                        src[r].check_sentinels(f"{what} in rank {r}")
                        assert np.array_equal(src[r].bits(), ins[r]), f"{what}: input of rank {r} changed"
    _free(comms)
    _free(small)


# -------------------------------------------------------------------------------------------------------- push exchange
def _bytes(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8)


@pytest.mark.parametrize("world", range(2, 9))
def test_allgather_broadcast_alltoall_exact(world):
    W = world
    comms = _comms(W, staging=2 << 20)
    stride = comms[0]._slot_stride()
    rng = np.random.default_rng(3000 + W)
    lengths = [0, 1, 15, 16, 17, stride - 1, stride, 2 * stride + 17]
    big = _staged_bufs(W, W * max(lengths) + 32)
    small = _staged_bufs(W, max(lengths) + 32)
    for i, L in enumerate(lengths):
        a, b = (7 * i + 1) % 16, (5 * i + 3) % 16  # input and output 1..15 bytes off alignment (0 once)
        xs = [_bytes(rng, L) for _ in range(W)]
        what = f"W={W} L={L} skews={a},{b}"
        # all-gather out of place
        outs = [_Placed(buf, W * L, "u8", rng, b) for buf in big]
        ins = [_Placed(buf, L, "u8", rng, a) for buf in small]
        for o, p, x in zip(outs, ins, xs):
            o.load()
            p.load(x)
        _run(comms, lambda r, c, s: c.allgather_(outs[r].t, ins[r].t, stream=s))
        _ok(comms)
        for r in range(W):
            assert np.array_equal(outs[r].bits(), np.concatenate(xs)), f"all-gather {what} rank {r}"
            outs[r].check_sentinels(f"all-gather {what} rank {r}")
            assert np.array_equal(ins[r].bits(), xs[r])
            ins[r].check_sentinels(f"all-gather input {what} rank {r}")
        # all-gather in place: the input is this rank's piece of the output
        for r, o in enumerate(outs):
            o.load(np.concatenate([xs[p] if p == r else _bytes(rng, L) for p in range(W)]))
        _run(comms, lambda r, c, s: c.allgather_(outs[r].t, outs[r].t[r * L:(r + 1) * L], stream=s))
        _ok(comms)
        for r in range(W):
            assert np.array_equal(outs[r].bits(), np.concatenate(xs)), f"in-place all-gather {what} rank {r}"
            outs[r].check_sentinels(f"in-place all-gather {what} rank {r}")
        # broadcast from every root, in place
        for root in range(W):
            ts = [_Placed(buf, L, "u8", rng, b) for buf in small]
            for t, x in zip(ts, xs):
                t.load(x)
            _run(comms, lambda r, c, s: c.broadcast_(ts[r].t, root, stream=s))
            _ok(comms)
            for r in range(W):
                assert np.array_equal(ts[r].bits(), xs[root]), f"broadcast {what} root {root} rank {r}"
                ts[r].check_sentinels(f"broadcast {what} root {root} rank {r}")
        # equal all-to-all: chunk p of rank r's input becomes chunk r of rank p's output
        chunks = [[_bytes(rng, L) for _ in range(W)] for _ in range(W)]
        ins = [_Placed(buf, W * L, "u8", rng, a) for buf in _staged_bufs(W, W * L + 32)]
        for p, ch in zip(ins, chunks):
            p.load(np.concatenate(ch))
        for o in outs:
            o.load()
        _run(comms, lambda r, c, s: c.alltoall_(outs[r].t, ins[r].t, stream=s))
        _ok(comms)
        for r in range(W):
            assert np.array_equal(outs[r].bits(), np.concatenate([chunks[p][r] for p in range(W)])), f"all-to-all {what} rank {r}"
            outs[r].check_sentinels(f"all-to-all {what} rank {r}")
    _free(comms)


def _threaded(comms, fn):
    """One host thread per rank, each on its own stream: for collectives that synchronise with the host mid-way."""
    streams = [torch.cuda.Stream(device=DEV) for _ in comms]
    errors = [None] * len(comms)

    def body(r):
        try:
            with torch.cuda.stream(streams[r]):
                fn(r, comms[r], streams[r])
            streams[r].synchronize()
        except BaseException as e:  # noqa: BLE001 -- re-raised on the main thread
            errors[r] = e

    torch.cuda.synchronize()
    threads = [threading.Thread(target=body, args=(r,)) for r in range(len(comms))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errors:
        if e is not None:
            raise e


def test_alltoallv_skewed_splits_agree_on_one_grid():
    """Ragged splits with zeros, a dominant self-send on rank 0 (three staging rounds; a few bytes to each peer), a rank
    that receives far more than it sends, and pairs that need different numbers of rounds. Every push-exchange CTA meets
    the same CTA of every peer only if every rank launches the same grid."""
    W = 4
    comms = _comms(W, staging=2 << 20, timeout=5.0)
    S = [[1 << 20, 3, 0, 17],              # S[p][q]: bytes rank p sends to rank q
         [5, 0, 1, 16],
         [0, 250_000, 70_001, 15],
         [17, 450_000, 0, 131_072]]
    rng = np.random.default_rng(44)
    data = [[_bytes(rng, S[p][q]) for q in range(W)] for p in range(W)]
    ins = [_Placed(b, sum(S[r]), "u8", rng, 5) for r, b in enumerate(_staged_bufs(W, max(map(sum, S)) + 16))]
    outs = [_Placed(b, sum(S[p][r] for p in range(W)), "u8", rng, 3)
            for r, b in enumerate(_staged_bufs(W, max(sum(S[p][r] for p in range(W)) for r in range(W)) + 16))]
    for r in range(W):
        ins[r].load(np.concatenate(data[r]))
        outs[r].load()
    _threaded(comms, lambda r, c, s: c.alltoallv_(outs[r].t, ins[r].t, [S[p][r] for p in range(W)], S[r], stream=s))
    _ok(comms)
    for r in range(W):
        assert np.array_equal(outs[r].bits(), np.concatenate([data[p][r] for p in range(W)])), f"rank {r}"
        outs[r].check_sentinels(f"rank {r}")
    _free(comms)


def test_alltoallv_in_one_rank_world_copies_its_own_split():
    comms = _comms(1)
    rng = np.random.default_rng(1)
    x = _bytes(rng, 1001)
    src = _Placed(_staged_bufs(1, 1024)[0], 1001, "u8", rng, 1)
    dst = _Placed(_staged_bufs(1, 1024)[0], 1001, "u8", rng, 7)
    src.load(x)
    dst.load()
    _run(comms, lambda r, c, s: c.alltoallv_(dst.t, src.t, [1001], [1001], stream=s))
    _ok(comms)
    assert np.array_equal(dst.bits(), x)
    dst.check_sentinels("world 1")
    _free(comms)


# ------------------------------------------------------------------------------------------------------------ send/recv
def test_send_recv_every_pair_unaligned_back_to_back():
    W = 4
    comms = _comms(W, staging=2 << 20)
    mb = comms[0]._mailbox_bytes
    rng = np.random.default_rng(4)
    sizes = [1, mb - 1, mb, mb + 1, 3 * mb + 5]
    bufs = _staged_bufs(3, 3 * mb + 64)
    for s_, d in [(s_, d) for s_ in range(W) for d in range(W) if s_ != d]:
        for i, L in enumerate(sizes):
            L2 = sizes[(i + 2) % len(sizes)]
            m1, m2 = _bytes(rng, L), _bytes(rng, L2)
            a = _Placed(bufs[0], L, "u8", rng, (i + s_) % 16)
            b = _Placed(bufs[1], L, "u8", rng, (3 * i + d + 1) % 16)
            b2 = _Placed(bufs[2], L2, "u8", rng, (5 * i + 2) % 16)
            a.load(m1)
            b.load()
            b2.load()
            src2 = torch.from_numpy(m2).to(DEV)

            def fn(r, c, s):  # two messages back to back on each side: FIFO per ordered pair
                if r == s_:
                    c.send_(a.t, d, s)
                    c.send_(src2, d, s)
                else:
                    c.recv_(b.t, s_, s)
                    c.recv_(b2.t, s_, s)

            _run(comms, fn, ranks=(s_, d))
            _ok(comms)
            what = f"{s_}->{d} L={L},{L2}"
            assert np.array_equal(b.bits(), m1) and np.array_equal(b2.bits(), m2), what
            assert np.array_equal(a.bits(), m1), what
            for p in (a, b, b2):
                p.check_sentinels(what)
    _free(comms)


# ------------------------------------------------------------------------------------------------------------ coverage
def test_every_kernel_instance_ran():
    """Every all-reduce and reduce-scatter instance the launchers can pick without multicast ran above (run the whole
    module): 3 dtypes x 3 ops x W 2..8 x {one-shot, two-shot} plus the world-1 scale-copy per dtype, and 3 dtypes x 3
    ops x W 2..8 reduce-scatters."""
    want = {("ar", d, w, op, a) for d in R.DTYPES for w in range(2, 9) for op in (R.SUM, R.MAX, R.MIN) for a in (0, 1)}
    want |= {("copy", d) for d in R.DTYPES}
    want |= {("rs", d, w, op) for d in R.DTYPES for w in range(2, 9) for op in (R.SUM, R.MAX, R.MIN)}
    missing = sorted(want - RAN, key=str)
    assert not missing, f"never launched: {missing}"
