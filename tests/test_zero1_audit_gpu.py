"""FT-ZeRO-1 replica audit on the GPU: the digest kernel bit for bit against the numpy specification, and the audit of
FT-ZeRO-1 replicas that signal each other for real (one stream per rank), through detection, localisation and repair.

The pre-signalled virtual world of the other FT-ZeRO-1 tests runs one rank at a time, so a compare would read peers'
slots before their digests exist; every audit here runs with real signalling."""

from __future__ import annotations

import threading
from datetime import timedelta

import pytest
import torch

from _zero1_replicas import HP, NUMEL, PG, SHIFT, UNITS, raws, seeded_weights

pytestmark = pytest.mark.gpu

CW = 8192  # Z1_DIGEST_CHUNK_WORDS


def K():
    from torchft_b200.ops import _native

    return _native.load()


def host_bytes(t):
    return t.contiguous().view(torch.uint8).cpu().numpy()


def digest_rows(rows):
    """Table rows ``(base, table, page_byte_shift, word0, nwords, seed, slot)`` with their chunk0; total chunks."""
    out, c = [], 0
    for r in rows:
        out.append(tuple(r) + (c,))
        c += (r[4] + CW - 1) // CW
    return torch.tensor(out, dtype=torch.int64, device="cuda"), len(out), c


def run_digest(rows, nslots, grid):
    slots = torch.zeros(nslots, dtype=torch.int64, device="cuda")
    tab, n, chunks = digest_rows(rows)
    K().z1_digest(tab.data_ptr(), n, chunks, slots.data_ptr(), grid, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return [int(x) & ((1 << 64) - 1) for x in slots.cpu().tolist()]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("grid", [1, 3, 132, 1024])
def test_digest_kernel_matches_numpy_flat(dtype, grid):
    from torchft_b200.parallel.zero1 import AUDIT_SEEDS, z1_digest

    es = torch.tensor([], dtype=dtype).element_size()
    g = torch.Generator(device="cuda").manual_seed(grid)
    n_el = (3 * CW + 40) * 8 // es  # the longest row ends at word 3 CW + 19
    x = torch.randn(n_el, device="cuda", generator=g).to(dtype)
    xb = host_bytes(x)
    rows, want = [], []
    lengths = [1, 2, 3, 4, CW - 1, CW, CW + 1, 2 * CW + 2, 3 * CW + 3]  # words: around a word, a vector and a chunk
    for slot, nw in enumerate(lengths):
        word0 = 2 * slot  # even: the range starts on a 16-byte vector
        seed = list(AUDIT_SEEDS.values())[slot % 5]
        rows.append((x.data_ptr(), 0, 0, word0, nw, seed, slot))
        want.append(z1_digest(xb[8 * word0:8 * (word0 + nw)], word0, seed))
    assert run_digest(rows, len(rows), grid) == want


@pytest.mark.parametrize("shuffled", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_digest_kernel_paged_equals_flat(shuffled, dtype):
    """The same global range digested from a flat array and from a page pool (slots in order or permuted)."""
    from torchft_b200.parallel.zero1 import AUDIT_SEEDS, z1_digest

    es = torch.tensor([], dtype=dtype).element_size()
    page = 1 << SHIFT
    npages = 200
    g = torch.Generator(device="cuda").manual_seed(7)
    flat = torch.randn(npages * page, device="cuda", generator=g).to(dtype)
    perm = torch.randperm(npages, generator=torch.Generator().manual_seed(1)) if shuffled else torch.arange(npages)
    table = perm.to(torch.int32).cuda()
    pool = torch.empty_like(flat)
    pool.view(npages, page)[perm.cuda()] = flat.view(npages, page)
    pbs = SHIFT + es.bit_length() - 1
    seed = AUDIT_SEEDS["m"]
    ranges = [(8, 16), (page - 8, page + 8), (3 * page + 16, 150 * page - 8), (0, npages * page)]  # elements
    rows, want = [], []
    fb = host_bytes(flat)
    for i, (lo, hi) in enumerate(ranges):
        w0, nw = lo * es // 8, (hi - lo) * es // 8
        rows.append((pool.data_ptr(), table.data_ptr(), pbs, w0, nw, seed, 2 * i))
        rows.append((flat.data_ptr(), 0, 0, w0, nw, seed, 2 * i + 1))
        want.append(z1_digest(fb[lo * es:hi * es], w0, seed))
    for grid in (1, 132):
        got = run_digest(rows, 2 * len(ranges), grid)
        assert got[0::2] == want and got[1::2] == want


@pytest.mark.parametrize("compact", [False, True])
def test_every_kernel_instance_ran(compact):
    """One real-signalling audit runs both kernels: every slot of the report is numpy's digest of that rank's weights or
    held state (so the digest kernel ran over every row and the compare kernel copied every rank's slots), and the
    update count is there. A digest that did nothing would leave zeros, which no digest here equals."""
    from torchft_b200.parallel.zero1 import AUDIT_SEEDS, z1_digest

    world, k = 3, 2
    w = World(world, k=k, audit_every=1, compact=compact)
    w.step(raws(world, 1)[0])
    w.settle()
    assert all(o.audits == 1 for o in w.opts) and all(c.errored() is None for c in w.comms)
    for o in w.opts:
        rep = o.audit_report()
        assert rep["mismatches"] == 0 and rep["world"] == world and rep["t"] == [1] * world
        for r in range(world):
            x = w.opts[r]
            arrays = x._state_arrays()
            for u, (lo, hi) in enumerate(UNITS):
                want = z1_digest(host_bytes(x.param[lo:hi]), lo // 4, AUDIT_SEEDS["weights"])
                assert rep["weights"][r][u] == want != 0
                for j in range(k):
                    a, b = x.layout.slice_bounds(u, world, (r - j) % world)
                    for i, (name, arr) in enumerate(arrays):
                        if b == a:  # an empty slice leaves its slot at 0
                            assert rep["state"][r][u][j][i] == 0
                            continue
                        data = torch.cat([arr[at:at + d - c] for c, d, at in x._pieces(x._table_host, a, b)])
                        want = z1_digest(host_bytes(data), a * arr.element_size() // 8, AUDIT_SEEDS[name])
                        assert rep["state"][r][u][j][i] == want, (r, u, j, name)


# --------------------------------------------------------------------------- replicas with real signalling
class World:
    """``n`` FT-ZeRO-1 replicas in one process on one GPU that signal each other for real: each rank runs on its own
    stream, and every rank's step is enqueued before anything is waited for."""

    def __init__(self, n, k=2, blocks=4, init=None, **options):
        from torch.distributed import HashStore

        from torchft_b200.parallel.symm_mem import SymmetricComm
        from torchft_b200.parallel.zero1 import GNORM_UNITS, ShardLayout, Zero1Optimizer, audit_stride, pool_pages

        self.n, self.k = n, k
        opts = {"lr": HP[0], "betas": HP[1:3], "eps": HP[3], "weight_decay": HP[4], "page_shift": SHIFT, **options}
        n_state = NUMEL
        if opts.get("compact"):
            n_state = pool_pages(ShardLayout(tuple(UNITS), k), opts.get("min_world", 1), 1 << SHIFT) << SHIFT
        seg = {"z1_grad": NUMEL * 2, "z1_param": NUMEL * 2, "z1_gnorm": GNORM_UNITS * 8,
               "z1_audit": (GNORM_UNITS * audit_stride(k) + 1) * 8,
               **{x: n_state * 4 for x in ("z1_master", "z1_m", "z1_v", "z1_ema")}}
        self.comms = SymmetricComm.virtual_world(n, seg, presignal=False, timeout=timedelta(seconds=20))
        self.streams = [torch.cuda.Stream() for _ in range(n)]
        self.opts = []
        init = seeded_weights(NUMEL) if init is None else init
        for c, s in zip(self.comms, self.streams):
            with torch.cuda.stream(s):
                o = Zero1Optimizer(PG(c), NUMEL, units=UNITS, replication=k, blocks=blocks, **opts)
            o.param.copy_(init)
            o.seed_master()
            self.opts.append(o)
        torch.cuda.synchronize()
        self.store = HashStore()
        self.epoch = 1
        self.pending = None
        self.configure(first=True)

    def configure(self, first=False):
        """A quorum change with the same members: fresh flags, cleared status, every rank's re-shard on its own thread."""
        from torch.distributed import PrefixStore

        self.settle()
        torch.cuda.synchronize()
        if not first:
            self.epoch += 1
            for r, c in enumerate(self.comms):
                c._status.clear()
                c._install({name: [cc._segments[name].ptr for cc in self.comms] for name in c._segments}, r, self.n,
                           self.epoch, floor=0)
        errs = {}

        def run(r):
            try:
                self.opts[r]._on_configured(PrefixStore(f"q/{self.epoch}", self.store), r, self.n, self.epoch)
            except Exception as e:  # noqa: BLE001
                errs[r] = e

        ts = [threading.Thread(target=run, args=(r,)) for r in range(self.n)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        torch.cuda.synchronize()
        assert not errs, errs

    def settle(self):
        if self.pending is not None:
            for r, seq in self.pending.items():
                self.opts[r].resolved(self.opts[r].wait(seq))
            self.pending = None

    def step(self, raw, veto=()):
        self.settle()
        torch.cuda.synchronize()  # the gradients were made on another stream
        self.pending = {}
        for r, (o, s) in enumerate(zip(self.opts, self.streams)):
            with torch.cuda.stream(s):
                o.grad.copy_(raw[r])
                for u in range(len(UNITS)):
                    o.reduce_scatter(u, 1.0 / self.n, True)
                self.pending[r] = o.enqueue(r not in veto)
                o.update()
        torch.cuda.synchronize()

    def verdicts(self):
        return [self.opts[r].comm.verdict(s) for r, s in self.pending.items()]

    def errors(self):
        return [None if c.errored() is None else c._status.error() for c in self.comms]

    def held(self, r, name):
        """Rank ``r``'s array ``name`` over each range it holds, as bytes keyed by range."""
        o = self.opts[r]
        x = dict(o._state_arrays())[name]
        return {(lo, hi): torch.cat([x[at:at + b - a] for a, b, at in o._pieces(o._table_host, lo, hi)]).view(torch.uint8)
                for lo, hi in o.layout.held(r, self.n)}

    def state_equal(self, other):
        for r in range(self.n):
            assert torch.equal(self.opts[r].param.view(torch.int16), other.opts[r].param.view(torch.int16)), r
            for name, _ in self.opts[r]._state_arrays():
                a, b = self.held(r, name), other.held(r, name)
                assert a.keys() == b.keys()
                for key in a:
                    assert torch.equal(a[key], b[key]), (r, name, key)

    def replicas_agree(self):
        for r in range(1, self.n):
            assert torch.equal(self.opts[0].param.view(torch.int16), self.opts[r].param.view(torch.int16)), r


def flip(x, e, bit=0):
    """Flip bit ``bit`` of element ``e`` of tensor ``x`` (a data write, nothing else). A flip that must survive a
    committed update takes a high mantissa bit: the lowest one can vanish when the update rounds."""
    v = x.view(torch.int16 if x.element_size() == 2 else torch.int32)
    v[e] ^= 1 << bit
    torch.cuda.synchronize()


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_clean_audits_do_not_latch(world):
    w = World(world, k=min(3, world), audit_every=1)
    g = raws(world, 3, scales=(1.0, 0.5, 2.0))
    for raw in g:
        w.step([x for x in raw])
        assert all(w.verdicts())
    w.settle()
    assert w.errors() == [None] * world
    for o in w.opts:
        rep = o.audit_report()
        assert o.audits == 3 and o.divergences == 0 and rep["mismatches"] == 0 and rep["t"] == [3] * world


OPTION_SETS = {
    "flat": {},
    "paged": {"compact": True},
    "bf16": {"moment_dtype": torch.bfloat16},
    "ema_clip": {"ema_decay": 0.9, "max_grad_norm": 1.0},
    "paged_bf16_ema_accum": {"compact": True, "moment_dtype": torch.bfloat16, "ema_decay": 0.99, "grad_accum_steps": 2},
}


@pytest.mark.parametrize("name", sorted(OPTION_SETS))
def test_audit_changes_no_byte(name):
    opts = OPTION_SETS[name]
    M = opts.get("grad_accum_steps", 1)
    world = 3
    runs = [World(world, k=2, audit_every=a, **opts) for a in (0, 1)]
    steps = raws(world, 5, scales=(1.0,) * (3 * M))
    for w in runs:
        for i in range(3):
            micro = steps[i * M:(i + 1) * M]
            if M == 1:
                w.step(micro[0])
            else:
                step_accum(w, micro)
        w.settle()
    runs[0].state_equal(runs[1])
    assert runs[1].errors() == [None] * world and all(o.audits == 3 for o in runs[1].opts)


def step_accum(w, micro):
    w.settle()
    torch.cuda.synchronize()
    w.pending = {}
    for r, (o, s) in enumerate(zip(w.opts, w.streams)):
        with torch.cuda.stream(s):
            for m, raw in enumerate(micro):
                o.grad.copy_(raw[r])
                for u in range(len(UNITS)):
                    o.reduce_scatter(u, 1.0 / w.n, True, m)
                # the next micro-batch's copy follows the trailing handshakes on this stream: the peers are done reading
            w.pending[r] = o.enqueue(True)
            o.update()
    torch.cuda.synchronize()


def localised(w, unit, array, s, rank):
    """Every rank latched the divergence, and its report names exactly (unit, array, slice) and ``rank``."""
    from torchft_b200.parallel.zero1 import audit_findings

    assert all(e is not None and e[0] == 3 for e in w.errors()), w.errors()
    reps = [o.audit_report() for o in w.opts]
    assert all(r["seq"] == reps[0]["seq"] and r["mismatches"] > 0 for r in reps)
    findings, _ = audit_findings(reps[0], w.opts[0].layout, w.n)
    hits = [f for f in findings if f["unit"] == unit and f["array"] == array and f["slice"] == s]
    assert hits and rank in hits[0]["ranks"], findings


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("where", ["primary_first", "buddy_last"])
@pytest.mark.parametrize("array", ["master", "m", "v", "ema"])
def test_flipped_bit_is_detected_and_localised(world, where, array):
    """A bit flipped in one holder's state between steps: the state digest of the next (vetoed, so nothing moves)
    step's audit differs on that holder."""
    w = World(world, k=2, audit_every=1, ema_decay=0.9)
    steps = raws(world, 9, scales=(1.0, 1.0))
    w.step(steps[0])
    w.settle()
    L = w.opts[0].layout
    unit, s = 1, world - 1
    lo, hi = L.slice_bounds(unit, world, s)
    j = 0 if where == "primary_first" else 1
    rank = (s + j) % world
    e = lo if where == "primary_first" else hi - 1
    o = w.opts[rank]
    x = dict(o._state_arrays())[array]
    flip(x, o._pieces(o._table_host, e, e + 1)[0][2])
    w.step(steps[1], veto=(0,))  # vetoed on every rank: the update moves nothing, the audit sees the flip
    assert w.verdicts() == [False] * world
    localised(w, unit, array, s, rank)
    assert w.errors()[0][1] == min(s, (s + 1) % world)  # the lowest rank of the group that disagrees


def test_weights_flip_is_repaired_by_the_next_quorum():
    world = 4
    w, twin = World(world, k=2, audit_every=1), World(world, k=2)
    steps = raws(world, 11, scales=(1.0, 1.0, 1.0))
    for x in (w, twin):
        x.step(steps[0])
        x.settle()
    e = UNITS[0][0] + 100
    flip(w.opts[2].param, e)
    for x in (w, twin):
        x.step(steps[1], veto=(0,))
    rep = w.opts[1].audit_report()
    from torchft_b200.parallel.zero1 import audit_findings

    findings, drops = audit_findings(rep, w.opts[1].layout, world)
    assert findings == [{"unit": 0, "array": "weights", "slice": None, "ranks": [2], "t": 1}]
    assert all(not d for d in drops.values())
    for x in (w, twin):
        x.configure()
        x.step(steps[2])
        x.settle()
    assert w.errors() == [None] * world and all(o.divergences == 1 for o in w.opts)
    w.replicas_agree()
    w.state_equal(twin)


@pytest.mark.parametrize("compact", [False, True])
def test_k3_minority_holder_repulls_and_matches_twin(compact):
    world, k = 4, 3
    w, twin = World(world, k=k, audit_every=1, compact=compact), World(world, k=k, compact=compact)
    steps = raws(world, 13, scales=(1.0, 1.0, 1.0, 1.0))
    for x in (w, twin):
        x.step(steps[0])
        x.settle()
    unit, s = 0, 1
    rank = (s + 2) % world  # the second buddy
    lo, hi = w.opts[0].layout.slice_bounds(unit, world, s)
    o = w.opts[rank]
    flip(o.m, o._pieces(o._table_host, lo + 8, lo + 9)[0][2], bit=20)
    for x in (w, twin):
        x.step(steps[1])   # the flipped m enters the update on one holder of three; the audit latches
        x.step(steps[2], veto=(0,) if x is twin else ())  # the latched error vetoes this step everywhere
        assert x.verdicts() == [False] * world
        x.configure()
        x.step(steps[3])
        x.settle()
    assert w.errors() == [None] * world and all(o.divergences == 1 for o in w.opts)
    assert all(o.lost_elements == 0 for o in w.opts) and w.opts[rank].pulled_bytes > 0
    w.replicas_agree()
    w.state_equal(twin)


def test_k2_disagreement_reseeds_the_slice():
    world = 3
    w = World(world, k=2, audit_every=1)
    steps = raws(world, 17, scales=(1.0, 1.0, 1.0, 1.0))
    w.step(steps[0])
    w.settle()
    unit, s = 1, 0
    lo, hi = w.opts[0].layout.slice_bounds(unit, world, s)
    flip(w.opts[(s + 1) % world].v, lo + 3, bit=20)
    w.step(steps[1])
    w.step(steps[2])
    assert w.verdicts() == [False] * world
    before = [o.lost_elements for o in w.opts]
    w.configure()
    grown = [o.lost_elements - b for o, b in zip(w.opts, before)]
    assert grown == [hi - lo if r in (s, (s + 1) % world) else 0 for r in range(world)]
    w.step(steps[3])
    w.settle()
    assert w.errors() == [None] * world
    w.replicas_agree()
    for name in ("master", "m", "v"):  # both holders were re-seeded alike and updated alike since
        a, b = (dict(w.opts[r]._state_arrays())[name][lo:hi].view(torch.uint8) for r in (s, (s + 1) % world))
        assert torch.equal(a, b)


# --------------------------------------------------------------------------- the trainer
def test_trainer_takes_audit_every_and_audits_nothing_alone(monkeypatch):
    from _zero1_replicas import trainer

    monkeypatch.delenv("TORCHFT_B200_Z1_AUDIT_EVERY", raising=False)
    g = torch.Generator().manual_seed(3)
    with trainer("llama3_debug", "aud_arg", audit_every=3) as tr:
        assert tr.zopt.audit_every == 3 and "z1_audit" in tr.pg.comm._segments
        for _ in range(4):
            tok = torch.randint(0, tr.cfg.vocab_size, (2, 64), generator=g).pin_memory()
            tr.step(tok, tok.clone())
        tr.manager.state_dict()
        assert tr.zopt.t == 4 and tr.zopt.audits == 0  # world 1: nothing to compare
    monkeypatch.setenv("TORCHFT_B200_Z1_AUDIT_EVERY", "2")
    with trainer("llama3_debug", "aud_env") as tr:
        assert tr.zopt.audit_every == 2
    monkeypatch.setenv("TORCHFT_B200_Z1_AUDIT_EVERY", "0")
    with trainer("llama3_debug", "aud_off") as tr:
        assert tr.zopt.audit_every == 0 and "z1_audit" not in tr.pg.comm._segments  # off: nothing allocated


def test_trainer_refuses_the_audit_on_the_classic_pipeline():
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    with pytest.raises(ValueError, match="audit_every"):
        FaultTolerantTrainer("llama3_debug", "http://127.0.0.1:1", zero1=False, audit_every=1)


def test_two_trainers_detect_and_repair_a_flipped_bit(tmp_path):
    """Two replicas in two processes on a local lighthouse, ``audit_every=1``. After step 2 replica 1 flips one bit of
    its moment ``m``: step 3's audit latches, step 4 fails on both replicas, the quorum re-forms, both holders of the
    diverged slice re-seed it, and training goes on. The replicas end with the same weights and state, bit for bit."""
    import json
    import os
    import subprocess
    import sys

    from torchft_b200.bench_utils import local_lighthouse, loopback

    steps = 7
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lh = local_lighthouse(min_replicas=2)
    try:
        procs = [subprocess.Popen([sys.executable, os.path.join(root, "bench", "audit_replica.py"), "--lighthouse",
                                   loopback(lh.address()), "--replica", str(r), "--steps", str(steps), "--flip-step", "2",
                                   "--out", str(tmp_path / f"r{r}.json")], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True) for r in range(2)]
        logs = [p.communicate(timeout=600)[0] for p in procs]
        for p, log in zip(procs, logs):
            assert p.returncode == 0, log[-4000:]
    finally:
        lh.shutdown()
    out = [json.loads((tmp_path / f"r{r}.json").read_text()) for r in range(2)]
    for o in out:
        assert o["divergences"] == 1, out
        assert o["t"] == steps - 1, out  # exactly one step failed
        assert o["lost_elements"] > 0 and o["errored"] is None, out
        assert o["audits"] >= steps - 1
    assert out[0]["param"] == out[1]["param"]
    assert out[0]["state"] == out[1]["state"] and out[0]["holdings"] == out[1]["holdings"]
