"""Launch geometry of the NVLink collectives and the FT-ZeRO-1 kernels, without a GPU.

``SymmetricComm`` runs against a kernel module that records the grid of every launch and launches nothing, with the
constants of an H100 SXM (132 SMs). The tables below say what each entry point launches at the defaults, per world size
and message size: the kernel (``o`` one-shot, ``t`` two-shot, ``n`` NVLS all-reduce, ``rs`` reduce-scatter, ``x`` a
push-exchange round, ``q8`` fp8 all-reduce or reduce-scatter, ``qr`` / ``qg`` the slice-reduce and gather-dequantise
launches of the fp8 scratch path, ``q`` its quantise launch, ``h`` a handshake, ``z1r`` / ``z1u`` the FT-ZeRO-1 reduce
and update), a colon, its CTAs (``x`` threads per CTA where the caller picks them; ``+mc`` on the multicast address),
and ``*k`` for k identical launches in a row; ``too-large`` is a message the entry point refuses. A grid that changes
changes the bytes each CTA moves and the SMs a collective takes from the backward pass it overlaps, so a change to these
tables is a change of behaviour that needs its own measurement on the GPU.
"""

from __future__ import annotations

from types import SimpleNamespace

import torch

import _q8_emulation as Q
from torchft_b200.ops import _native
from torchft_b200.parallel import zero1 as zero1_mod
from torchft_b200.parallel.symm_mem import Segment, SymmetricComm

SMS = 132
# message sizes in bytes: every power of two from 16 B to 1 GiB, and 3 * 2**k + 2 B, which ends inside a 16-byte vector
SIZES = sorted({1 << k for k in range(4, 31)} | {(3 << k) + 2 for k in range(3, 28)})
UNITS = {  # FT-ZeRO-1 unit sizes in elements: a transformer block and the token embedding of Llama-3 1B and 8B, and two
    # units small enough for their grids to follow their size
    "1b_block": 60_821_504, "1b_embed": 128_256 * 2048, "8b_block": 218_112_000, "8b_embed": 128_256 * 4096,
    "2 Ki": 2048, "1 Mi": 1 << 20,
}
_HEAP = 1 << 48  # ordinary device memory, outside every segment


class _Table:
    def __init__(self, data, pads, rank, world):
        self.data = data

    def set_timeout_ms(self, ms):
        pass

    def with_data(self, data):
        return _Table(data, None, 0, 0)


class _Kernels:
    """The extension's constants and host-side sizes; every launcher appends its kernel and grid to ``calls``."""

    NUM_SMS = SMS
    MAX_BLOCKS = 2 * SMS
    ZERO1_MAX_BLOCKS = 32 * SMS
    SIGNAL_PAD_BYTES = 4 * 2 * SMS * 8 * 8
    PeerTable = _Table

    def __init__(self):
        self.calls = []

    q8_ngroups = staticmethod(Q.ngroups)
    q8_buffer_bytes = staticmethod(Q.buffer_bytes)
    q8_slice_buffer_bytes = staticmethod(Q.slice_buffer_bytes)

    @staticmethod
    def q8_rs_buffer_bytes(slice_elems, world):
        g = world * ((slice_elems + Q.GROUP - 1) // Q.GROUP)
        return Q.payload_off(g) + g * Q.GROUP

    def _rec(self, what):
        self.calls.append(what)

    def allreduce(self, *a):
        self._rec(f"{'ot'[a[12]]}:{a[13]}x{a[14]}")

    def allreduce_nvls(self, *a):
        self._rec(f"n:{a[10]}x{a[11]}")

    def reduce_scatter(self, *a):
        self._rec(f"rs:{a[11]}")

    def push_exchange(self, *a):
        self._rec(f"x:{a[-2]}")

    def q8_allreduce(self, *a):
        self._rec(f"q8:{a[-2]}")

    def q8_reduce_scatter(self, *a):
        self._rec(f"q8:{a[-2]}")

    def q8_quantize(self, *a):
        self._rec("q")

    def memset_async(self, *a):
        self._rec("z")

    def q8_slice_reduce(self, *a):
        self._rec(f"qr:{a[-2]}")

    def q8_gather_dequant(self, *a):
        self._rec(f"qg:{a[-2]}")

    def zero1_handshake(self, *a):
        self._rec("h")

    def zero1_reduce(self, *a):
        self._rec(f"z1r:{a[-3]}x{a[-2]}{'+mc' if a[2] else ''}")

    def zero1_update(self, *a):
        self._rec(f"z1u:{a[-3]}x{a[-2]}{'+mc' if a[1] else ''}")


class _T:
    """What ``SymmetricComm`` reads of a contiguous CUDA tensor: an address, an element count and a dtype."""

    is_cuda = True

    def __init__(self, ptr, numel, dtype=torch.bfloat16):
        self.ptr, self.n, self.dtype = ptr, numel, dtype
        self.rows = 1

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n

    def element_size(self):
        return self.dtype.itemsize

    def is_contiguous(self):
        return True

    def contiguous(self):
        return _T(_HEAP, self.n, self.dtype)

    def record_stream(self, stream):
        pass

    def view(self, *shape):
        t = _T(self.ptr, self.n, self.dtype)
        t.rows = shape[0] if len(shape) == 2 else 1
        return t

    def __getitem__(self, idx):
        cols = idx[1] if isinstance(idx, tuple) else idx  # rows[:, lo:hi] of a (W, n) view, or flat[lo:hi]
        return _T(self.ptr + cols.start * self.element_size(), self.rows * (cols.stop - cols.start), self.dtype)


STREAM = SimpleNamespace(cuda_stream=0)


def _comm(monkeypatch, world, mc=False, q8_scratch=False):
    """Rank 0 of a configured ``world``-rank quorum at the constructor's defaults, with a 16 GiB user segment ``buf``
    (on a multicast object with ``mc``), FT-ZeRO-1 segments and, with ``q8_scratch``, an fp8 scratch segment."""
    K = _Kernels()
    monkeypatch.setattr(_native, "load", lambda: K)
    c = SymmetricComm(torch.device("cpu"))
    sizes = {"core": c._pad_bytes + c._staging_bytes, "buf": 16 << 30, "z1_grad": 2 << 30, "z1_param": 2 << 30}
    if q8_scratch:
        sizes["x_q8"] = 4 << 30
    base = 1 << 40
    for name, nbytes in sizes.items():
        c._segments[name] = Segment(name, base, nbytes, b"", None)
        base += nbytes + (1 << 30)
    c._install({n: [s.ptr + (r << 44) for r in range(world)] for n, s in c._segments.items()}, 0, world, 1, 0)
    c._configured = True
    if mc:
        for name in ("buf", "z1_grad", "z1_param"):
            c._mc[name] = (1, 1 << 45, sizes[name])
    return c, K


def _launches(K, fn):
    del K.calls[:]
    try:
        fn()
    except ValueError:
        return "too-large"
    runs = []
    for call in K.calls:
        if runs and runs[-1][0] == call:
            runs[-1][1] += 1
        else:
            runs.append([call, 1])
    return "+".join(c if k == 1 else f"{c}*{k}" for c, k in runs)


def _allreduce(monkeypatch):
    table = {}
    for W in range(1, 9):
        for path in ("zero-copy", "multicast", "staged"):
            c, K = _comm(monkeypatch, W, mc=path == "multicast")
            ptr = _HEAP if path == "staged" else c._segments["buf"].ptr
            table[(W, path)] = [_launches(K, lambda: c.allreduce_(_T(ptr, nb // 2), scale=0.5, stream=STREAM))
                                for nb in SIZES]
    return table


def _reduce_scatter(monkeypatch):
    """``nb`` bytes per rank slice, ``W * nb`` of input."""
    table = {}
    for W in range(2, 9):
        c, K = _comm(monkeypatch, W)
        for path in ("zero-copy", "staged"):
            ptr = _HEAP if path == "staged" else c._segments["buf"].ptr
            table[(W, path)] = [_launches(K, lambda: c.reduce_scatter_(_T(_HEAP, nb // 2), _T(ptr, W * (nb // 2)),
                                                                       stream=STREAM)) for nb in SIZES]
        table[(W, "xgrid")] = [f"x:{c._xgrid(nb)}" for nb in SIZES]
    return table


def _q8(monkeypatch):
    """fp8 all-reduce of ``nb`` bytes of bf16 through staging and through an fp8 scratch segment; fp8 reduce-scatter
    of ``nb`` bytes per rank slice."""
    table = {}
    for W in range(2, 9):
        for path in ("staged", "scratch"):
            c, K = _comm(monkeypatch, W, q8_scratch=path == "scratch")
            table[(W, f"allreduce {path}")] = [
                _launches(K, lambda: c.q8_allreduce_(_T(_HEAP, nb // 2), _T(_HEAP, nb // 2), scale=0.5, stream=STREAM))
                for nb in SIZES]
        table[(W, "reduce_scatter")] = [
            _launches(K, lambda: c.q8_reduce_scatter_(_T(_HEAP, nb // 2), _T(_HEAP, W * (nb // 2)), nb // 2, stream=STREAM))
            for nb in SIZES]
    return table


def _zero1_optimizer(monkeypatch, comm, **kw):
    """A ``Zero1Optimizer`` over ``comm`` with host memory in place of the symmetric segments (no quorum, no kernel)."""
    monkeypatch.setattr(torch.cuda, "Stream", lambda device=None: None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: None)
    pg = SimpleNamespace(comm=comm, alloc_symmetric=lambda name, nbytes: torch.zeros(nbytes, dtype=torch.uint8),
                         add_configure_hook=lambda fn: None)
    return zero1_mod.Zero1Optimizer(pg, 64, **kw)


def _zero1(monkeypatch):
    """Reduce-scatter (with the gradient norm) and update of one unit, at the grids ``Zero1Optimizer`` passes."""
    table = {}
    for W in range(1, 9):
        c, K = _comm(monkeypatch, W, mc=True)
        opt = _zero1_optimizer(monkeypatch, c)
        gate = _T(_HEAP, 2, torch.int32)
        for name, n in UNITS.items():
            rs = _launches(K, lambda: c.zero1_reduce_scatter_("z1_grad", 0, n, 0.5, True, 2, opt._rs_blocks, STREAM,
                                                               gnorm=_HEAP))
            upd = _launches(K, lambda: c.zero1_update_("z1_param", 0, _HEAP, _HEAP, _HEAP, _HEAP, n, (1e-3, 0.9, 0.95, 1e-8,
                                                       0.1), gate, 2, 0, opt._upd_blocks, STREAM))
            table[(W, name)] = f"{rs} {upd}"
        n = UNITS["1b_block"]  # a grid asked for beyond the kernels' cap
        rs = _launches(K, lambda: c.zero1_reduce_scatter_("z1_grad", 0, n, 0.5, True, 2, 1 << 20, STREAM))
        upd = _launches(K, lambda: c.zero1_update_("z1_param", 0, _HEAP, _HEAP, _HEAP, _HEAP, n, (1e-3, 0.9, 0.95, 1e-8, 0.1),
                                                   gate, 2, 0, 1 << 20, STREAM))
        table[(W, "capped")] = f"{rs} {upd}"
        table[(W, "norm scratch")] = c._z1_norm_scratch.numel()
    return table


def _check(got, want):
    assert got.keys() == want.keys()
    for key in want:
        if isinstance(want[key], list):
            assert len(got[key]) == len(want[key]), key
            bad = [(nb, g, w) for nb, g, w in zip(SIZES, got[key], want[key]) if g != w]
            assert not bad, f"{key}: (bytes, got, want) {bad[:4]}"
        else:
            assert got[key] == want[key], key


def test_allreduce_geometry(monkeypatch):
    _check(_allreduce(monkeypatch), ALLREDUCE)


def test_reduce_scatter_and_exchange_geometry(monkeypatch):
    _check(_reduce_scatter(monkeypatch), REDUCE_SCATTER)


def test_q8_geometry(monkeypatch):
    _check(_q8(monkeypatch), Q8)


def test_zero1_geometry(monkeypatch):
    _check(_zero1(monkeypatch), ZERO1)


def test_zero1_replication_is_the_argument(monkeypatch):
    """The holders per slice are what the caller asked for, whatever the environment holds."""
    monkeypatch.setenv("TORCHFT_B200_Z1_REPLICATION", "1")
    c, _ = _comm(monkeypatch, 4)
    opt = _zero1_optimizer(monkeypatch, c, replication=3)
    assert opt._replication == 3 and opt.layout.replication == 3


# ---------------------------------------------------------------------------------------------------------------- tables
ALLREDUCE = {
    (1, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 'o:97x512', 'o:128x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (1, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 'o:97x512', 'o:128x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (1, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 'o:97x512', 'o:128x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (2, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 'o:97x512', 'o:128x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (2, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 'o:97x512', 'o:128x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (2, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 'o:97x512', 'o:128x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (3, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (3, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (3, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (4, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (4, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (4, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 'o:25x512', 'o:32x512', 'o:49x512', 'o:64x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (5, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (5, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'n:8x512', 't:8x512', 'n:8x512', 't:12x512', 'n:16x512', 't:24x512', 'n:32x512', 't:48x512',
        'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512',
        't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 'n:64x512',
    ],
    (5, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (6, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (6, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'n:8x512', 't:8x512', 'n:8x512', 't:12x512', 'n:16x512', 't:24x512', 'n:32x512', 't:48x512',
        'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512',
        't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 'n:64x512',
    ],
    (6, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (7, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (7, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'n:8x512', 't:8x512', 'n:8x512', 't:12x512', 'n:16x512', 't:24x512', 'n:32x512', 't:48x512',
        'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512',
        't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 'n:64x512',
    ],
    (7, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
    (8, 'zero-copy'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
    ],
    (8, 'multicast'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'n:8x512', 't:8x512', 'n:8x512', 't:12x512', 'n:16x512', 't:24x512', 'n:32x512', 't:48x512',
        'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512',
        't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 't:64x512', 'n:64x512', 'n:64x512',
    ],
    (8, 'staged'): [
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512', 'o:1x512',
        'o:1x512', 'o:1x512', 'o:1x512', 'o:2x512', 'o:2x512', 'o:4x512', 'o:4x512', 'o:7x512', 'o:8x512',
        'o:13x512', 'o:16x512', 't:8x512', 't:8x512', 't:12x512', 't:16x512', 't:24x512', 't:32x512', 't:48x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512', 't:64x512',
        't:64x512', 't:64x512', 't:64x512', 't:64x512*2', 't:64x512*2', 't:64x512*3', 't:64x512*5',
    ],
}

REDUCE_SCATTER = {
    (2, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (2, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64*2', 'rs:64*2', 'rs:64*3',
        'rs:64*4', 'rs:64*5', 'rs:64*10',
    ],
    (2, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
    (3, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (3, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64*2', 'rs:64*2', 'rs:64*3', 'rs:64*4',
        'rs:64*6', 'rs:64*7', 'rs:64*14',
    ],
    (3, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
    (4, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (4, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64*2', 'rs:64*2', 'rs:64*3', 'rs:64*4', 'rs:64*5',
        'rs:64*7', 'rs:64*10', 'rs:64*19',
    ],
    (4, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
    (5, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (5, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64+rs:51', 'rs:64*2', 'rs:64*3', 'rs:64*3', 'rs:64*5',
        'rs:64*6', 'rs:64*9', 'rs:64*12', 'rs:64*23',
    ],
    (5, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
    (6, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (6, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64*2', 'rs:64*2', 'rs:64*3', 'rs:64*4', 'rs:64*6',
        'rs:64*7', 'rs:64*11', 'rs:64*14', 'rs:64*28',
    ],
    (6, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
    (7, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (7, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64*2', 'rs:64*2', 'rs:64*3+rs:1', 'rs:64*4',
        'rs:64*6+rs:1', 'rs:64*8', 'rs:64*12+rs:1', 'rs:64*16', 'rs:64*32',
    ],
    (7, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
    (8, 'zero-copy'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64',
        'rs:64', 'rs:64',
    ],
    (8, 'staged'): [
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1', 'rs:1',
        'rs:2', 'rs:3', 'rs:4', 'rs:6', 'rs:8', 'rs:12', 'rs:16', 'rs:24', 'rs:32', 'rs:48', 'rs:64', 'rs:64',
        'rs:64', 'rs:64', 'rs:64', 'rs:64', 'rs:64*2', 'rs:64*2', 'rs:64*3', 'rs:64*4', 'rs:64*5', 'rs:64*7',
        'rs:64*10', 'rs:64*14', 'rs:64*19', 'rs:64*37',
    ],
    (8, 'xgrid'): [
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1',
        'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:1', 'x:2', 'x:3', 'x:4', 'x:6',
        'x:8', 'x:12', 'x:16', 'x:24', 'x:32', 'x:48', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
        'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64', 'x:64',
    ],
}

Q8 = {
    (2, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (2, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:2', 'q+h+qr:2+h+qg:3', 'q+h+qr:2+h+qg:4', 'q+h+qr:3+h+qg:5',
        'q+h+qr:4+h+qg:7', 'q+h+qr:5+h+qg:9', 'q+h+qr:7+h+qg:13', 'q+h+qr:9+h+qg:17', 'q+h+qr:13+h+qg:25',
        'q+h+qr:17+h+qg:33', 'q+h+qr:25+h+qg:49', 'q+h+qr:33+h+qg:65', 'q+h+qr:49+h+qg:97', 'q+h+qr:65+h+qg:129',
        'q+h+qr:97+h+qg:193', 'q+h+qr:129+h+qg:257', 'q+h+qr:193+h+qg:385', 'q+h+qr:257+h+qg:513',
        'q+h+qr:385+h+qg:769', 'q+h+qr:513+h+qg:1025', 'q+h+qr:769+h+qg:1537', 'q+h+qr:1025+h+qg:2049',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (2, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:5', 'q8:7',
        'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
    (3, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (3, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:3', 'q+h+qr:2+h+qg:4', 'q+h+qr:2+h+qg:5',
        'q+h+qr:3+h+qg:7', 'q+h+qr:3+h+qg:9', 'q+h+qr:5+h+qg:13', 'q+h+qr:6+h+qg:17', 'q+h+qr:9+h+qg:25',
        'q+h+qr:11+h+qg:33', 'q+h+qr:17+h+qg:49', 'q+h+qr:22+h+qg:65', 'q+h+qr:33+h+qg:97', 'q+h+qr:43+h+qg:129',
        'q+h+qr:65+h+qg:193', 'q+h+qr:86+h+qg:257', 'q+h+qr:129+h+qg:385', 'q+h+qr:171+h+qg:513',
        'q+h+qr:257+h+qg:769', 'q+h+qr:342+h+qg:1025', 'q+h+qr:513+h+qg:1537', 'q+h+qr:683+h+qg:2049',
        'q+h+qr:1025+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (3, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:5', 'q8:7', 'q8:10',
        'q8:13', 'q8:19', 'q8:25', 'q8:37', 'q8:49', 'q8:73', 'q8:97', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'too-large', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
    (4, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (4, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:2',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:3', 'q+h+qr:1+h+qg:4', 'q+h+qr:2+h+qg:5',
        'q+h+qr:2+h+qg:7', 'q+h+qr:3+h+qg:9', 'q+h+qr:4+h+qg:13', 'q+h+qr:5+h+qg:17', 'q+h+qr:7+h+qg:25',
        'q+h+qr:9+h+qg:33', 'q+h+qr:13+h+qg:49', 'q+h+qr:17+h+qg:65', 'q+h+qr:25+h+qg:97', 'q+h+qr:33+h+qg:129',
        'q+h+qr:49+h+qg:193', 'q+h+qr:65+h+qg:257', 'q+h+qr:97+h+qg:385', 'q+h+qr:129+h+qg:513',
        'q+h+qr:193+h+qg:769', 'q+h+qr:257+h+qg:1025', 'q+h+qr:385+h+qg:1537', 'q+h+qr:513+h+qg:2049',
        'q+h+qr:769+h+qg:2112', 'q+h+qr:1025+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (4, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:5', 'q8:7', 'q8:9', 'q8:13',
        'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'too-large',
        'too-large', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
    (5, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (5, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:3', 'q+h+qr:1+h+qg:4', 'q+h+qr:1+h+qg:5',
        'q+h+qr:2+h+qg:7', 'q+h+qr:2+h+qg:9', 'q+h+qr:3+h+qg:13', 'q+h+qr:4+h+qg:17', 'q+h+qr:5+h+qg:25',
        'q+h+qr:7+h+qg:33', 'q+h+qr:10+h+qg:49', 'q+h+qr:13+h+qg:65', 'q+h+qr:20+h+qg:97', 'q+h+qr:26+h+qg:129',
        'q+h+qr:39+h+qg:193', 'q+h+qr:52+h+qg:257', 'q+h+qr:77+h+qg:385', 'q+h+qr:103+h+qg:513',
        'q+h+qr:154+h+qg:769', 'q+h+qr:205+h+qg:1025', 'q+h+qr:308+h+qg:1537', 'q+h+qr:410+h+qg:2049',
        'q+h+qr:615+h+qg:2112', 'q+h+qr:820+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (5, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:6', 'q8:8', 'q8:11', 'q8:16',
        'q8:21', 'q8:31', 'q8:41', 'q8:61', 'q8:81', 'q8:121', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'too-large', 'too-large',
        'too-large', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
    (6, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (6, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:2',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:3', 'q+h+qr:1+h+qg:4', 'q+h+qr:1+h+qg:5',
        'q+h+qr:2+h+qg:7', 'q+h+qr:2+h+qg:9', 'q+h+qr:3+h+qg:13', 'q+h+qr:3+h+qg:17', 'q+h+qr:5+h+qg:25',
        'q+h+qr:6+h+qg:33', 'q+h+qr:9+h+qg:49', 'q+h+qr:11+h+qg:65', 'q+h+qr:17+h+qg:97', 'q+h+qr:22+h+qg:129',
        'q+h+qr:33+h+qg:193', 'q+h+qr:43+h+qg:257', 'q+h+qr:65+h+qg:385', 'q+h+qr:86+h+qg:513',
        'q+h+qr:129+h+qg:769', 'q+h+qr:171+h+qg:1025', 'q+h+qr:257+h+qg:1537', 'q+h+qr:342+h+qg:2049',
        'q+h+qr:513+h+qg:2112', 'q+h+qr:683+h+qg:2112', 'q+h+qr:1025+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (6, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:5', 'q8:7', 'q8:10', 'q8:13', 'q8:19',
        'q8:25', 'q8:37', 'q8:49', 'q8:73', 'q8:97', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'too-large', 'too-large',
        'too-large', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
    (7, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (7, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:3', 'q+h+qr:1+h+qg:4', 'q+h+qr:1+h+qg:5',
        'q+h+qr:1+h+qg:7', 'q+h+qr:2+h+qg:9', 'q+h+qr:2+h+qg:13', 'q+h+qr:3+h+qg:17', 'q+h+qr:4+h+qg:25',
        'q+h+qr:5+h+qg:33', 'q+h+qr:7+h+qg:49', 'q+h+qr:10+h+qg:65', 'q+h+qr:14+h+qg:97', 'q+h+qr:19+h+qg:129',
        'q+h+qr:28+h+qg:193', 'q+h+qr:37+h+qg:257', 'q+h+qr:55+h+qg:385', 'q+h+qr:74+h+qg:513',
        'q+h+qr:110+h+qg:769', 'q+h+qr:147+h+qg:1025', 'q+h+qr:220+h+qg:1537', 'q+h+qr:293+h+qg:2049',
        'q+h+qr:439+h+qg:2112', 'q+h+qr:586+h+qg:2112', 'q+h+qr:878+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (7, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:6', 'q8:8', 'q8:11', 'q8:15', 'q8:22',
        'q8:29', 'q8:43', 'q8:57', 'q8:85', 'q8:113', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'too-large', 'too-large', 'too-large',
        'too-large', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
    (8, 'allreduce staged'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25', 'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132*2', 'q8:132*3',
    ],
    (8, 'allreduce scratch'): [
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1',
        'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:1', 'q+h+qr:1+h+qg:2',
        'q+h+qr:1+h+qg:2', 'q+h+qr:1+h+qg:3', 'q+h+qr:1+h+qg:3', 'q+h+qr:1+h+qg:4', 'q+h+qr:1+h+qg:5',
        'q+h+qr:1+h+qg:7', 'q+h+qr:2+h+qg:9', 'q+h+qr:2+h+qg:13', 'q+h+qr:3+h+qg:17', 'q+h+qr:4+h+qg:25',
        'q+h+qr:5+h+qg:33', 'q+h+qr:7+h+qg:49', 'q+h+qr:9+h+qg:65', 'q+h+qr:13+h+qg:97', 'q+h+qr:17+h+qg:129',
        'q+h+qr:25+h+qg:193', 'q+h+qr:33+h+qg:257', 'q+h+qr:49+h+qg:385', 'q+h+qr:65+h+qg:513',
        'q+h+qr:97+h+qg:769', 'q+h+qr:129+h+qg:1025', 'q+h+qr:193+h+qg:1537', 'q+h+qr:257+h+qg:2049',
        'q+h+qr:385+h+qg:2112', 'q+h+qr:513+h+qg:2112', 'q+h+qr:769+h+qg:2112', 'q+h+qr:1025+h+qg:2112',
        'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112', 'q+h+qr:1056+h+qg:2112',
        'q+h+qr:1056+h+qg:2112',
    ],
    (8, 'reduce_scatter'): [
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4',
        'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:4', 'q8:5', 'q8:7', 'q8:9', 'q8:13', 'q8:17', 'q8:25',
        'q8:33', 'q8:49', 'q8:65', 'q8:97', 'q8:129', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132',
        'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'q8:132', 'too-large', 'too-large', 'too-large',
        'too-large', 'too-large', 'too-large', 'too-large', 'too-large',
    ],
}

ZERO1 = {
    (1, '1b_block'): 'z1r:128x512 z1u:2112x512',
    (1, '1b_embed'): 'z1r:128x512 z1u:2112x512',
    (1, '8b_block'): 'z1r:128x512 z1u:2112x512',
    (1, '8b_embed'): 'z1r:128x512 z1u:2112x512',
    (1, '2 Ki'): 'z1r:1x512 z1u:1x512',
    (1, '1 Mi'): 'z1r:128x512 z1u:256x512',
    (1, 'capped'): 'z1r:4224x512 z1u:4224x512',
    (1, 'norm scratch'): 4225,
    (2, '1b_block'): 'h+z1r:128x512+h z1u:2112x512',
    (2, '1b_embed'): 'h+z1r:128x512+h z1u:2112x512',
    (2, '8b_block'): 'h+z1r:128x512+h z1u:2112x512',
    (2, '8b_embed'): 'h+z1r:128x512+h z1u:2112x512',
    (2, '2 Ki'): 'h+z1r:1x512+h z1u:1x512',
    (2, '1 Mi'): 'h+z1r:128x512+h z1u:256x512',
    (2, 'capped'): 'h+z1r:4224x512+h z1u:4224x512',
    (2, 'norm scratch'): 4225,
    (3, '1b_block'): 'h+z1r:128x512+h z1u:2112x512+h',
    (3, '1b_embed'): 'h+z1r:128x512+h z1u:2112x512+h',
    (3, '8b_block'): 'h+z1r:128x512+h z1u:2112x512+h',
    (3, '8b_embed'): 'h+z1r:128x512+h z1u:2112x512+h',
    (3, '2 Ki'): 'h+z1r:1x512+h z1u:1x512+h',
    (3, '1 Mi'): 'h+z1r:128x512+h z1u:256x512+h',
    (3, 'capped'): 'h+z1r:4224x512+h z1u:4224x512+h',
    (3, 'norm scratch'): 4225,
    (4, '1b_block'): 'h+z1r:128x512+h z1u:2112x512+h',
    (4, '1b_embed'): 'h+z1r:128x512+h z1u:2112x512+h',
    (4, '8b_block'): 'h+z1r:128x512+h z1u:2112x512+h',
    (4, '8b_embed'): 'h+z1r:128x512+h z1u:2112x512+h',
    (4, '2 Ki'): 'h+z1r:1x512+h z1u:1x512+h',
    (4, '1 Mi'): 'h+z1r:128x512+h z1u:256x512+h',
    (4, 'capped'): 'h+z1r:4224x512+h z1u:4224x512+h',
    (4, 'norm scratch'): 4225,
    (5, '1b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (5, '1b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (5, '8b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (5, '8b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (5, '2 Ki'): 'h+z1r:1x512+h z1u:1x512+h',
    (5, '1 Mi'): 'h+z1r:128x512+mc+h z1u:256x512+mc+h',
    (5, 'capped'): 'h+z1r:4224x512+mc+h z1u:4224x512+mc+h',
    (5, 'norm scratch'): 4225,
    (6, '1b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (6, '1b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (6, '8b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (6, '8b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (6, '2 Ki'): 'h+z1r:1x512+h z1u:1x512+h',
    (6, '1 Mi'): 'h+z1r:128x512+mc+h z1u:256x512+mc+h',
    (6, 'capped'): 'h+z1r:4224x512+mc+h z1u:4224x512+mc+h',
    (6, 'norm scratch'): 4225,
    (7, '1b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (7, '1b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (7, '8b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (7, '8b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (7, '2 Ki'): 'h+z1r:1x512+h z1u:1x512+h',
    (7, '1 Mi'): 'h+z1r:128x512+mc+h z1u:256x512+mc+h',
    (7, 'capped'): 'h+z1r:4224x512+mc+h z1u:4224x512+mc+h',
    (7, 'norm scratch'): 4225,
    (8, '1b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (8, '1b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (8, '8b_block'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (8, '8b_embed'): 'h+z1r:128x512+mc+h z1u:2112x512+mc+h',
    (8, '2 Ki'): 'h+z1r:1x512+h z1u:1x512+h',
    (8, '1 Mi'): 'h+z1r:128x512+mc+h z1u:256x512+mc+h',
    (8, 'capped'): 'h+z1r:4224x512+mc+h z1u:4224x512+mc+h',
    (8, 'norm scratch'): 4225,
}
