"""Optimizer state for direct ``zero1_update_`` launches: full-size, or a pool of pages in a shuffled slot order with
spare slots, and the state arguments of a launch over it."""

from __future__ import annotations

import torch

BF16, FP32 = torch.bfloat16, torch.float32
S16, S32 = 0x7FA5, 0x7FA5A5A5  # sentinel bit patterns (NaNs no kernel produces)
CHUNK = 1 << 24


def chunks(lo, hi):
    for a in range(lo, hi, CHUNK):
        yield a, min(hi, a + CHUNK)


class State:
    """One rank's optimizer state of ``n`` elements: full-size (``shift`` None; element e at e) or a pool of pages in a
    shuffled slot order with spare slots (element e, flat index soff + e, at
    ``table[(soff + e) >> shift] << shift | ((soff + e) & mask)``). Everything outside the ``held`` ranges is a sentinel.
    ``md`` is the moment type, "f32" or "bf16"."""

    def __init__(self, n, held, shift, soff, md, seed):
        self.n, self.held, self.shift, self.soff, self.md = n, held, shift, soff, md
        self.table = None
        if shift is None:
            size = n
        else:
            page = 1 << shift
            pages = sorted({p for lo, hi in held for p in range((soff + lo) >> shift, ((soff + hi - 1) >> shift) + 1)})
            nslots = len(pages) + 3
            slots = torch.randperm(nslots, generator=torch.Generator().manual_seed(seed))[:len(pages)]
            tab = torch.full((((soff + n) >> shift) + 1,), -1, dtype=torch.int32)
            if pages:
                tab[torch.tensor(pages)] = slots.int()
            self.table = tab.cuda()
            size = nslots * page
        self.master = torch.empty(max(size, 8), device="cuda")
        self.master.view(torch.int32).fill_(S32)
        mdt = FP32 if md == "f32" else BF16
        self.m = torch.empty(max(size, 8), dtype=mdt, device="cuda")
        self.v = torch.empty(max(size, 8), dtype=mdt, device="cuda")
        for x in (self.m, self.v):
            x.view(torch.int32 if mdt == FP32 else torch.int16).fill_(S32 if mdt == FP32 else S16)
        self.mask = torch.zeros(max(size, 8), dtype=torch.bool, device="cuda")
        for lo, hi in held:
            for a, b in chunks(lo, hi):
                self.mask[self.pos(a, b)] = True

    @classmethod
    def seeded(cls, init, shift=None, seed=0):
        """fp32 state over the whole of ``init``: the master weights ``init``, zero moments."""
        n = init.numel()
        st = cls(n, [(0, n)], shift, 0, "f32", seed)
        st.put(0, n, init.float(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"))
        return st

    def pos(self, lo, hi):
        if self.table is None:
            return slice(lo, hi)
        e = torch.arange(self.soff + lo, self.soff + hi, device="cuda")
        return (self.table[e >> self.shift].long() << self.shift) | (e & ((1 << self.shift) - 1))

    def get(self, lo, hi):
        """Copies of (master, m, v) over elements [lo, hi)."""
        p = self.pos(lo, hi)
        return self.master[p].clone(), self.m[p].clone(), self.v[p].clone()

    def put(self, lo, hi, w, m, v):
        p = self.pos(lo, hi)
        self.master[p], self.m[p], self.v[p] = w, m, v

    def args(self, lo=0):
        """The state arguments of ``zero1_update_`` for a unit that starts at element ``lo``."""
        kw = {"state_off": self.soff + lo, "moment_dtype": self.m.dtype}
        if self.table is None:
            return {"master": self.master.data_ptr() + 4 * lo, "m": self.m.data_ptr() + self.m.element_size() * lo,
                    "v": self.v.data_ptr() + self.v.element_size() * lo, **kw}
        return {"master": self.master.data_ptr(), "m": self.m.data_ptr(), "v": self.v.data_ptr(),
                "table": self.table.data_ptr(), "page_shift": self.shift, **kw}

    def untouched(self):
        out = ~self.mask
        ok = bool((self.master.view(torch.int32)[out] == S32).all())
        if self.m.dtype == FP32:
            ok &= bool((self.m.view(torch.int32)[out] == S32).all()) and bool((self.v.view(torch.int32)[out] == S32).all())
        else:
            ok &= bool((self.m.view(torch.int16)[out] == S16).all()) and bool((self.v.view(torch.int16)[out] == S16).all())
        return ok
