"""The one-GPU virtual world the collective tests run in: W ranks of one quorum whose kernels run concurrently on W
streams and synchronise through the real signal-pad protocol."""

from __future__ import annotations

from datetime import timedelta

import torch

DEV = torch.device("cuda", 0)


def _world(world, presignal=False, segs=None, timeout=20.0, staging=8 << 20):
    from torchft_b200.parallel.symm_mem import SymmetricComm

    return SymmetricComm.virtual_world(world, segs or {"buf": 4 << 20}, DEV, presignal=presignal,
                                       timeout=timedelta(seconds=timeout), staging_bytes=staging)


def _run(comms, fn, ranks=None):
    streams = getattr(_run, "_streams", None)
    if streams is None or len(streams) < len(comms):
        streams = _run._streams = [torch.cuda.Stream(device=DEV) for _ in range(8)]
    torch.cuda.synchronize()
    for r, c in enumerate(comms):
        if ranks is not None and r not in ranks:
            continue
        with torch.cuda.stream(streams[r]):
            fn(r, c, streams[r])
    torch.cuda.synchronize()


def _ok(comms):
    assert [c.errored() for c in comms] == [None] * len(comms)
