"""Debug aid: multi-piece send/recv between two in-process ranks; prints errors, timing and the pair's flag slots."""
import os
import sys
import time
from datetime import timedelta

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from torchft_b200.parallel.symm_mem import SymmetricComm  # noqa: E402

dev = torch.device("cuda", 0)
for staging, n in ((4 << 20, 300_001), (4 << 20, 20_000), (64 << 20, 300_001)):
    comms = SymmetricComm.virtual_world(3, {"buf": 1 << 20}, dev, presignal=False, timeout=timedelta(seconds=3), staging_bytes=staging)
    a = torch.arange(n, device=dev, dtype=torch.float32)
    ra = torch.zeros_like(a)
    s0, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    t0 = time.time()
    with torch.cuda.stream(s0):
        comms[0].send_(a, 2, s0)
    with torch.cuda.stream(s2):
        comms[2].recv_(ra, 0, s2)
    torch.cuda.synchronize()
    c0 = comms[0]
    pad0 = comms[0].segment("core")[: c0._K.SIGNAL_PAD_BYTES].view(torch.int64).view(4, c0._K.MAX_BLOCKS, 8)
    pad2 = comms[2].segment("core")[: c0._K.SIGNAL_PAD_BYTES].view(torch.int64).view(4, c0._K.MAX_BLOCKS, 8)
    print("staging", staging, "n", n, "mailbox", c0._mailbox_bytes, "took %.2fs" % (time.time() - t0), "match", bool(torch.equal(a, ra)),
          "first_bad", int((a != ra).nonzero()[0]) if not torch.equal(a, ra) else -1)
    print("  errs", [str(c.errored()) for c in comms])
    print("  rank2 pad data slots (from rank0):", [hex(int(pad2[3, 16 + b, 0])) for b in range(8)])
    print("  rank0 pad ack  slots (from rank2):", [hex(int(pad0[3, 24 + b, 2])) for b in range(8)], flush=True)
