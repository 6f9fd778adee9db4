"""One replica of a two-replica FT-ZeRO-1 ``FaultTolerantTrainer`` with the replica audit on (``audit_every=1``), for
``tests/test_zero1_audit_gpu.py`` and ``bench/audit_bench.py``. Start two of them, ``--replica 0`` and ``--replica 1``,
against one Lighthouse that waits for two replicas; both may share one GPU.

* ``--flip-step s``: after step ``s`` replica 1 flips one bit of its optimizer moment ``m`` in the middle of unit 1
  (a data write). Its next update diverges from its peer's, that step's audit latches, the step after fails on both
  replicas, the quorum re-forms and the diverged slice is re-seeded; training goes on.
* ``--bench-blocks n``: after the steps, ``n`` blocks of ``--block`` steps alternate the audit off and on (both replicas
  switch at the same step), each block timed by the host clock between device synchronisations.

Writes one JSON file (``--out``): update count, audit counters, SHA-256 of the bf16 weights and of the held state, and
the block times.

    python bench/audit_replica.py --lighthouse http://127.0.0.1:PORT --replica 0 --steps 6 --flip-step 2 --out r0.json
"""

from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time
from datetime import timedelta

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lighthouse", required=True)
    ap.add_argument("--replica", type=int, required=True)
    ap.add_argument("--model", default="llama3_debug")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--flip-step", type=int, default=-1)
    ap.add_argument("--bench-blocks", type=int, default=0)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    tr = FaultTolerantTrainer(a.model, a.lighthouse, replica_id=f"audit_{a.replica}", min_replica_size=2,
                              timeout=timedelta(seconds=60), lr=1e-3, seed=0, audit_every=1)
    z = tr.zopt
    g = torch.Generator().manual_seed(100 + a.replica)

    def step() -> None:
        tok = torch.randint(0, tr.cfg.vocab_size, (a.batch, a.seq), generator=g).pin_memory()
        tgt = torch.randint(0, tr.cfg.vocab_size, (a.batch, a.seq), generator=g).pin_memory()
        tr.step(tok, tgt)

    try:
        for i in range(a.steps):
            step()
            if i == a.flip_step and a.replica == 1:
                tr.join()
                torch.cuda.synchronize()
                lo, hi = z.layout.units[1]
                z.m.view(torch.int32)[(lo + hi) // 2] ^= 1 << 20
                torch.cuda.synchronize()
        blocks = {"off": [], "on": []}
        for b in range(2 * a.bench_blocks):
            mode = "off" if b % 2 == 0 else "on"
            z.audit_every = 0 if mode == "off" else 1
            tr.join()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.block):
                step()
            tr.join()
            torch.cuda.synchronize()
            blocks[mode].append((time.perf_counter() - t0) * 1e3 / a.block)
        tr.manager.state_dict()  # resolves the last step's verdict
        tr.join()
        torch.cuda.synchronize()
        state = hashlib.sha256()
        for (lo, hi), arrays in sorted(z.held_state().items()):
            state.update(f"{lo}:{hi}".encode())
            for x in arrays:
                state.update(x.contiguous().view(torch.uint8).cpu().numpy().tobytes())
        out = {"replica": a.replica, "t": z.t, "audits": z.audits, "divergences": z.divergences,
               "lost_elements": z.lost_elements, "holdings": z._holdings,
               "param": hashlib.sha256(z.param.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest(),
               "state": state.hexdigest(), "ms_per_step": blocks,
               "errored": None if tr.pg.errored() is None else str(tr.pg.errored())}
        with open(a.out, "w") as f:
            json.dump(out, f)
    finally:
        tr.shutdown()


if __name__ == "__main__":
    main()
