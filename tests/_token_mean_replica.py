"""One run of ``FaultTolerantTrainer(global_token_mean=True)`` on ``llama3_debug`` for
``tests/test_zero1_token_mean_gpu.py``: either one of two replicas that each train one micro-batch of every step
(``--replica r``, ``min_replica_size=2``), or one replica that trains both micro-batches with ``grad_accum_steps=2``
(``--replica all``). Each step's two micro-batches of ``--batch`` rows have different masks (see :func:`batch`), and
attention runs SDPA's flash kernels with deterministic algorithms on, so that every run computes each micro-batch's
gradient with the same bits.

Writes one JSON file (``--out``): the reported losses (as ``float.hex``), the update count and SHA-256 digests of the
bf16 weights and of the fp32 master weights and moments (full-size state: every replica holds every slice here).

    python tests/_token_mean_replica.py --lighthouse http://127.0.0.1:PORT --replica 0 --steps 3 --out r0.json
"""

from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
from datetime import timedelta

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # required by deterministic algorithms, before cuBLAS starts

import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def batch(step: int, vocab: int, B: int, S: int):
    """The ``(2 B, S)`` tokens and targets of ``step``: micro-batch 0 (rows ``0 .. B-1``) ignores the second half of
    every row, micro-batch 1 every third target."""
    g = torch.Generator().manual_seed(1000 + step)
    tok = torch.randint(0, vocab, (2 * B, S), generator=g)
    tgt = torch.randint(0, vocab, (2 * B, S), generator=g)
    tgt[:B, S // 2:] = -100
    tgt[B:, ::3] = -100
    return tok, tgt


def digest(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lighthouse", required=True)
    ap.add_argument("--replica", required=True, help="0 or 1 (one of two replicas), or all (one replica, M = 2)")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    alone = a.replica == "all"
    tr = FaultTolerantTrainer("llama3_debug", a.lighthouse, replica_id=f"tokmean_{a.replica}",
                              min_replica_size=1 if alone else 2, timeout=timedelta(seconds=60), seed=0,
                              grad_accum_steps=2 if alone else 1, global_token_mean=True)
    B = a.batch
    rows = slice(0, 2 * B) if alone else slice(int(a.replica) * B, (int(a.replica) + 1) * B)
    losses = []
    torch.use_deterministic_algorithms(True)
    try:
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
            for step in range(a.steps):
                tok, tgt = batch(step, tr.cfg.vocab_size, B, a.seq)
                losses.append(tr.step(tok[rows].contiguous().pin_memory(), tgt[rows].contiguous().pin_memory()))
        tr.manager.state_dict()  # resolves the last step's verdict
        tr.join()
        torch.cuda.synchronize()
        z = tr.zopt
        out = {"losses": [float(x).hex() for x in losses], "t": z.t, "param": digest(z.param),
               "master": digest(z.master), "m": digest(z.m), "v": digest(z.v),
               "row_mismatch_steps": z.row_mismatch_steps}
    finally:
        torch.use_deterministic_algorithms(False)
        tr.shutdown()
    with open(a.out, "w") as f:
        json.dump(out, f)


if __name__ == "__main__":
    main()
