"""The cost of FT-ZeRO-1's global token mean: a trainer step with the option off and on, and the commit kernel alone.

    python bench/token_mean_step.py --model llama3_1b --seq 8192 --steps 10 --warmup 3 --virtual 8

* step: two ``FaultTolerantTrainer`` (FT-ZeRO-1, one replica each, on their own local lighthouses) in one process, one
  without and one with ``global_token_mean``, stepped in alternated rounds (so that clocks and neighbours weigh on both
  arms alike) on the same batch of packed documents (10 per row of ``--seq`` tokens). Each step is timed from the
  host's call to the end of its update, with CUDA events.
* commit: the commit kernel of every rank of a pre-signalled ``--virtual``-rank world, with and without the token slots
  (plus clipping in both), timed over ``--commits`` launches per rank.

Prints one JSON line with the medians, the spread (min, max), the card's name and power limit read in the same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from datetime import timedelta

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def stats(t) -> dict:
    t = np.asarray(t)
    return {"median": round(float(np.median(t)), 3), "min": round(float(t.min()), 3), "max": round(float(t.max()), 3),
            "n": int(t.size)}


def step_bench(args) -> dict:
    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.data import pack_documents
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    B, S = args.batch, args.seq
    rng = np.random.default_rng(0)
    arms, lhs = {}, []
    for name, tm in (("off", False), ("on", True)):
        lh = local_lighthouse()
        lhs.append(lh)
        arms[name] = FaultTolerantTrainer(args.model, loopback(lh.address()), replica_id=f"tm_{name}_0",
                                          timeout=timedelta(seconds=60), global_token_mean=tm)
    vocab = arms["off"].cfg.vocab_size
    docs = [rng.integers(0, vocab, size=S // 10) for _ in range(10 * B + 1)]
    tok, tgt, cu = next(pack_documents(docs, B, S))
    tok, tgt = tok.pin_memory(), tgt.pin_memory()
    times = {n: [] for n in arms}
    losses = {}
    try:
        for i in range(args.warmup + args.steps):
            for name, tr in arms.items():
                torch.cuda.synchronize()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                losses[name] = tr.step(tok, tgt, cu)
                tr.join()
                e.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[name].append(s.elapsed_time(e))
    finally:
        for tr in arms.values():
            tr.shutdown()
        for lh in lhs:
            lh.shutdown()
    out = {"model": args.model, "seq": S, "batch": B, "documents_per_row": 10,
           "valid_targets": int((tgt != -100).sum()), "targets": int(tgt.numel())}
    for name in arms:
        out[name] = {"ms_per_step": stats(times[name]), "loss": losses[name]}
    out["on_minus_off_ms"] = round(out["on"]["ms_per_step"]["median"] - out["off"]["ms_per_step"]["median"], 3)
    return out


def commit_bench(args) -> dict:
    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import GNORM_UNITS

    W, dev = args.virtual, torch.device("cuda", 0)
    seg = {"z1_gnorm": GNORM_UNITS * 8, "z1_tokmean": 64}
    comms = SymmetricComm.virtual_world(W, seg, presignal=True, timeout=timedelta(seconds=20))
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    norm = [torch.zeros(2, dtype=torch.float32, device=dev) for _ in comms]
    out_ = [torch.zeros(2, dtype=torch.float32, device=dev) for _ in comms]
    cnt = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in comms]
    n = torch.full((1,), 1000, dtype=torch.int64, device=dev)
    loss = torch.full((1,), 2500.0, dtype=torch.float64, device=dev)
    nunits = 18  # the units of llama3_1b: embedding, 16 blocks, final norm + head

    def commit(r, i, tm):
        kw = dict(gnorm="z1_gnorm", nunits=nunits, max_norm=1.0, norm=norm[r])
        if tm:
            kw.update(tokens="z1_tokmean", slot=i % 2, n_valid=n, loss_sum=loss, rows=8192, divisor=W * 8192,
                      token_out=out_[r], token_count=cnt[r])
        comms[r].zero1_commit_(gates[r], True, True, None, **kw)

    res = {"off": [], "on": []}
    for i in range(args.warmup + args.rounds):
        for name, tm in (("off", False), ("on", True)):
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for j in range(args.commits):
                for r in range(W):
                    commit(r, j, tm)
            e.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                res[name].append(s.elapsed_time(e) * 1e3 / (args.commits * W))
    return {"world": W, "clipping": True, "units": nunits,
            **{name: {"us_per_commit": stats(t)} for name, t in res.items()}}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--virtual", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--commits", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("token_mean_step.py measures on a GPU; none is visible")
    res = {"card_before": card(), "commit": commit_bench(args), "step": step_bench(args), "card_after": card()}
    print("TOKEN_MEAN_STEP " + json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
