"""Tied embeddings: a ``llama3_2_1b`` training step against its untied twin ``llama3_1b``, and the embedding backward
kernel against torch's dense embedding backward.

    python bench/tied_step.py --seq 8192 --steps 10 --warmup 3 --rounds 3

Steps: each round builds a ``FaultTolerantTrainer`` (FT-ZeRO-1, one replica) of each model in turn, runs ``--warmup``
steps, times ``--steps`` steps with CUDA events around each (the step's update joined), and records the peak allocated
memory and ``Zero1Optimizer.state_bytes_held()``. Rounds alternate the two models, so clocks and neighbours weigh on both
alike. Reported: the median and the spread (min, max) of ms per step over all timed steps, tokens/s at the median.

Kernel: ``ops.fused.embedding_bwd`` (stable sort of the ids + the two-launch in-place sum) at T tokens for d = 2048 and
3072, ids uniform over the 128256-row vocabulary and all equal, against ``aten.embedding_dense_backward`` plus the add
of its dense ``[V, d]`` result into the gradient slot, the untied model's path. CUDA events around ``--launches``
calls after 10 warm-up calls. The card's name, power limit and clocks are read in the same run.
"""

from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
from datetime import timedelta

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def time_steps(model: str, args, tag: str) -> dict:
    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    gc.collect()
    torch.cuda.empty_cache()  # the symmetric segments are plain cudaMalloc: hand them what the caching allocator holds
    lh = local_lighthouse()
    tr = None
    try:
        tr = FaultTolerantTrainer(model, loopback(lh.address()), replica_id=f"{tag}_0", timeout=timedelta(seconds=120))
        g = torch.Generator().manual_seed(0)
        V, B, S = tr.cfg.vocab_size, args.batch, args.seq
        tok = torch.randint(0, V, (B, S), generator=g).cuda()
        tgt = torch.randint(0, V, (B, S), generator=g).cuda()
        for _ in range(args.warmup):
            tr.step_device(tok, tgt)
        tr.join()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        times = []
        for _ in range(args.steps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            loss = tr.step_device(tok, tgt)
            tr.join()
            e.record()
            torch.cuda.synchronize()
            times.append(s.elapsed_time(e))
        return {"ms": times, "loss": float(loss.item()), "peak_alloc_gib": torch.cuda.max_memory_allocated() / 2**30,
                "state_bytes_held": int(tr.zopt.state_bytes_held()), "params": tr.cfg.num_params(), "tokens": B * S}
    finally:
        if tr is not None:
            tr.shutdown()
            if hasattr(tr.pg, "comm"):
                tr.pg.comm.free_segments()  # the symmetric segments are not the caching allocator's to release
        lh.shutdown()
        del tr
        gc.collect()
        torch.cuda.empty_cache()


def step_bench(args) -> dict:
    models = ("llama3_2_1b", "llama3_1b")
    runs = {m: [] for m in models}
    for r in range(args.rounds):
        for m in models:
            runs[m].append(time_steps(m, args, f"tied_bench_{r}_{m}"))
    out = {}
    for m in models:
        t = np.array([x for run in runs[m] for x in run["ms"]])
        last = runs[m][-1]
        out[m] = {"ms_median": round(float(np.median(t)), 2), "ms_min": round(float(t.min()), 2),
                  "ms_max": round(float(t.max()), 2),
                  "round_medians": [round(float(np.median(run["ms"])), 2) for run in runs[m]],
                  "tokens_per_s": round(last["tokens"] / float(np.median(t)) * 1e3, 1),
                  "peak_alloc_gib": round(max(run["peak_alloc_gib"] for run in runs[m]), 2),
                  "state_bytes_held": last["state_bytes_held"], "params": last["params"], "loss": last["loss"]}
    return out


def kernel_bench(args) -> dict:
    from torchft_b200.ops import fused

    V, T = 128256, args.tokens
    out = {}
    for d in (2048, 3072):
        g = torch.Generator(device="cuda").manual_seed(d)
        dx = torch.randn(T, d, device="cuda", generator=g).bfloat16()
        slot = torch.zeros(V, d, device="cuda", dtype=torch.bfloat16)
        for kind in ("uniform", "equal"):
            ids = (torch.randint(0, V, (T,), device="cuda", generator=g) if kind == "uniform"
                   else torch.full((T,), 1234, dtype=torch.int64, device="cuda"))

            def ours():
                fused.embedding_bwd(ids, dx, slot)

            def dense():
                slot.add_(torch.ops.aten.embedding_dense_backward(dx, ids, V, -1, False))

            res = {}
            for name, f in (("embedding_bwd", ours), ("dense_plus_add", dense)):
                for _ in range(10):
                    f()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(args.launches):
                    f()
                e.record()
                torch.cuda.synchronize()
                res[name] = round(s.elapsed_time(e) * 1e3 / args.launches, 1)  # us per call
            out[f"d{d}_{kind}"] = {"us_per_call": res, "T": T}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tied_step.py measures on a GPU; none is visible")
    res = {"card_before": card(), "kernel": kernel_bench(args)}
    if not args.skip_steps:
        res["step"] = step_bench(args)
    res["card_after"] = card()
    print("TIED_STEP " + json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
