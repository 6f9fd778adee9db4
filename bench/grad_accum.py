"""FT-ZeRO-1 gradient accumulation: trainer throughput at M = 1, 2, 4 micro-batches per step on one GPU.

    python bench/grad_accum.py --model llama3_1b --seq 8192 --micro-batch 1 --accum 1 2 4 --steps 6 --repeats 2

Every arm runs the same micro-batch shape; a step of M micro-batches processes ``M * micro_batch * seq`` tokens. One
trainer is built with the largest M (so its accumulator exists) and the arms alternate between timed windows by
setting the step's micro-batch count; at M = 1 the accumulator is simply unused and every launch is the plain
pipeline's. At world 1 the cost of accumulating is the accumulate pass of each micro-batch (read the bf16 gradient,
read-modify-write the fp32 accumulator) on the comm stream under backward; this measures how much of it stays exposed.

Prints one ``GRAD_ACCUM {json}`` line with tok/s and step time per arm (median and spread over ``--repeats``), the
accumulator's bytes, the device memory peak, and the card's name and power limit.
"""

from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time
from datetime import timedelta

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--micro-batch", type=int, default=1)
    ap.add_argument("--accum", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--steps", type=int, default=6, help="timed steps per arm and repeat")
    ap.add_argument("--warmup", type=int, default=2, help="untimed steps per arm before each timed window")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--ac", default=None, help="activation checkpointing (default: the model config's; 'full' on OOM)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.parallel.trainer import FaultTolerantTrainer
    from zero1_bench import gpu_info  # noqa: E402 - bench/ is the script's directory

    torch.cuda.set_device(0)
    lh = local_lighthouse()
    M_max = max(a.accum)

    def build(ac):
        return FaultTolerantTrainer(a.model, loopback(lh.address()), replica_id="gacc_0", activation_checkpoint=ac,
                                    timeout=timedelta(seconds=120), grad_accum_steps=M_max)

    ac = a.ac
    tr = build(ac)
    cfg = tr.cfg
    gen = torch.Generator().manual_seed(1234)
    B, S = a.micro_batch * M_max, a.seq
    tok = torch.randint(0, cfg.vocab_size, (B, S), generator=gen).to("cuda")
    tgt = torch.randint(0, cfg.vocab_size, (B, S), generator=gen).to("cuda")

    def set_m(m):
        tr.grad_accum_steps = m
        tr.zopt.grad_accum_steps = m

    def window(m, steps):
        set_m(m)
        n = a.micro_batch * m
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            loss = tr.step_device(tok[:n], tgt[:n])
        tr.join()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / max(steps, 1), float(loss.detach())

    try:
        for m in sorted(a.accum, reverse=True):
            window(m, a.warmup)
    except torch.OutOfMemoryError:
        if ac == "full":
            raise
        tr.shutdown()
        tr.pg.comm.free_segments()
        del tr
        gc.collect()
        torch.cuda.empty_cache()
        ac = "full"
        tr = build(ac)
        for m in sorted(a.accum, reverse=True):
            window(m, a.warmup)
    torch.cuda.reset_peak_memory_stats()
    times = {m: [] for m in a.accum}
    losses = {}
    for _ in range(a.repeats):
        for m in a.accum:
            window(m, a.warmup)
            ms, losses[m] = window(m, a.steps)
            times[m].append(ms)
    res = {"model": a.model, "seq": S, "micro_batch": a.micro_batch, "ac": ac or cfg.activation_checkpoint,
           "accum_bytes": tr.zopt.accum_bytes(), "peak_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
           "committed": tr.manager.current_step(), "arms": {}}
    for m, ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        res["arms"][f"M{m}"] = {"step_ms": {"median": round(med, 2), "min": round(ts[0], 2), "max": round(ts[-1], 2)},
                                "tok_s": round(a.micro_batch * m * S / med * 1e3, 1), "loss": losses[m]}
    m0 = min(a.accum)
    base = res["arms"][f"M{m0}"]["tok_s"]
    for m in a.accum:
        res["arms"][f"M{m}"][f"tok_s_over_M{m0}"] = round(res["arms"][f"M{m}"]["tok_s"] / base, 4)
    res.update(gpu_info())
    print("GRAD_ACCUM " + json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    tr.shutdown()
    lh.shutdown()


if __name__ == "__main__":
    main()
