"""Single-GPU training-step timing/memory probe for the Llama configs (no FT plumbing).

    python bench/model_step.py --model llama3_1b --seq 8192 --batch 1 --steps 5

Used to size the flagship benchmark (do the model's weights + AdamW state + activations fit in
the 80 GB of an H100, what does a step cost, where does the time go).
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.models.llama import CONFIGS, FlatParams, Llama  # noqa: E402
from torchft_b200.ops.fused import FlatAdamW  # noqa: E402


def run(args, ac: str) -> dict:
    import dataclasses

    cfg = dataclasses.replace(CONFIGS[args.model], activation_checkpoint=ac)
    dev = torch.device("cuda")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    model = Llama(cfg, device=dev)
    model.init_weights(0)
    flat = FlatParams(model)
    opt = FlatAdamW(flat.param, flat.grad, lr=3e-4)
    torch.cuda.synchronize()
    init_s = time.perf_counter() - t0
    mem_state = torch.cuda.memory_allocated() / 2**30
    tok = torch.randint(0, cfg.vocab_size, (args.batch, args.seq), device=dev)
    tgt = torch.randint(0, cfg.vocab_size, (args.batch, args.seq), device=dev)
    times = []
    loss_v = None
    for i in range(args.warmup + args.steps):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        opt.zero_grad()
        loss = model(tok, tgt)
        loss.backward()
        opt.step()
        e.record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            times.append(s.elapsed_time(e))
        loss_v = float(loss.item())
    ms = sum(times) / len(times)
    toks = args.batch * args.seq
    flops = cfg.flops_per_token(args.seq) * toks
    return {
        "model": args.model, "ac": ac, "seq": args.seq, "batch": args.batch, "params_b": cfg.num_params() / 1e9,
        "ms_per_step": round(ms, 2), "tokens_per_s": round(toks / ms * 1e3, 1),
        "tflops": round(flops / ms / 1e9, 1), "loss": loss_v, "init_s": round(init_s, 1),
        "state_gib": round(mem_state, 1), "peak_gib": round(torch.cuda.max_memory_allocated() / 2**30, 1),
        "times_ms": [round(t, 1) for t in times],
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ac", default="none")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    try:
        res = run(args, args.ac)
    except torch.OutOfMemoryError as e:
        print("OOM with ac=%s: %s" % (args.ac, str(e)[:200]), flush=True)
        torch.cuda.empty_cache()
        res = run(args, "full")
    print("MODEL_STEP " + json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
