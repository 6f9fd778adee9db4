"""Packed documents against plain rows: one training step of a Llama config (FlatParams + FlatAdamW, no FT plumbing),
and attention alone.

    python bench/packed_step.py --model llama3_1b --seq 8192 --batch 1 --steps 10 --warmup 3

In one process, step by step in turn (so that clocks and neighbours weigh on every arm alike), on the same tokens:

* ``unpacked``: every row is one causal sequence (SDPA);
* ``packed``: the row cut into documents whose lengths are drawn from a log-normal with a median of 600 tokens and
  sigma 1.2 (seed 0), the shape of web-text corpora, where most documents hold a few hundred to a few thousand tokens
  and a long tail reaches the row length; lengths are capped at the row;
* ``one_per_row``: the packed path with one document per row (the cost of the variable-length kernel itself).

Then attention alone, forward + backward: SDPA causal against ``varlen_attn`` at one document per row, 32 query heads
over 8 KV heads at D = 64 and 128. The card's name, power limit and clocks are read in the same run. With
``--profile`` one unpacked step runs under ``torch.profiler`` first and the attention kernels it launched are listed
(which library backend SDPA picked).
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.data import pack_documents  # noqa: E402
from torchft_b200.models.llama import CONFIGS, FlatParams, Llama  # noqa: E402
from torchft_b200.ops.fused import FlatAdamW  # noqa: E402


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def packed_batch(vocab: int, B: int, S: int, seed: int = 0):
    """(tokens, targets, cu_seqlens) of documents with log-normal lengths (median 600, sigma 1.2), capped at S."""
    rng = np.random.default_rng(seed)
    docs, n = [], 0
    while n < B * S:
        L = int(min(S, max(1, round(rng.lognormal(np.log(600.0), 1.2)))))
        docs.append(rng.integers(0, vocab, size=L))
        n += L
    return next(pack_documents(docs, B, S))


def attention_flops(cu: torch.Tensor, cfg) -> float:
    """Causal attention FLOPs of a training step over the documents of ``cu``, counted as
    ``LlamaConfig.flops_per_token`` counts them (QK^T and PV, 3x the forward), with sum L_i^2 / 2 in place of S^2 / 2."""
    L = np.diff(cu.numpy().astype(np.int64)).astype(np.float64)
    return float(cfg.n_layers * 3.0 * 2 * 2 * cfg.dim * (L * L / 2).sum())


def step_bench(args) -> dict:
    import dataclasses

    cfg = dataclasses.replace(CONFIGS[args.model], activation_checkpoint=args.ac)
    dev = torch.device("cuda")
    model = Llama(cfg, device=dev)
    model.init_weights(0)
    flat = FlatParams(model)
    opt = FlatAdamW(flat.param, flat.grad, lr=3e-4)
    B, S = args.batch, args.seq
    tok_p, tgt_p, cu_p = packed_batch(cfg.vocab_size, B, S)
    tok, tgt = tok_p.to(dev), tgt_p.to(dev)
    rows = torch.arange(0, B * S + 1, S, dtype=torch.int32)
    arms = {"unpacked": None, "packed": cu_p, "one_per_row": rows}
    times = {a: [] for a in arms}
    losses = {}

    def one(cu):
        opt.zero_grad()
        loss = model(tok, tgt, cu_seqlens=cu)
        loss.backward()
        opt.step()
        return loss

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        one(None)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            one(None)
            torch.cuda.synchronize()
        names = sorted({e.key for e in prof.key_averages() if any(
            s in e.key.lower() for s in ("flash", "fmha", "cudnn", "attn", "attention", "sdpa"))})
        print("SDPA_KERNELS " + json.dumps(names), flush=True)
    for i in range(args.warmup + args.steps):
        for name, cu in arms.items():
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            loss = one(cu)
            e.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[name].append(s.elapsed_time(e))
            losses[name] = float(loss.item())
    L = np.diff(cu_p.numpy().astype(np.int64))
    out = {"model": args.model, "seq": S, "batch": B, "ac": args.ac, "documents": int(L.size),
           "doc_len_median": float(np.median(L)), "doc_len_max": int(L.max()),
           "attn_flops_packed_over_unpacked": attention_flops(cu_p, cfg) / attention_flops(rows, cfg)}
    for name in arms:
        t = np.array(times[name])
        out[name] = {"ms_per_step": round(float(t.mean()), 2), "ms_min": round(float(t.min()), 2),
                     "ms_max": round(float(t.max()), 2), "tokens_per_s": round(B * S / t.mean() * 1e3, 1),
                     "loss": losses[name]}
    return out


def attention_bench(args) -> dict:
    from torch.nn.attention.varlen import varlen_attn

    B, S, Hq, Hkv = args.batch, args.seq, 32, 8
    T = B * S
    out = {}
    for D in (64, 128):
        g = torch.Generator(device="cuda").manual_seed(D)
        qkv = torch.randn(T, (Hq + 2 * Hkv) * D, device="cuda", generator=g).bfloat16().requires_grad_()
        do = torch.randn(T, Hq, D, device="cuda", generator=g).bfloat16()
        cu = torch.arange(0, T + 1, S, dtype=torch.int32, device="cuda")

        def sdpa():
            x = qkv.view(B, S, Hq + 2 * Hkv, D).transpose(1, 2)
            o = torch.nn.functional.scaled_dot_product_attention(x[:, :Hq], x[:, Hq:Hq + Hkv], x[:, Hq + Hkv:],
                                                                 is_causal=True, enable_gqa=True)
            o.transpose(1, 2).backward(do.view(B, S, Hq, D))

        def varlen():
            q = qkv[:, :Hq * D].view(T, Hq, D)
            k = qkv[:, Hq * D:(Hq + Hkv) * D].view(T, Hkv, D)
            v = qkv[:, (Hq + Hkv) * D:].view(T, Hkv, D)
            varlen_attn(q, k, v, cu, cu, S, S, window_size=(-1, 0)).backward(do)

        fns = {"sdpa_causal": sdpa, "varlen_one_per_row": varlen}
        res = {n: [] for n in fns}
        for i in range(args.warmup + 20):
            for n, f in fns.items():
                qkv.grad = None
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(5):
                    f()
                e.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    res[n].append(s.elapsed_time(e) / 5)
        flops = 3.5 * 2 * 2 * B * Hq * D * S * S / 2  # fwd 2 GEMMs, bwd 5 GEMMs, causal half
        out[f"D{D}"] = {n: {"ms_fwd_bwd": round(float(np.mean(t)), 3),
                            "tflops": round(flops / float(np.mean(t)) / 1e9, 1)} for n, t in res.items()}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ac", default="none")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("packed_step.py measures on a GPU; none is visible")
    res = {"card_before": card(), "step": step_bench(args), "attention": attention_bench(args), "card_after": card()}
    print("PACKED_STEP " + json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
