"""Does one rank of FT-ZeRO-1 with compact optimizer state fit a full training step of a model on one GPU?

One real rank of a W-rank quorum runs on this GPU; the other W - 1 ranks are aliases of it
(``SymmetricComm.virtual_world(..., alias=True)``), so only rank 0's buffers exist. Rank 0 holds the slices a rank of
a W-rank quorum holds, in page pools sized for every quorum from ``--min-world`` to 8 (``zero1.pool_pages``). The script
drives the re-shard of the first quorum (every aliased peer has published ``t = 0``), then runs forward, backward, the
per-unit reduce-scatter, the device commit and the paged update for a few steps, and reports peak device memory:
``cudaMemGetInfo`` (the symmetric segments live outside torch's allocator) and torch's own peaks next to it.

It tries ``--seq`` first without and then with activation checkpointing, and halves the sequence length until a step
fits; every attempt runs in a fresh process and records the device's free memory before it starts (``cudaMemGetInfo``
sees the whole device, so memory other processes hold counts against the attempt). Step times come from the aliased peers' buffers in local HBM, not from NVLink, and are not multi-GPU step times.

    python bench/zero1_fit.py --model llama3_8b --world 8 --min-world 7 --replication 2 --seq 8192 [--moments bf16]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.models.llama import CONFIGS, FlatParams, Llama  # noqa: E402
from torchft_b200.parallel.symm_mem import SymmetricComm  # noqa: E402
from torchft_b200.parallel.trainer import FaultTolerantTrainer  # noqa: E402
from torchft_b200.parallel.zero1 import Zero1Optimizer  # noqa: E402


class _AliasedGroup:
    """What ``Zero1Optimizer`` needs of a process group, over a virtual world whose peers alias rank 0: a segment
    allocated here exists once and every peer entry points at it."""

    def __init__(self, comms):
        self.comms = comms
        self.comm = comms[0]
        self.comm_stream = torch.cuda.current_stream()

    def alloc_symmetric(self, name, nbytes):
        return SymmetricComm.virtual_alloc(self.comms, name, nbytes)

    def add_configure_hook(self, fn):
        pass


def _card():
    out = {}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,memory.total,memory.used",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["gpu"], out["power_limit"], out["memory_total"], out["memory_used_before"] = [
            x.strip() for x in q.stdout.strip().split(",")]
    except Exception as e:  # noqa: BLE001
        out["error"] = repr(e)
    return out


def _used():
    free, total = torch.cuda.mem_get_info()
    return total - free


def attempt(args, seq, ckpt):
    """Build the rank, run ``args.steps`` steps at ``seq``; returns the measurements (raises on out-of-memory)."""
    import dataclasses

    cfg = dataclasses.replace(CONFIGS[args.model], activation_checkpoint=ckpt, max_seq_len=max(seq, 1))
    dev = torch.device("cuda", 0)
    torch.cuda.reset_peak_memory_stats()
    free0, _ = torch.cuda.mem_get_info()
    base = _used()
    comms = SymmetricComm.virtual_world(args.world, {}, device=dev, presignal=True, alias=True)
    try:
        res = _run(args, cfg, seq, ckpt, dev, base, comms)
        res["device_free_before_gib"] = round(free0 / 2**30, 2)
        return res
    finally:  # the segments live outside torch's allocator: give them back before the next attempt
        torch.cuda.synchronize()
        for c in comms:
            c.shutdown()
        for c in comms:
            c.free_segments()


def _run(args, cfg, seq, ckpt, dev, base, comms):
    from torch.distributed import HashStore

    pg = _AliasedGroup(comms)
    model = Llama(cfg, device="meta")
    numel = sum((p.numel() + FlatParams.ALIGN - 1) // FlatParams.ALIGN * FlatParams.ALIGN for p in model.parameters())
    opt = Zero1Optimizer(pg, numel, replication=args.replication, compact=True, min_world=args.min_world,
                         moment_dtype={"fp32": torch.float32, "bf16": torch.bfloat16}[args.moments])
    flat = FlatParams(model, grad_alloc=lambda n: opt.grad, device=dev, param_alloc=lambda n: opt.param)
    model.init_weights(0)
    units = FaultTolerantTrainer._compute_stage_ranges(SimpleNamespace(flat=flat, model=model))
    opt.set_units(units)
    opt.seed_master()
    store = HashStore()
    for r in range(1, args.world):  # the aliased peers: fresh replicas at t = 0
        store.set(f"z1/{r}", json.dumps({"t": 0, "hold": [], "pages": []}))
    store.add("z1/pulled", args.world - 1)
    opt._on_configured(store, 0, args.world, 1)
    torch.cuda.synchronize()
    after_setup = _used()
    gen = torch.Generator(device=dev).manual_seed(0)
    tok = torch.randint(0, cfg.vocab_size, (args.batch, seq), device=dev, generator=gen)
    tgt = torch.randint(0, cfg.vocab_size, (args.batch, seq), device=dev, generator=gen)
    peak_used, times = after_setup, []
    for step in range(args.steps):
        t0 = time.perf_counter()
        flat.reset_grads()
        loss = model(tok, tgt)
        peak_used = max(peak_used, _used())
        loss.backward()
        for p in flat.params:
            flat.adopt_grad(p)
        peak_used = max(peak_used, _used())
        for lo, hi in opt.layout.units:
            comms[0].zero1_reduce_scatter_("z1_grad", lo * 2, hi - lo, 1.0 / args.world, True, opt.layout.replication, 128)
        seq_no = opt.enqueue(True)
        opt.update()
        torch.cuda.synchronize()
        opt.resolved(opt.wait(seq_no))
        times.append((time.perf_counter() - t0) * 1e3)
        # torch may have released cached blocks it no longer needs: add back what it held at its peak
        peak_used = max(peak_used, _used() + torch.cuda.max_memory_reserved() - torch.cuda.memory_reserved())
        del loss
    assert opt.t == args.steps and opt.lost_elements == 0
    res = {
        "model": args.model, "world": args.world, "min_world": args.min_world, "replication": opt.layout.replication,
        "seq": seq, "batch": args.batch, "activation_checkpoint": ckpt, "moments": args.moments,
        "pool_pages": opt.capacity, "state_gib_allocated": round(opt.state_bytes_allocated() / 2**30, 2),
        "state_gib_held": round(opt.state_bytes_held() / 2**30, 2),
        "device_used_before_gib": round(base / 2**30, 2),
        "device_used_after_setup_gib": round(after_setup / 2**30, 2),
        "device_peak_gib": round(peak_used / 2**30, 2),
        "torch_max_allocated_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
        "torch_max_reserved_gib": round(torch.cuda.max_memory_reserved() / 2**30, 2),
        "step_ms_local_hbm_not_nvlink": [round(t, 1) for t in times],
    }
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_8b", choices=sorted(CONFIGS))
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--min-world", type=int, default=7)
    ap.add_argument("--replication", type=int, default=2)
    ap.add_argument("--moments", default="fp32", choices=["fp32", "bf16"], help="type of the AdamW moments m and v")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--min-seq", type=int, default=512)
    ap.add_argument("--out", default="")
    ap.add_argument("--one", default="", help=argparse.SUPPRESS)  # "SEQ,CKPT": run one attempt in this process
    a = ap.parse_args()
    if a.one:
        seq, ckpt = a.one.split(",")
        torch.cuda.set_device(0)
        free0, _ = torch.cuda.mem_get_info()
        try:
            r = attempt(a, int(seq), ckpt)
        except torch.cuda.OutOfMemoryError as e:
            r = {"seq": int(seq), "activation_checkpoint": ckpt, "device_free_before_gib": round(free0 / 2**30, 2),
                 "out_of_memory": str(e).splitlines()[0]}
        print("ZERO1_ATTEMPT " + json.dumps(r), flush=True)
        return
    report = {"card": _card(), "attempts": []}
    seq, fit = a.seq, None
    while seq >= a.min_seq and fit is None:
        for ckpt in ("none", "full"):
            # every attempt in a fresh process: nothing an earlier (failed) attempt allocated can count against it
            cmd = [sys.executable, os.path.abspath(__file__), "--one", f"{seq},{ckpt}"] + [
                f"--{k.replace('_', '-')}={v}" for k, v in vars(a).items() if k not in ("one", "out")]
            out = subprocess.run(cmd, capture_output=True, text=True)
            line = [x for x in out.stdout.splitlines() if x.startswith("ZERO1_ATTEMPT ")]
            r = json.loads(line[-1].split(" ", 1)[1]) if line else {
                "seq": seq, "activation_checkpoint": ckpt, "failed": (out.stderr or out.stdout).strip().splitlines()[-1:]}
            report["attempts"].append(r)
            if "device_peak_gib" in r:
                fit = r
                break
        seq //= 2
    report["fits_at_requested_seq"] = fit is not None and fit["seq"] == a.seq
    report["largest_fitting"] = None if fit is None else {"seq": fit["seq"], "activation_checkpoint": fit["activation_checkpoint"],
                                                          "device_peak_gib": fit["device_peak_gib"]}
    print("ZERO1_FIT " + json.dumps(report), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
