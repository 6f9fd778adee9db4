"""Flagship benchmark: fault-tolerant Llama-3 training throughput on H100.

    python bench.py --gpus 1 --steps 5 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W

Metric: whole-job tokens/s of Llama-3 bf16 training (default ``llama3_1b``, 1.5 B parameters: its
weights, gradients and fp32 AdamW state take 24 GB, so one replica group fits one 80 GB H100; the
8B model's 128 GB of training state does not) with the
per-step fault-tolerance protocol ON (Lighthouse quorum + cross-replica gradient
reduction + commit decision + AdamW), N replica groups of one GPU each (HSDP with
shard degree 1; weak scaling: per-GPU batch fixed), synthetic tokens, random-init
weights. Every native step runs FT-ZeRO-1 (torchft_b200/parallel/zero1.py): start_quorum
(async), forward, backward with one fused reduce-scatter kernel per transformer block
overlapped, ONE device-side commit-verdict kernel (no host sync, no RPC), gated AdamW on
the held slices fused with the all-gather of the new bf16 weights under the next forward.

`value`   : device-timed (CUDA events), inputs resident on the GPU, max over ranks.
`e2e`     : same loop through the public trainer API (`FaultTolerantTrainer.step_async`),
            wall-clock, including per step the pinned-host -> device copy of tokens/targets
            and a device -> host read of the loss (pinned, read back one step late so the
            host never drains the GPU queue).
`--impl reference` : upstream torchft builds its native module with maturin + cargo/protoc;
            without them it cannot be installed -> prints {"unavailable": ...}.
`--impl nccl`      : same model/loop with the reference-EQUIVALENT structure: stock
            ProcessGroupNCCL re-created per quorum, all-reduce SUM then /N, host-synchronous
            should_commit RPC, full AdamW on every replica (reference manager.py:466-478,
            884-903, optim.py:52-55).
The native arm also runs the nccl arm afterwards IN THE SAME PROCESS (the reference publishes
no numbers) and reports `vs_baseline` = native / nccl-equivalent; `--no-baseline-arm` skips it.
`--dump-outputs DIR` : after the timed steps, rank 0 writes what the device-timed loop computed in
            its last step as float32 .npy files: `loss.npy` and `weights_sample.npy` (the updated bf16
            weights at a fixed, seeded set of positions in every parameter tensor). Inputs and weights
            are seeded, so two builds can be compared output for output.
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import threading
import time
from datetime import timedelta

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


class ClockSampler:
    """Samples SM clock + throttle reasons during the timed region (NVML, else nvidia-smi)."""

    BAD = {"hw_slowdown": 0x8, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20}
    NOTE = {"sw_power_cap": 0x4, "hw_power_brake": 0x80}

    def __init__(self, index: int) -> None:
        self.index = index
        self.sm: list = []
        self.reasons: set = set()
        self.max_mhz = 0
        self._stop = threading.Event()
        self._t: threading.Thread | None = None
        self._h = None
        try:
            import pynvml

            pynvml.nvmlInit()
            self._nv = pynvml
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[index]) if vis and vis.split(",")[index].isdigit() else index
            self._h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self._nv = None

    def _run(self) -> None:
        while not self._stop.is_set():
            try:
                if self._nv is not None and self._h is not None:
                    self.sm.append(self._nv.nvmlDeviceGetClockInfo(self._h, self._nv.NVML_CLOCK_SM))
                    mask = self._nv.nvmlDeviceGetCurrentClocksEventReasons(self._h)
                    for k, bit in {**self.BAD, **self.NOTE}.items():
                        if mask & bit:
                            self.reasons.add(k)
            except Exception:
                pass
            self._stop.wait(0.2)

    def start(self) -> None:
        self._stop.clear()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def stop(self) -> dict:
        self._stop.set()
        if self._t is not None:
            self._t.join(timeout=2)
        out = {
            "sm_mhz": int(statistics.median(self.sm)) if self.sm else None,
            "sm_max_mhz": int(self.max_mhz) if self.max_mhz else None,
            "reasons": sorted(self.reasons),
            "samples": len(self.sm),
        }
        if not self.sm:  # NVML unavailable: one nvidia-smi sample
            try:
                import subprocess

                q = subprocess.run(["nvidia-smi", f"--id={self.index}", "--query-gpu=clocks.sm,clocks.max.sm",
                                    "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
                a, b = q.stdout.strip().split(",")
                out.update(sm_mhz=int(a), sm_max_mhz=int(b), samples=1)
            except Exception:
                pass
        return out


def _sample_outputs(trainer, loss) -> dict:
    """Host copies of the last step's loss and of the updated weights at seeded positions: up to 16384 elements of
    every parameter tensor, in the trainer's fixed parameter order (16384 x 4 B x ~150 tensors of Llama-3 ~ 10 MB)."""
    import numpy as np
    import torch

    gen = torch.Generator().manual_seed(0)
    parts = []
    for p in trainer.flat.params:
        flat = p.detach().reshape(-1)
        idx = torch.randint(0, flat.numel(), (16384,), generator=gen).sort().values if flat.numel() > 16384 else None
        parts.append((flat if idx is None else flat[idx.to(flat.device)]).float().cpu())
    return {"loss": np.asarray([float(loss.item())], dtype=np.float32),
            "weights_sample": torch.cat(parts).numpy().astype(np.float32)}


def run_arm(impl: str, args, rank: int, world: int, local: int, lh_addr: str) -> dict:
    """Build a trainer for ``impl``, warm up, time K steps on the device and K steps end to end, tear down."""
    import gc

    import torch
    import torch.distributed as dist

    from torchft_b200.ops import _native
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    dev = torch.device("cuda", local)
    backend = "b200" if impl == "native" else "nccl"

    def build(ac):
        if args.shards > 1:
            from torchft_b200.parallel.hsdp import HSDPTrainer

            return HSDPTrainer(args.model, lh_addr, args.shards, backend=backend, timeout=timedelta(seconds=120), device=dev,
                               replica_prefix=impl)
        return FaultTolerantTrainer(args.model, lh_addr, replica_id=f"{impl}_{rank}", min_replica_size=world,
                                    backend=backend, bucket_mb=args.bucket_mb, should_quantize=args.quantize,
                                    activation_checkpoint=ac, timeout=timedelta(seconds=120), device=dev,
                                    replication=args.replication)

    ac = args.ac
    trainer = build(ac)
    cfg = trainer.cfg
    B, S = args.batch, args.seq
    gen = torch.Generator().manual_seed(1234 + rank)
    tok_cpu = torch.randint(0, cfg.vocab_size, (B, S), generator=gen).pin_memory()
    tgt_cpu = torch.randint(0, cfg.vocab_size, (B, S), generator=gen).pin_memory()
    tok = tok_cpu.to(dev)
    tgt = tgt_cpu.to(dev)

    def barrier() -> None:
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    warmup = max(args.warmup, 3)
    # ---- warm-up (untimed); falls back to full activation checkpointing on OOM ----
    try:
        for _ in range(warmup):
            trainer.step_device(tok, tgt)
        torch.cuda.synchronize()
    except torch.OutOfMemoryError:
        if ac == "full":
            raise
        trainer.shutdown()
        if hasattr(trainer.pg, "comm"):
            trainer.pg.comm.free_segments()
        del trainer
        gc.collect()
        torch.cuda.empty_cache()
        ac = "full"
        trainer = build(ac)
        for _ in range(warmup):
            trainer.step_device(tok, tgt)
        torch.cuda.synchronize()

    sampler = ClockSampler(local)
    # ---- phase A: device-timed, inputs resident on the GPU ----
    barrier()
    launches0 = _native.kernel_launches()
    sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        loss = trainer.step_device(tok, tgt)
    trainer.join()  # the last step's optimizer update / weight all-gather (side stream) is inside the timed region
    ev1.record()
    barrier()
    clocks = sampler.stop()
    launches = _native.kernel_launches() - launches0
    dev_ms = ev0.elapsed_time(ev1) / args.steps
    loss_v = float(loss.item())
    outputs = _sample_outputs(trainer, loss) if args.dump_outputs and rank == 0 else None
    committed = trainer.manager.current_step()

    # ---- phase B: end to end through the public API (H2D inputs + D2H loss every step) ----
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        trainer.step_async(tok_cpu, tgt_cpu)
    loss_e2e = trainer.last_loss()  # the last step's loss has reached the host
    barrier()  # device-wide synchronize: the last update is inside the timed region too
    e2e_ms = (time.perf_counter() - t0) * 1e3 / args.steps
    committed_total = trainer.manager.current_step()

    t = torch.tensor([dev_ms, e2e_ms], dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, e2e_ms = float(t[0]), float(t[1])
    out = {
        "impl": impl, "dev_ms": dev_ms, "e2e_ms": e2e_ms, "launches": int(launches), "clocks": clocks,
        "loss": loss_v, "loss_e2e": loss_e2e, "committed": int(committed), "committed_total": int(committed_total),
        "peak_gib": torch.cuda.max_memory_allocated() / 2**30, "ac": ac or cfg.activation_checkpoint,
        "warmup": warmup, "cfg": cfg, "h2d": int(tok_cpu.numel() * 8 + tgt_cpu.numel() * 8),
        "zero1": bool(getattr(trainer, "zero1", False)),
        "state_gib": (trainer.zopt.state_bytes_held() / 2**30) if getattr(trainer, "zopt", None) is not None else None,
        "outputs": outputs,
    }
    trainer.shutdown()
    barrier()  # every peer has unmapped our segments
    if hasattr(trainer.pg, "comm"):
        trainer.pg.comm.free_segments()
    del trainer, tok, tgt
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference", "nccl"])
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=1, help="sequences per GPU per step")
    ap.add_argument("--bucket-mb", type=float, default=512.0)
    ap.add_argument("--quantize", action="store_true")
    ap.add_argument("--replication", type=int, default=2, help="FT-ZeRO-1: holders per slice of optimizer state")
    ap.add_argument("--shards", type=int, default=1,
                    help="FSDP2 shard degree INSIDE a replica group (--gpus 8 --shards 2 = 4 groups x 2 shards); default 1 = "
                         "every GPU is a replica group holding the full model")
    ap.add_argument("--ac", default=None, help="activation checkpointing: none|full (default: auto)")
    ap.add_argument("--no-baseline-arm", action="store_true",
                    help="native arm only: skip the in-process run of the reference-equivalent NCCL arm")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's loss and a seeded sample of the updated weights as DIR/<name>.npy")
    ap.add_argument("--config", default="hsdp", choices=["hsdp", "diloco", "heal"],
                    help="hsdp (default: the flagship step), diloco (Llama-3 DiLoCo, outer step every "
                         "100, fused fp8 outer all-reduce; launch under torchrun), heal (kill a replica group at step 50, "
                         "rejoin at 80; launch WITHOUT torchrun, it spawns one process per GPU)")
    args, extra = ap.parse_known_args()

    if args.config != "hsdp":
        import runpy

        script = {"diloco": "diloco_bench.py", "heal": "heal_bench.py"}[args.config]
        if args.config == "diloco":
            argv = ["--model", args.model, "--seq", str(args.seq), "--sync-every", "100", "--outer-steps", "1",
                    "--out", os.path.join(tempfile.gettempdir(), "bench_diloco.json")] + (["--quantize"] if args.quantize or "--no-quantize" not in extra else [])
        else:
            argv = ["--gpus", str(args.gpus), "--model", args.model, "--seq", str(args.seq), "--kill-at", "50", "--rejoin-at", "80",
                    "--steps", "100", "--out", os.path.join(tempfile.gettempdir(), "bench_heal.json")]
        argv += [x for x in extra if x != "--no-quantize"]
        sys.argv = [os.path.join(ROOT, "bench", script)] + argv
        runpy.run_path(sys.argv[0], run_name="__main__")
        return

    if args.impl == "reference":
        if int(os.environ.get("RANK", "0")) != 0:  # under torchrun only rank 0 reports
            return
        print(json.dumps({
            "impl": "reference",
            "unavailable": "upstream torchft's build backend (maturin) and its toolchain (cargo/rustc, protoc) are not "
                           "installed, so it cannot be built here (see DESIGN.md)",
        }))
        return

    import torch
    import torch.distributed as dist

    if args.dump_outputs and args.shards > 1:
        ap.error("--dump-outputs needs --shards 1")
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    assert world == args.gpus or world == 1, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    torch.cuda.set_device(local)

    from torchft_b200.coordination import LighthouseServer

    # bootstrap only (publish the lighthouse address, reduce timings): gloo on CPU
    lighthouse = None
    assert world % args.shards == 0, "--shards must divide the number of GPUs"
    if world > 1:
        if args.shards > 1:  # FSDP's intra-group collectives need NCCL; everything else here only uses the CPU side
            dist.init_process_group("cpu:gloo,cuda:nccl", timeout=timedelta(seconds=300), device_id=torch.device("cuda", local))
        else:
            dist.init_process_group("gloo", timeout=timedelta(seconds=300))
        if rank == 0:
            lighthouse = LighthouseServer(bind="[::]:0", min_replicas=world // args.shards, join_timeout_ms=60000)
            addr = [lighthouse.address()]
        else:
            addr = [None]
        dist.broadcast_object_list(addr, src=0)
        lh_addr = addr[0]
    else:
        lighthouse = LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=100)
        lh_addr = lighthouse.address()
    host = lh_addr.split("//")[1].rsplit(":", 1)[0]
    lh_addr = lh_addr.replace(host, "127.0.0.1")

    res = run_arm(args.impl, args, rank, world, local, lh_addr)
    base = None
    if args.impl == "native" and not args.no_baseline_arm:
        try:
            base = run_arm("nccl", args, rank, world, local, lh_addr)
        except Exception as e:  # noqa: BLE001 - the headline must not depend on the comparison arm
            base = {"error": f"{type(e).__name__}: {e}"}

    cfg = res["cfg"]
    B, S = args.batch, args.seq
    tokens = B * S * world
    value = tokens / res["dev_ms"] * 1e3
    e2e_value = tokens / res["e2e_ms"] * 1e3
    flops = cfg.flops_per_token(S) * B * S  # per GPU per step

    if rank == 0:
        native = args.impl == "native"
        out = {
            "metric": f"tokens/sec (whole job, {args.model} fault-tolerant training step, bf16)",
            "value": round(value, 1),
            "unit": "tokens/s",
            "n_gpus": world,
            "steps": args.steps,
            "warmup": res["warmup"],
            "ms_per_step": round(res["dev_ms"], 2),
            "higher_is_better": True,
            "scaling": "weak",
            "vs_baseline": None,
            "dtype": "bf16",
            "data": "synthetic tokens (uniform random ids), random-init weights",
            "impl": "torchft_b200" if native else "nccl-equivalent-baseline (stock ProcessGroupNCCL data plane)",
            "config": {
                "model": args.model,
                "params_b": round(cfg.num_params() / 1e9, 3),
                "global_batch": B * world,
                "seq_len": S,
                "parallelism": (f"ft-hsdp: {world // args.shards} replica groups x {args.shards}-GPU FSDP2 shards (cross-replica "
                                f"all-reduce of every reduce-scattered shard through ManagedProcessGroup)") if args.shards > 1 else
                               (f"ft-ddp over {world} replica group(s) x 1 GPU (HSDP shard degree 1)"
                                + (f" + FT-ZeRO-1: optimizer state partitioned over the replicas, k={min(args.replication, world)} holders per slice"
                                   if res["zero1"] else "")),
                "optimizer": ("AdamW (fp32 master/m/v) on the held 1/N slices, gated by the device-side commit verdict, fused with the "
                              "all-gather of the new bf16 weights; one launch per transformer block under the next forward") if res["zero1"]
                             else ("torch AdamW (fused) on FSDP2 fp32 parameter shards, applied only after should_commit" if args.shards > 1
                                   else "AdamW (fp32 master/m/v), full on every replica, applied only after the host-synchronous should_commit"),
                "activation_checkpoint": res["ac"],
                "grad_reduction": ("fused reduce-scatter kernel per block over NVLink peer memory (1/N scale, bf16 cast, zero "
                                   "contribution, buddy push), zero-copy symmetric buffers, overlapped with backward") if res["zero1"]
                                  else ("fused P2P all-reduce" if native else "NCCL allreduce SUM + div"),
                "commit": "device-side verdict kernel, host learns lazily (no stream sync, no RPC per step)" if res["zero1"]
                          else "host stream synchronize + should_commit RPC per step",
                "quantized_allreduce": bool(args.quantize),
                "l2_policy": (f"inputs larger than L2 ({cfg.num_params() * 2 / 1e9:.0f} GB of weights + as many of gradients "
                              "stream through every step)"),
                "ft_protocol_per_step": "start_quorum(async, C++ control plane) + commit decision, in the timed region",
            },
            "e2e": {
                "value": round(e2e_value, 1),
                "unit": "tokens/s",
                "ms_per_step": round(res["e2e_ms"], 2),
                "h2d_bytes_per_step": res["h2d"],
                "d2h_bytes_per_step": 4,
                "timing": "host wall clock between barriers, max over ranks; loss read back from pinned memory one step late",
            },
            "gpu_launches": res["launches"],
            "clocks": res["clocks"],
            "model_tflops_per_gpu": round(flops / res["dev_ms"] / 1e9, 1),
            "peak_mem_gib": round(res["peak_gib"], 1),
            "optimizer_state_gib_held": None if res["state_gib"] is None else round(res["state_gib"], 1),
            "loss": round(res["loss"], 4),
            "steps_committed": res["committed"],
            "steps_committed_incl_e2e": res["committed_total"],
        }
        if base is not None:
            if "error" in base:
                out["baseline_arm"] = base
            else:
                bval = tokens / base["dev_ms"] * 1e3
                out["vs_baseline"] = round(value / bval, 4)
                out["baseline_arm"] = {
                    "what": "reference-equivalent arm run in this same process right after the native arm (the reference "
                            "publishes no number and cannot be installed offline): stock ProcessGroupNCCL, allreduce SUM + /N, "
                            "host-synchronous should_commit RPC, full AdamW per replica",
                    "value": round(bval, 1), "ms_per_step": round(base["dev_ms"], 2),
                    "e2e_value": round(tokens / base["e2e_ms"] * 1e3, 1), "e2e_ms_per_step": round(base["e2e_ms"], 2),
                    "e2e_ratio": round(base["e2e_ms"] / res["e2e_ms"], 4),
                    "clocks": base["clocks"], "peak_mem_gib": round(base["peak_gib"], 1), "loss": round(base["loss"], 4),
                }
        print(json.dumps(out), flush=True)
        if args.dump_outputs:
            import numpy as np

            os.makedirs(args.dump_outputs, exist_ok=True)
            for name, arr in res["outputs"].items():
                np.save(os.path.join(args.dump_outputs, f"{name}.npy"), arr)

    if world > 1:
        dist.barrier()  # every rank is done with the lighthouse before rank 0 stops it
    if lighthouse is not None:
        lighthouse.shutdown()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
