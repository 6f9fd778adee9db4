"""DiLoCo throughput + outer-sync cost (BASELINE.md config 3, scaled to fit next to the optimizer state).

    torchrun --nproc-per-node N bench/diloco_bench.py --model llama3_1b --sync-every 20 --outer-steps 3 [--quantize]

Each rank is a replica group (1 GPU). Inner loop: plain AdamW steps with NO communication; every
``sync-every`` steps the fused pseudo-gradient all-reduce runs (delta + fp8 quantise + exchange +
reduce + dequantise in one kernel with --quantize; bf16 two-shot otherwise), then the Nesterov
outer step. Reports whole-job tokens/s (device-timed over full sync windows, max over ranks) and
the time of the sync step itself vs an average inner step.
"""

from __future__ import annotations

import argparse
import json
import os
import sys
from datetime import timedelta

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--sync-every", type=int, default=20)
    ap.add_argument("--outer-steps", type=int, default=3)
    ap.add_argument("--quantize", action="store_true")
    ap.add_argument("--no-flat", action="store_true", help="generic per-parameter DiLoCo path instead of the flat fast path")
    ap.add_argument("--out", default="gpurun_out/diloco_bench.json")
    a = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("gloo", timeout=timedelta(seconds=300))

    from torch.distributed import TCPStore

    from torchft_b200 import Manager, ProcessGroupB200
    from torchft_b200.bench_utils import loopback
    from torchft_b200.coordination import LighthouseServer
    from torchft_b200.local_sgd import DiLoCo
    from torchft_b200.models.llama import CONFIGS, FlatParams, Llama

    lh = None
    addr = [None]
    if rank == 0:
        lh = LighthouseServer(bind="[::]:0", min_replicas=world, join_timeout_ms=60000)
        addr = [loopback(lh.address())]
    dist.broadcast_object_list(addr, src=0)

    cfg = CONFIGS[a.model]
    model = Llama(cfg, device=dev)
    if not a.no_flat:
        # one flat weight buffer: DiLoCo then syncs with ONE fused delta all-reduce + ONE fused outer-step kernel
        FlatParams(model)
    model.init_weights(0)
    inner = torch.optim.AdamW(model.parameters(), lr=3e-4, fused=True)
    outer = torch.optim.SGD(model.parameters(), lr=0.7, momentum=0.9, nesterov=True)
    store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
    pg = ProcessGroupB200(timeout=timedelta(seconds=60))
    manager = Manager(pg=pg, min_replica_size=world, use_async_quorum=False, load_state_dict=lambda sd: None,
                      state_dict=lambda: {}, replica_id=f"diloco_{rank}", store_addr="127.0.0.1", store_port=store.port,
                      rank=0, world_size=1, lighthouse_addr=addr[0], timeout=timedelta(seconds=60),
                      quorum_timeout=timedelta(seconds=120), init_sync=False)
    tok = torch.randint(0, cfg.vocab_size, (1, a.seq), device=dev)
    tgt = torch.randint(0, cfg.vocab_size, (1, a.seq), device=dev)
    step_ms, sync_ms = [], []
    with DiLoCo(manager, [model], inner, outer, sync_every=a.sync_every, backup_device=dev, should_quantize=a.quantize,
                use_bucketization=True, bucket_cap_mb=512):
        total = a.sync_every * (a.outer_steps + 1)
        for i in range(total):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            inner.zero_grad(set_to_none=True)
            model(tok, tgt).backward()
            inner.step()  # DiLoCo hooks run the outer sync on schedule
            e.record()
            torch.cuda.synchronize()
            if i >= a.sync_every:  # first window = warm-up
                (sync_ms if (i + 1) % a.sync_every == 0 else step_ms).append(s.elapsed_time(e))
    window_ms = sum(step_ms) / len(step_ms) * (a.sync_every - 1) + sum(sync_ms) / len(sync_ms)
    t = torch.tensor([window_ms, sum(step_ms) / len(step_ms), sum(sync_ms) / len(sync_ms)], dtype=torch.float64)
    # replicas run their inner steps unsynchronised, so at the sync the fast ones WAIT for the slowest (GPU clocks differ by a
    # few % under a power cap, which adds up over the inner steps). The slowest replica arrives last and waits for nobody:
    # MIN over ranks of (sync step - own inner step) is the cost of the sync itself, MAX - MIN is straggler wait.
    own = torch.tensor([t[2] - t[1]], dtype=torch.float64)
    lo = own.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        nparam = cfg.num_params()
        res = {"model": a.model, "params_b": round(nparam / 1e9, 3), "world": world, "seq": a.seq, "sync_every": a.sync_every,
               "quantize": a.quantize, "tokens_per_s": round(world * a.seq * a.sync_every / float(t[0]) * 1e3, 1),
               "inner_step_ms": round(float(t[1]), 2), "sync_step_ms": round(float(t[2]), 2),
               "outer_sync_overhead_ms": round(float(t[2] - t[1]), 2),
               "outer_sync_cost_ms_slowest_replica": round(float(lo[0]), 2),
               "straggler_wait_ms_fastest_replica": round(float(t[2] - t[1]) - float(lo[0]), 2), "outer_steps_committed": manager.current_step(),
               "pseudo_grad_bytes": nparam * 2, "flat_fast_path": not a.no_flat,
               "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 1),
               "link_time_ms_at_450GBps": round((nparam * (1 if a.quantize else 2)) * 2 * (world - 1) / world / 450e6, 2)}
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "a") as f:
            f.write(json.dumps(res) + "\n")
        print("DILOCO_BENCH " + json.dumps(res), flush=True)
    manager.shutdown(wait=False)
    pg.shutdown()
    dist.barrier()
    if lh is not None:
        lh.shutdown()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
