"""Where does a fault-tolerant step go at N GPUs? torch.profiler timeline of rank 0, reduced to numbers.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29611 \
        bench/timeline.py --impl native --out gpurun_out/timeline_n8_native.json

Every rank trains (same loop as bench.py); rank 0 profiles ``--steps`` steady-state steps and the chrome trace is
reduced to: wall time per step, busy time per CUDA stream, time of OUR collective / optimizer kernels, how much of it is
hidden under compute kernels of other streams, idle gaps of the compute stream (with the kernel that ended the gap),
and the top kernels. This is the attribution the 1 -> N scaling loss needs (which kernels are exposed, how long the compute
stream waits and for whom).
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
from collections import defaultdict
from datetime import timedelta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OURS = ("zero1_", "allreduce_", "q8_", "push_exchange", "reduce_scatter_kernel", "p2p_", "heal_copy", "adamw", "scale_copy")


def union(iv):
    iv = sorted(iv)
    out = []
    for a, b in iv:
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def total(iv):
    return sum(b - a for a, b in iv)


def intersect(a, b):
    i = j = 0
    out = []
    while i < len(a) and j < len(b):
        lo, hi = max(a[i][0], b[j][0]), min(a[i][1], b[j][1])
        if lo < hi:
            out.append([lo, hi])
        if a[i][1] < b[j][1]:
            i += 1
        else:
            j += 1
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="native", choices=["native", "nccl"])
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default="gpurun_out/timeline.json")
    a = ap.parse_args()

    import torch
    import torch.distributed as dist

    from torchft_b200.bench_utils import loopback
    from torchft_b200.coordination import LighthouseServer
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    lh, addr = None, [None]
    if world > 1:
        dist.init_process_group("gloo", timeout=timedelta(seconds=300))
    if rank == 0:
        lh = LighthouseServer(bind="[::]:0", min_replicas=world, join_timeout_ms=60000)
        addr = [loopback(lh.address())]
    if world > 1:
        dist.broadcast_object_list(addr, src=0)
    tr = FaultTolerantTrainer(a.model, addr[0], replica_id=f"tl_{rank}", min_replica_size=world,
                              backend="b200" if a.impl == "native" else "nccl", timeout=timedelta(seconds=120), device=dev)
    cfg = tr.cfg
    tok = torch.randint(0, cfg.vocab_size, (1, a.seq), device=dev)
    tgt = torch.randint(0, cfg.vocab_size, (1, a.seq), device=dev)
    for _ in range(a.warmup):
        tr.step_device(tok, tgt)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()

    from torch.profiler import ProfilerActivity, profile

    if rank == 0:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                tr.step_device(tok, tgt)
            tr.join()
            torch.cuda.synchronize()
        path = os.path.join(tempfile.mkdtemp(), "trace.json")
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
        t0 = min(e["ts"] for e in ev)
        t1 = max(e["ts"] + e["dur"] for e in ev)
        by_stream = defaultdict(list)
        names = defaultdict(lambda: [0.0, 0])
        for e in ev:
            by_stream[e["args"].get("stream")].append((e["ts"], e["ts"] + e["dur"], e["name"]))
            k = names[e["name"][:70]]
            k[0] += e["dur"]
            k[1] += 1
        busy = {s: total(union([(x, y) for x, y, _ in v])) for s, v in by_stream.items()}
        compute_stream = max(busy, key=busy.get)
        ours = union([(x, y) for s, v in by_stream.items() for x, y, n in v if any(o in n for o in OURS) and s != compute_stream])
        comp = union([(x, y) for x, y, _ in by_stream[compute_stream]])
        hidden = total(intersect(ours, comp))
        # idle gaps of the compute stream inside the profiled window and what ran on the other streams meanwhile
        gaps = []
        cs = sorted(by_stream[compute_stream])
        for (a0, a1, n0), (b0, b1, n1) in zip(cs, cs[1:]):
            if b0 - a1 > 200:  # > 0.2 ms
                during = defaultdict(float)
                for s, v in by_stream.items():
                    if s == compute_stream:
                        continue
                    for x, y, n in v:
                        ov = min(y, b0) - max(x, a1)
                        if ov > 0:
                            during[n[:50]] += ov
                top = sorted(during.items(), key=lambda kv: -kv[1])[:3]
                gaps.append({"ms": round((b0 - a1) / 1e3, 3), "after": n0[:50], "before": n1[:50],
                             "other_streams": [[k, round(vv / 1e3, 3)] for k, vv in top]})
        gaps.sort(key=lambda g: -g["ms"])
        res = {
            "impl": a.impl, "world": world, "steps": a.steps, "ms_per_step_profiled": round((t1 - t0) / 1e3 / a.steps, 2),
            "compute_stream_busy_ms_per_step": round(busy[compute_stream] / 1e3 / a.steps, 2),
            "compute_stream_idle_ms_per_step": round(((t1 - t0) - busy[compute_stream]) / 1e3 / a.steps, 2),
            "streams_busy_ms_per_step": {str(s): round(b / 1e3 / a.steps, 2) for s, b in sorted(busy.items(), key=lambda kv: -kv[1])},
            "our_side_stream_kernels_ms_per_step": round(total(ours) / 1e3 / a.steps, 2),
            "of_which_hidden_under_compute_ms_per_step": round(hidden / 1e3 / a.steps, 2),
            "exposed_ms_per_step": round((total(ours) - hidden) / 1e3 / a.steps, 2),
            "largest_compute_gaps": gaps[:12],
            "sum_of_gaps_over_0p2ms_per_step": round(sum(g["ms"] for g in gaps) / a.steps, 2),
            "top_kernels_ms_per_step": [[k, round(v[0] / 1e3 / a.steps, 2), v[1] // a.steps] for k, v in sorted(names.items(), key=lambda kv: -kv[1][0])[:25]],
        }
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
        print("TIMELINE " + json.dumps({k: res[k] for k in res if k not in ("top_kernels_ms_per_step", "largest_compute_gaps")}), flush=True)
    else:
        for _ in range(a.steps):
            tr.step_device(tok, tgt)
        tr.join()
        torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    tr.shutdown()
    if world > 1:
        dist.barrier()
    if lh is not None:
        lh.shutdown()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
