"""Hardware tuning sweep for the fused P2P all-reduce: algorithm x grid size.

    torchrun --nproc-per-node N bench/comm_tune.py --out gpurun_out/comm_tune.json

For each message size prints the best (algo, blocks) and the NCCL AVG time; the winning
table is what ``SymmetricComm._plan`` encodes.
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
from torchft_b200.parallel.symm_mem import SymmetricComm  # noqa: E402


def timed(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/comm_tune.json")
    ap.add_argument("--max-mb", type=int, default=256)
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", timeout=timedelta(seconds=120), device_id=torch.device("cuda", local))
    store = dist.distributed_c10d._get_default_store()
    comm = SymmetricComm(timeout=timedelta(seconds=20))
    symm = comm.alloc("tune", args.max_mb << 20)
    comm.configure(dist.PrefixStore("tune", store), rank, world, 1)
    sizes = [1 << k for k in range(12, 31, 1) if (1 << k) <= (args.max_mb << 20)]
    rows = []
    for nbytes in sizes:
        buf = symm[:nbytes].view(torch.bfloat16)
        buf.normal_()
        x = torch.randn(nbytes // 2, device="cuda").bfloat16()
        iters = 40 if nbytes <= (4 << 20) else 12
        nccl = timed(lambda: dist.all_reduce(x, op=dist.ReduceOp.AVG), iters)
        best = None
        table = {}
        for algo in (0, 1):
            for blocks in (4, 16, 32, 64, 128):
                if algo == 0:
                    # in-place one-shot keeps <= 64 KB per block in registers
                    if (nbytes + blocks - 1) // blocks > (64 << 10):
                        continue
                else:
                    if nbytes // blocks < 2048 and blocks > 1:
                        continue
                comm._force_plan = (algo, blocks)
                ms = timed(lambda: comm.allreduce_(buf, scale=1.0 / world), iters)
                table[f"a{algo}_b{blocks}"] = round(ms * 1e3, 2)
                if best is None or ms < best[0]:
                    best = (ms, algo, blocks)
        err = comm.errored()
        row = {"bytes": nbytes, "nccl_avg_us": round(nccl * 1e3, 2), "best_us": round(best[0] * 1e3, 2),
               "best": {"algo": best[1], "blocks": best[2]}, "err": str(err) if err else None, "all_us": table}
        rows.append(row)
        if rank == 0:
            top = sorted(table.items(), key=lambda kv: kv[1])[:6]
            print(json.dumps({"bytes": nbytes, "nccl_avg_us": row["nccl_avg_us"], "top": top}), flush=True)
    if rank == 0:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"world": world, "rows": rows}, f, indent=1)
    comm._force_plan = None
    comm.shutdown()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
