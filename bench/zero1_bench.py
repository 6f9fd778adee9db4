"""FT-ZeRO-1 kernel micro-benchmark: reduce-scatter (+buddy push) and gated AdamW + weight all-gather.

Multi-GPU (device-timed, max over ranks, bus bytes per rank vs the H100 data-sheet NVLink 4 rate, 450 GB/s per direction):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29517 bench/zero1_bench.py --mb 436 --out gpurun_out/zero1_bench_nN.json

Single GPU, for ncu / compute-sanitizer (ranks emulated in-process, flags pre-signalled, one kernel at a time; the
"peer" loads then hit local HBM, so these captures show instruction mix / occupancy / HBM behaviour, not NVLink):

    ncu --set full -k regex:zero1 ... python bench/zero1_bench.py --virtual 8 --mb 64 --iters 2

Per unit of S bytes of bf16 gradients and W ranks with k holders per slice, each rank moves over NVLink:
  reduce-scatter  in  (W-1)/W * S      (+ (k-1)/W * S out for the buddy push)
  update          out (W-1)/W * S      (bf16 weights to every peer)        [NVLS: S/W in, S/W out]
and touches HBM: 28 B/param * k/W of the unit for AdamW (vs 28 B/param for the full replicated update).
"""

from __future__ import annotations

import argparse
import json
import os
import sys
from datetime import timedelta

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.parallel.symm_mem import SymmetricComm  # noqa: E402

HP = (3e-4, 0.9, 0.95, 1e-8, 0.1)


def run_rank(comm, nelem, k, rs_blocks, upd_blocks, iters, warmup, sync, reduce_max):
    upd_blocks = upd_blocks or comm._K.NUM_SMS * 16
    dev = comm.device
    grad = comm.segment("z1_grad")[: nelem * 2].view(torch.bfloat16)
    grad.normal_()
    master = torch.randn(nelem, device=dev)
    m = torch.zeros(nelem, device=dev)
    v = torch.zeros(nelem, device=dev)
    gate = torch.ones(2, dtype=torch.int32, device=dev)

    def rs():
        comm.zero1_reduce_scatter_("z1_grad", 0, nelem, 1.0 / max(comm.world, 1), True, k, rs_blocks)

    def upd():
        comm.zero1_update_("z1_param", 0, grad.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), nelem, HP, gate, k, 0, upd_blocks)

    out = {}
    for name, fn in (("reduce_scatter", rs), ("adamw_allgather", upd)):
        if name == "reduce_scatter" and comm.world == 1:
            continue
        for _ in range(warmup):
            fn()
        sync()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        out[name] = reduce_max(s.elapsed_time(e) / iters)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=436.0, help="unit size in MB of bf16 gradients (one Llama-3-8B block = 436 MB)")
    ap.add_argument("--replication", type=int, default=2)
    ap.add_argument("--rs-blocks", type=int, default=128)
    ap.add_argument("--upd-blocks", type=int, default=0, help="grid cap of the update kernel (0: 16 per SM, the trainer default)")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--virtual", type=int, default=0, help="emulate this many ranks on ONE GPU (presignalled; for ncu)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    nelem = int(a.mb * (1 << 20)) // 2 // 4096 * 4096
    S = nelem * 2

    if a.virtual:
        torch.cuda.set_device(0)
        comms = SymmetricComm.virtual_world(a.virtual, {"z1_grad": S, "z1_param": S}, presignal=True)
        res = {"mode": f"virtual{a.virtual}", "unit_mb": S / 2**20}
        for c in comms[:1]:  # rank 0's kernels are representative; every rank does the same work
            res.update(run_rank(c, nelem, a.replication, a.rs_blocks, a.upd_blocks, a.iters, a.warmup, torch.cuda.synchronize, lambda x: x))
        print("ZERO1_BENCH " + json.dumps(res), flush=True)
        return

    import torch.distributed as dist

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo", timeout=timedelta(seconds=120))
    store = dist.distributed_c10d._get_default_store()
    comm = SymmetricComm(timeout=timedelta(seconds=30))
    comm.alloc("z1_grad", S)
    comm.alloc("z1_param", S)
    comm.configure(dist.PrefixStore("z1b", store), rank, world, 1)

    def sync():
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()

    def reduce_max(ms):
        t = torch.tensor([ms], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    res = {"world": world, "unit_mb": round(S / 2**20, 1), "replication": min(a.replication, world), "rs_blocks": a.rs_blocks, "upd_blocks": a.upd_blocks or comm._K.NUM_SMS * 16,
           "mode": comm._mode, "nvls": bool(comm._mc)}
    t = run_rank(comm, nelem, a.replication, a.rs_blocks, a.upd_blocks, a.iters, a.warmup, sync, reduce_max)
    k = min(a.replication, world)
    link = 450.0  # GB/s per direction per GPU: H100 SXM data sheet (NVLink 4, 900 GB/s bidirectional)
    hbm = 3350.0  # GB/s: H100 SXM data sheet (HBM3)
    if "reduce_scatter" in t:
        inb = (world - 1) / world * S
        res["reduce_scatter"] = {"ms": round(t["reduce_scatter"], 3), "nvlink_in_gb": round(inb / 1e9, 3),
                                 "in_gbps": round(inb / t["reduce_scatter"] / 1e6, 1),
                                 "frac_of_link": round(inb / t["reduce_scatter"] / 1e6 / link, 3)}
    outb = max(0, world - k) / world * S  # holders compute their own copy: the primary pushes to W - k ranks
    hbm_b = 28.0 * nelem * k / world
    floor_ms = max(outb / (link * 1e6), hbm_b / (hbm * 1e6)) if world > 1 else hbm_b / (hbm * 1e6)
    res["adamw_allgather"] = {"ms": round(t["adamw_allgather"], 3), "nvlink_out_gb": round(outb / 1e9, 3),
                              "hbm_gb": round(hbm_b / 1e9, 3), "roofline_ms": round(floor_ms, 3),
                              "frac_of_roofline": round(floor_ms / t["adamw_allgather"], 3),
                              "full_replicated_adamw_hbm_gb": round(28.0 * nelem / 1e9, 3)}
    if rank == 0:
        print("ZERO1_BENCH " + json.dumps(res), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
    dist.barrier()
    comm.shutdown()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
