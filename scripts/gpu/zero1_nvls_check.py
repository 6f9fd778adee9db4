"""VMM + NVLS data plane check on >= 2 real GPUs (the one-GPU test tier cannot bind a multicast object):

    TORCHFT_B200_SYMM=vmm python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29544 scripts/gpu/zero1_nvls_check.py --out gpurun_out/zero1_nvls_n2.json

* reconfigure cost: first configure (fd import + multicast create/bind), a second one over the same members (everything
  cached) and one after dropping the multicast objects (batched rebuild);
* FT-ZeRO-1 reduce-scatter and update through the multimem (in-switch) variants against the P2P variants on the same
  inputs: element-wise difference of the reduced gradients and of the new weights, and device time of both.
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time
from datetime import timedelta

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from torchft_b200.parallel.symm_mem import SymmetricComm  # noqa: E402

HP = (3e-4, 0.9, 0.95, 1e-8, 0.1)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=128.0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("gloo", timeout=timedelta(seconds=120))
    store = dist.distributed_c10d._get_default_store()
    nelem = int(a.mb * (1 << 20)) // 2 // 4096 * 4096
    S = nelem * 2
    comm = SymmetricComm(timeout=timedelta(seconds=20))
    for n in ("z1_grad", "z1_param", "z1_master", "z1_m", "z1_v"):
        comm.alloc(n, S if n in ("z1_grad", "z1_param") else 4096)
    res = {"world": world, "mode": comm._mode, "unit_mb": round(S / 2**20, 1)}

    def configure(epoch: int) -> float:
        dist.barrier()
        t0 = time.perf_counter()
        comm.configure(dist.PrefixStore(f"q{epoch}", store), rank, world, epoch)
        dt = (time.perf_counter() - t0) * 1e3
        t = torch.tensor([dt], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return round(float(t.item()), 3)

    res["configure_first_ms"] = configure(1)
    res["nvls_objects"] = sorted(comm._mc)
    res["configure_same_members_ms"] = configure(2)
    comm._release_multicast()
    res["configure_rebuild_multicast_ms"] = configure(3)

    grad = comm.segment("z1_grad")[:S].view(torch.bfloat16)
    param = comm.segment("z1_param")[:S].view(torch.bfloat16)
    gate = torch.ones(2, dtype=torch.int32, device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(100 + rank)
    g0 = torch.randn(nelem, device=dev, generator=gen).bfloat16()
    gen.manual_seed(7)
    w0 = torch.randn(nelem, device=dev, generator=gen)

    def sync():
        torch.cuda.synchronize()
        dist.barrier()

    def run(k: int, nvls: bool):
        comm._nvls_min = 0 if nvls else (1 << 62)
        master, m, v = w0.clone(), torch.zeros(nelem, device=dev), torch.zeros(nelem, device=dev)
        grad.copy_(g0)
        param.zero_()
        sync()
        comm.zero1_reduce_scatter_("z1_grad", 0, nelem, 1.0 / world, True, k, 128)
        sync()
        reduced = grad.clone()
        comm.zero1_update_("z1_param", 0, grad.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), nelem, HP, gate, k, 0, comm._K.NUM_SMS * 16)
        sync()
        weights = param.clone()
        times = {}
        for name, fn in (("reduce_scatter_ms", lambda: comm.zero1_reduce_scatter_("z1_grad", 0, nelem, 1.0 / world, True, k, 128)),
                         ("update_ms", lambda: comm.zero1_update_("z1_param", 0, grad.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), nelem, HP, gate, k, 0, comm._K.NUM_SMS * 16))):
            for _ in range(2):
                fn()
            sync()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                fn()
            e.record()
            sync()
            t = torch.tensor([s.elapsed_time(e) / a.iters], dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            times[name] = round(float(t.item()), 4)
        return reduced, weights, times

    sl = nelem // world
    for k in sorted({1, min(2, world)}):
        ref_r, ref_w, t_p2p = run(k, False)
        out = {"p2p": t_p2p}
        if comm._mc:
            nv_r, nv_w, t_nv = run(k, True)
            held = [(rank - j) % world for j in range(k)]  # slices this rank holds after the reduce-scatter
            dr = max(float((nv_r[s * sl:(s + 1) * sl].float() - ref_r[s * sl:(s + 1) * sl].float()).abs().max()) for s in held)
            dw = float((nv_w.float() - ref_w.float()).abs().max())
            stats = torch.tensor([dr, dw, float(ref_w.float().abs().max())], dtype=torch.float64)
            dist.all_reduce(stats, op=dist.ReduceOp.MAX)
            out.update({"nvls": t_nv, "max_abs_diff_reduced_grad": float(stats[0]), "max_abs_diff_weights": float(stats[1]),
                        "weights_nonzero": bool(stats[2] > 0)})
        res[f"k{k}"] = out
    if rank == 0:
        print("ZERO1_NVLS " + json.dumps(res), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
    dist.barrier()
    comm.shutdown()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
