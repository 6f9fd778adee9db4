"""NVLink traffic of every peer-memory kernel, measured by the link counters, against the algorithmic byte count.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29533 \
        bench/nvlink_bytes.py --mb 512 --out gpurun_out/nvlink_bytes_nN.json

Each rank reads its GPU's NVLink data counters (NVML field NVLINK_THROUGHPUT_DATA_TX/RX summed over links, KiB; fallback:
``nvidia-smi nvlink -gt d``) before and after ``--iters`` launches of one kernel, device-times the launches (CUDA events,
MAX over ranks), and reports per launch: counted TX/RX bytes (mean over ranks), the algorithmic bytes the kernel should
move per rank, their ratio, and the achieved fraction of the 450 GB/s per-direction NVLink 4 rate of the H100 data sheet. A kernel that
moved more than its algorithmic bytes (protocol overhead, N x traffic) shows a ratio above 1.
"""

from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from datetime import timedelta

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.checkpointing.p2p_transport import device_copy  # noqa: E402
from torchft_b200.parallel.symm_mem import SymmetricComm  # noqa: E402

LINK_GBS = 450.0


class Counters:
    """(tx_bytes, rx_bytes) of one GPU summed over its NVLinks."""

    def __init__(self, index: int) -> None:
        self.index = index
        self.how = "nvidia-smi"
        self._h = None
        self.nlinks = 0
        try:
            import pynvml

            pynvml.nvmlInit()
            self._nv = pynvml
            self._h = pynvml.nvmlDeviceGetHandleByIndex(index)
            # scopeId = link index (a bare field id reads link 0 only: round 2's first run counted exactly 1/18 of the
            # algorithmic bytes that way); ask the device how many links it has and sum them
            try:
                nlinks = int(pynvml.nvmlDeviceGetFieldValues(self._h, [pynvml.NVML_FI_DEV_NVLINK_LINK_COUNT])[0].value.uiVal)
            except Exception:
                nlinks = 0
            self.nlinks = nlinks if 0 < nlinks <= pynvml.NVML_NVLINK_MAX_LINKS else pynvml.NVML_NVLINK_MAX_LINKS
            self._ids = [(f, l) for l in range(self.nlinks) for f in (pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX,
                                                                     pynvml.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX)]
            tx, rx = self._nvml()
            if tx >= 0:
                self.how = "nvml_field_values"
            else:
                self._h = None
        except Exception:
            self._h = None

    def _nvml(self):
        vals = self._nv.nvmlDeviceGetFieldValues(self._h, self._ids)
        tx = rx = 0
        good = 0
        for i, v in enumerate(vals):
            if v.nvmlReturn != 0:
                continue  # inactive link
            good += 1
            if i % 2 == 0:
                tx += int(v.value.ullVal) * 1024
            else:
                rx += int(v.value.ullVal) * 1024
        return (tx, rx) if good else (-1, -1)

    def read(self):
        if self._h is not None:
            return self._nvml()
        txt = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", str(self.index)], capture_output=True, text=True).stdout
        tx = sum(int(x) for x in re.findall(r"Data Tx:\s*(\d+)\s*KiB", txt)) * 1024
        rx = sum(int(x) for x in re.findall(r"Data Rx:\s*(\d+)\s*KiB", txt)) * 1024
        return tx, rx


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=512.0)
    ap.add_argument("--iters", type=int, default=8)
    ap.add_argument("--replication", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo", timeout=timedelta(seconds=180))
    store = dist.distributed_c10d._get_default_store()
    nelem = int(a.mb * (1 << 20)) // 2 // 4096 * 4096  # bf16 elements
    S = nelem * 2
    comm = SymmetricComm(timeout=timedelta(seconds=30))
    for name in ("z1_grad", "z1_param", "buf"):
        comm.alloc(name, S)
    n32 = nelem // 2  # fp32 elements for the quantised all-reduce (same S bytes of input)
    qb = 0
    if world > 1:
        qb = (comm._K.q8_buffer_bytes(n32, world) + 255) // 256 * 256 + comm._K.q8_slice_buffer_bytes(n32, world)
        comm.alloc("buf_q8", qb)
    comm.configure(dist.PrefixStore("nvl", store), rank, world, 1)
    ctr = Counters(local)
    k = min(a.replication, world)
    dev = torch.device("cuda", local)

    grad = comm.segment("z1_grad")[:S].view(torch.bfloat16)
    grad.normal_()
    buf = comm.segment("buf")[:S].view(torch.bfloat16)
    buf.normal_()
    master = torch.randn(nelem, device=dev)
    m = torch.zeros(nelem, device=dev)
    v = torch.zeros(nelem, device=dev)
    gate = torch.ones(2, dtype=torch.int32, device=dev)
    hp = (3e-4, 0.9, 0.95, 1e-8, 0.1)
    nxt = (rank + 1) % world
    peer_buf = comm.peer_pointers("buf")[nxt]
    local_dst = torch.empty(S, dtype=torch.uint8, device=dev)
    f32 = comm.segment("buf")[: n32 * 4].view(torch.float32)

    W = world
    ops = {
        # name: (fn, algorithmic bytes received per rank, algorithmic bytes sent per rank)
        "allreduce_twoshot_bf16": (lambda: comm.allreduce_(buf, scale=1.0 / W), 2 * (W - 1) / W * S, 2 * (W - 1) / W * S),
        "zero1_reduce_scatter": (lambda: comm.zero1_reduce_scatter_("z1_grad", 0, nelem, 1.0 / W, True, k, 128),
                                 ((W - 1) + (k - 1)) / W * S, ((W - 1) + (k - 1)) / W * S),
        "zero1_update_allgather": (lambda: comm.zero1_update_("z1_param", 0, grad.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                              nelem, hp, gate, k, 0, comm._K.NUM_SMS * 16), (W - k) / W * S, (W - k) / W * S),
        "heal_copy_pull_lsu": (lambda: device_copy([(peer_buf, local_dst.data_ptr(), S)], blocks=128, bulk=False), S, S),
        "heal_copy_pull_bulk_tma": (lambda: device_copy([(peer_buf, local_dst.data_ptr(), S)], blocks=comm._K.MAX_BLOCKS, bulk=True), S, S),
    }
    if qb:
        q_total = n32 * (1 + 4.0 / 512)  # fp8 payload + one fp32 scale per 512 elements
        ops["q8_allreduce_pipeline_fp32"] = (lambda: comm.q8_allreduce_(f32, f32, None, scale=1.0 / W),
                                             2 * (W - 1) / W * q_total, 2 * (W - 1) / W * q_total)

    def barrier():
        torch.cuda.synchronize()
        dist.barrier()

    res = {"world": W, "input_mb": round(S / 2**20, 1), "replication": k, "counter_source": ctr.how, "links_summed": ctr.nlinks, "iters": a.iters, "ops": {}}
    for name, (fn, alg_rx, alg_tx) in ops.items():
        if W == 1:
            break
        try:
            for _ in range(2):
                fn()
            barrier()
            tx0, rx0 = ctr.read()
            barrier()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                fn()
            e.record()
            barrier()
            tx1, rx1 = ctr.read()
            ms = s.elapsed_time(e) / a.iters
            t = torch.tensor([ms, (tx1 - tx0) / a.iters, (rx1 - rx0) / a.iters], dtype=torch.float64)
            mx = t.clone()
            dist.all_reduce(mx, op=dist.ReduceOp.MAX)
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
            tx, rx = float(t[1]) / W, float(t[2]) / W
            res["ops"][name] = {
                "ms_max_over_ranks": round(float(mx[0]), 3),
                "counted_tx_mb_per_rank": round(tx / 1e6, 2), "counted_rx_mb_per_rank": round(rx / 1e6, 2),
                "algorithmic_rx_mb_per_rank": round(alg_rx / 1e6, 2),
                "counted_over_algorithmic": round(max(tx, rx) / max(alg_rx, alg_tx), 3) if alg_rx else None,
                "achieved_gbs_per_direction": round(max(alg_rx, alg_tx) / float(mx[0]) / 1e6, 1),
                "frac_of_link": round(max(alg_rx, alg_tx) / float(mx[0]) / 1e6 / LINK_GBS, 3),
            }
        except Exception as ex:  # keep the sweep going; the failure is part of the report
            res["ops"][name] = {"error": repr(ex)[:200]}
        if rank == 0:
            print(name, res["ops"][name], flush=True)
    if rank == 0:
        print("NVLINK_BYTES " + json.dumps(res), flush=True)
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
    dist.barrier()
    comm.shutdown()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
