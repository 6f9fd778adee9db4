"""Multi-PROCESS worker for ``ProcessGroupB200`` (launched through torchrun by tests/test_pg_b200_gpu.py).

Ranks are mapped round-robin onto the visible GPUs, so a world of 3 runs on a ONE-GPU box (CUDA IPC works between
processes on one device; the GPU time-slices their spinning kernels). Checks, through the c10d surface and with exact
values (strategy of the reference's process_group_test.py:143-492): every collective, the heal-over-process-group
transport on native send/recv, the fp8 collectives, that no NCCL sidecar was needed, and the resiliency contract
(:890-949): after the last rank goes away the survivors' collective errors within the timeout and ``errored()`` is set.
"""

from __future__ import annotations

import json
import os
import sys
import time
from datetime import timedelta

import torch
import torch.distributed as dist
from torch.distributed import ReduceOp
from torch.distributed.distributed_c10d import (AllgatherOptions, AllreduceOptions, AllToAllOptions, BroadcastOptions,
                                                ReduceScatterOptions)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.checkpointing.pg_transport import PGTransport  # noqa: E402
from torchft_b200.collectives import allocate_reduce_scatter_output, allreduce_quantized, reduce_scatter_quantized  # noqa: E402
from torchft_b200.parallel.process_group_b200 import ProcessGroupB200  # noqa: E402


def main() -> None:
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", timeout=timedelta(seconds=300))
    store_addr = f"{os.environ['MASTER_ADDR']}:{os.environ['MASTER_PORT']}"
    fails = []

    def check(name, ok, **info):
        if not ok:
            fails.append({"what": name, **info})

    pg = ProcessGroupB200(timeout=timedelta(seconds=60), device=dev)
    pg.configure(f"{store_addr}/pgtest/1", f"r{rank}", rank, world, quorum_id=1)

    def ar(t, op):
        o = AllreduceOptions()
        o.reduceOp = op
        pg.allreduce([t], o).wait()
        torch.cuda.synchronize()

    base = torch.arange(5000, device=dev, dtype=torch.float32)
    x = base * (rank + 1)
    ar(x, ReduceOp.SUM)
    check("allreduce_sum", torch.equal(x, base * sum(range(1, world + 1))))
    x = base * (rank + 1)
    ar(x, ReduceOp.AVG)
    check("allreduce_avg", torch.allclose(x, base * sum(range(1, world + 1)) / world))
    x = base + rank
    ar(x, ReduceOp.MAX)
    check("allreduce_max", torch.equal(x, base + world - 1))
    xs = [torch.full((100,), float(rank), device=dev), torch.full((7,), float(rank + 1), device=dev, dtype=torch.bfloat16)]
    o = AllreduceOptions()
    pg.allreduce_coalesced(xs, o).wait()
    torch.cuda.synchronize()
    check("allreduce_coalesced", bool((xs[0] == sum(range(world))).all()) and bool((xs[1] == sum(range(1, world + 1))).all()))

    b = BroadcastOptions()
    b.rootRank = world - 1
    y = torch.full((12345,), rank, device=dev, dtype=torch.int64)
    pg.broadcast([y], b).wait()
    torch.cuda.synchronize()
    check("broadcast_int64", bool((y == world - 1).all()))

    inp = torch.arange(333, device=dev, dtype=torch.float32) + 1000 * rank
    outs = [torch.empty(333, device=dev) for _ in range(world)]
    pg.allgather([outs], [inp], AllgatherOptions()).wait()
    torch.cuda.synchronize()
    check("allgather", all(torch.equal(outs[r], torch.arange(333, device=dev, dtype=torch.float32) + 1000 * r) for r in range(world)))
    flat = torch.empty(world * 333, device=dev)
    pg.allgather_into_tensor_coalesced([flat], [inp], AllgatherOptions()).wait()
    torch.cuda.synchronize()
    check("allgather_into_tensor", torch.equal(flat, torch.cat([torch.arange(333, device=dev, dtype=torch.float32) + 1000 * r for r in range(world)])))

    ro = ReduceScatterOptions()
    ro.reduceOp = ReduceOp.SUM
    ins = [torch.full((64,), float(rank * 10 + p), device=dev) for p in range(world)]
    out = torch.empty(64, device=dev)
    pg.reduce_scatter([out], [ins], ro).wait()
    torch.cuda.synchronize()
    check("reduce_scatter", bool((out == sum(r * 10 + rank for r in range(world))).all()), got=out[:2].tolist())
    big = ((torch.arange(world * 1000, device=dev) % 7) * (rank + 1)).to(torch.bfloat16)
    out2 = torch.empty(1000, device=dev, dtype=torch.bfloat16)
    ro.reduceOp = ReduceOp.AVG
    pg.reduce_scatter_tensor_coalesced([out2], [big], ro).wait()
    torch.cuda.synchronize()
    want = (torch.arange(world * 1000, device=dev, dtype=torch.float32) % 7)[rank * 1000:(rank + 1) * 1000] * sum(range(1, world + 1)) / world
    check("reduce_scatter_tensor_avg", torch.allclose(out2.float(), want, rtol=1e-2, atol=1e-2))

    a_in = torch.arange(world * 50, device=dev, dtype=torch.int32) + 10000 * rank
    a_out = torch.empty_like(a_in)
    pg.alltoall_base(a_out, a_in, [], [], AllToAllOptions()).wait()
    torch.cuda.synchronize()
    check("alltoall_base", torch.equal(a_out, torch.cat([torch.arange(rank * 50, (rank + 1) * 50, device=dev, dtype=torch.int32) + 10000 * p for p in range(world)])))

    # unequal splits: rank r sends (r + p + 1) rows of 3 int64 to rank p, every row tagged with (sender, destination)
    in_rows = [rank + p + 1 for p in range(world)]
    out_rows = [p + rank + 1 for p in range(world)]
    v_in = torch.cat([torch.full((in_rows[p], 3), 1000 * rank + p, device=dev, dtype=torch.int64) for p in range(world)])
    v_out = torch.full((sum(out_rows), 3), -1, device=dev, dtype=torch.int64)
    pg.alltoall_base(v_out, v_in, out_rows, in_rows, AllToAllOptions()).wait()
    torch.cuda.synchronize()
    check("alltoall_base_unequal_splits", torch.equal(v_out, torch.cat([torch.full((out_rows[p], 3), 1000 * p + rank, device=dev, dtype=torch.int64) for p in range(world)])))
    # skewed splits: rank 0 keeps 1 MiB rows for itself and sends one row to each peer, so its own row and column of
    # the split matrix call for a larger grid than any peer's; every rank must still launch the same one
    row = 1 << 18  # fp32 elements: 1 MiB per row
    in_rows = [1] * world
    out_rows = [1] * world
    if rank == 0:
        in_rows[0] = out_rows[0] = 2
    v_in = torch.cat([torch.full((in_rows[p], row), float(1000 * rank + p), device=dev) for p in range(world)])
    v_out = torch.full((sum(out_rows), row), -1.0, device=dev)
    pg.alltoall_base(v_out, v_in, out_rows, in_rows, AllToAllOptions()).wait()
    torch.cuda.synchronize()
    check("alltoall_base_skewed_splits", pg.errored() is None and torch.equal(v_out, torch.cat(
        [torch.full((out_rows[p], row), float(1000 * p + rank), device=dev) for p in range(world)])), err=str(pg.errored()))

    # ring send/recv (both posted before either is waited on: sends and receives run on separate streams)
    msg = torch.full((200_000,), float(rank), device=dev)
    got = torch.empty_like(msg)
    ws = pg.send([msg], (rank + 1) % world, 0)
    wr = pg.recv([got], (rank - 1) % world, 0)
    ws.wait(), wr.wait()
    torch.cuda.synchronize()
    check("send_recv_ring", bool((got == (rank - 1) % world).all()))
    pg.barrier().wait()
    torch.cuda.synchronize()

    # heal over the process group itself (reference pg_transport.py) on the native send/recv kernels
    state = {"w": torch.arange(70_000, device=dev, dtype=torch.float32) * (1 if rank == 0 else 0), "step": 7 if rank == 0 else 0,
             "nested": {"b": torch.ones(33, device=dev, dtype=torch.bfloat16) * (3 if rank == 0 else 0)}}
    tr = PGTransport(pg, timeout=timedelta(seconds=60), device=dev)
    if rank == 0:
        tr.send_checkpoint(list(range(1, world)), 7, state, timedelta(seconds=60))
    else:
        got_sd = tr.recv_checkpoint(0, tr.metadata(), 7, timedelta(seconds=60))
        torch.cuda.synchronize()
        check("pg_transport_heal", got_sd["step"] == 7 and torch.equal(got_sd["w"], torch.arange(70_000, device=dev, dtype=torch.float32))
              and bool((got_sd["nested"]["b"] == 3).all()))
    dist.barrier()

    # fp8 collectives through the fused kernels
    gen = torch.Generator(device=dev).manual_seed(100 + rank)
    ts = [(torch.rand(256, 64, device=dev, generator=gen) * 9 + 1) for _ in range(2)]
    refs = []
    for t in ts:
        r_ = t.float().cpu()
        dist.all_reduce(r_)
        refs.append((r_ / world).to(dev))
    allreduce_quantized([t for t in ts], ReduceOp.AVG, pg).wait()
    torch.cuda.synchronize()
    for t, r_ in zip(ts, refs):
        check("allreduce_quantized", ((t - r_).abs().mean() / r_.abs().mean()).item() <= 0.04)
    ts = [(torch.rand(64 * world, 128, device=dev, generator=gen) + 0.5) for _ in range(2)]
    out_q, padded = allocate_reduce_scatter_output(ts, world)
    refs = []
    for t in ts:
        r_ = t.float().cpu()
        dist.all_reduce(r_)
        refs.append(r_.to(dev))
    before = pg.comm.launches
    reduce_scatter_quantized(out_q, ts, ReduceOp.SUM, pg).wait()
    torch.cuda.synchronize()
    check("reduce_scatter_quantized_is_fused", pg.comm.launches - before == len(ts), launches=pg.comm.launches - before)
    off = 0
    for r_, ps in zip(refs, padded):
        rows = ps[0] // world
        mine = r_[rank * rows:(rank + 1) * rows].reshape(-1)
        got_q = out_q[off: off + mine.numel()]
        off += mine.numel()
        check("reduce_scatter_quantized", ((got_q - mine).abs().mean() / mine.abs().mean()).item() <= 0.05)

    # ---- a symmetric segment allocated AFTER the first quorum: ordinary memory (staged path) until the next quorum change,
    # zero-copy from then on; the last rank allocates it only after that reconfigure -> still staged, still correct ----
    late = None
    if rank != world - 1 or world == 1:
        late = pg.alloc_symmetric("late", 1 << 20).view(torch.float32)
    check("late_segment_not_symmetric_yet", late is None or not pg.comm.is_symmetric("late"))
    v = late[:4096] if late is not None else torch.empty(4096, device=dev)
    v.fill_(float(rank + 1))
    ar(v, ReduceOp.SUM)
    check("late_segment_allreduce_staged", bool((v == sum(range(1, world + 1))).all()))

    check("no_sidecar", pg._sidecar is None)
    check("no_latched_error", pg.errored() is None, err=str(pg.errored()))

    # ---- resiliency: reconfigure with a short timeout; the last rank leaves; survivors must error, not hang ----
    dist.barrier()
    pg.set_timeout(timedelta(seconds=2))
    pg.configure(f"{store_addr}/pgtest/2", f"r{rank}", rank, world, quorum_id=2)
    z = torch.ones(1 << 16, device=dev)
    ar(z, ReduceOp.SUM)
    check("post_reconfigure", bool((z == world).all()) and pg.errored() is None)
    # the last rank never registered "late": the segment stays local-only on everybody (intersection rule) and works
    check("late_segment_needs_every_rank", late is None or pg.comm.is_symmetric("late") == (world == 1))
    v = late[:4096] if late is not None else torch.empty(4096, device=dev)
    v.fill_(2.0)
    ar(v, ReduceOp.SUM)
    check("late_segment_allreduce_after_reconfigure", bool((v == 2.0 * world).all()))
    if world > 1 and rank == world - 1:
        late = pg.alloc_symmetric("late", 1 << 20).view(torch.float32)
    dist.barrier()
    pg.configure(f"{store_addr}/pgtest/3", f"r{rank}", rank, world, quorum_id=3)
    check("late_segment_symmetric_once_everybody_has_it", pg.comm.is_symmetric("late"))
    before = pg.comm.launches
    v = late[:4096]
    v.fill_(3.0)
    ar(v, ReduceOp.SUM)
    check("late_segment_allreduce_zero_copy", bool((v == 3.0 * world).all()) and pg.comm.launches - before == 1)
    dist.barrier()
    took = 0.0
    if rank == world - 1:
        pg.shutdown()
    else:
        t0 = time.monotonic()
        z = torch.ones(1 << 16, device=dev)
        o = AllreduceOptions()
        try:
            pg.allreduce([z], o).wait()
            torch.cuda.synchronize()
        except RuntimeError:
            pass
        err = pg.errored()
        took = time.monotonic() - t0
        check("survivor_errors_within_timeout", err is not None and took < 15.0, took=took, err=str(err))
        raised = False
        try:  # a latched group refuses new work on the host
            pg.allreduce([z], o)
        except RuntimeError:
            raised = True
        check("latched_group_refuses_work", raised)
    dist.barrier()
    if rank != world - 1:
        pg.shutdown()

    nf = torch.tensor([len(fails)])
    dist.all_reduce(nf)
    if fails:
        print(f"[rank {rank}] FAIL " + json.dumps(fails[:8]), flush=True)
    if rank == 0:
        print("PG_B200 " + json.dumps({"world": world, "gpus": torch.cuda.device_count(), "failures": int(nf.item()),
                                       "survivor_error_s": round(took, 2)}), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if int(nf.item()) else 0)


if __name__ == "__main__":
    main()
