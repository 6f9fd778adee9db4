"""FT-ZeRO-1 kernel micro-benchmark: reduce-scatter (+buddy push) and gated AdamW + weight all-gather.

Multi-GPU (device-timed, max over ranks, bus bytes per rank vs the H100 data-sheet NVLink 4 rate, 450 GB/s per direction):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29517 bench/zero1_bench.py --mb 436 --out gpurun_out/zero1_bench_nN.json

Single GPU, for ncu / compute-sanitizer (ranks emulated in-process, flags pre-signalled, one kernel at a time; the
"peer" loads then hit local HBM, so these captures show instruction mix / occupancy / HBM behaviour, not NVLink):

    ncu --set full -k regex:zero1 ... python bench/zero1_bench.py --virtual 8 --mb 64 --iters 2

``--virtual W --compact`` times the update with flat state and with paged state (compact optimizer state: 64 Ki-element
pages in a pool behind a page table, once in slot order and once in a random slot order) in the same process,
alternating the three ``--repeats`` times; it
reports the median and the spread of each. The peer stores hit local HBM there, so this compares the state addressing,
not NVLink.

``--virtual W --clip`` times reduce-scatter + commit + update of one unit (rank 0's launches) without and with global
gradient-norm clipping, alternating the two ``--repeats`` times, and reports the median and the spread of each with the
card's name and power limit. Clipping adds squares to the reduce, per-rank partial loads to the commit and one multiply
per element to the update; the peer loads hit local HBM there, so NVLink costs are not part of the comparison.

``--virtual W --accum`` times rank 0's reduce launch of one unit in the gradient-accumulation modes off (today's launch),
acc (a middle micro-batch: 32 B of fp32 accumulator read and written per 8 elements, no bf16 store, no push) and last
(accumulator read, bf16 store and buddy push), alternating ``--repeats`` times, with the card's name and power limit.
It first checks that an accumulated pair gives the off result bit for bit. The peer loads hit local HBM, so this
compares the kernels' HBM behaviour, not NVLink.

``--virtual W --sched`` times the update of one unit (rank 0's launch) without a learning-rate schedule and with a
table of rates and two weight-decay exemptions, alternating the two ``--repeats`` times, with the card's name and power
limit. The scheduled launch adds one uniform table load per thread and a few integer compares per 8 elements to a kernel
bound by HBM; it first checks that a constant table and no exemptions give the plain launch's bits.

``--virtual W --moments`` times the update of one unit (rank 0's launch) with fp32 and with bf16 moments, alternating
the two ``--repeats`` times, on flat state or (with ``--compact``) on page pools in slot order, with the card's name and
power limit. It reports medians, spread and the bytes the launch moves, computed from the shapes: per updated element
2 (gradient) + 8 (master in and out) + 2 (weight) + 4 x the moment size, i.e. 28 B with fp32 and 20 B with bf16 moments,
plus 2 B per primary element and peer the weights are pushed to (local HBM here, NVLink on real ranks).

``--virtual W --ema`` times the update of one unit (rank 0's launch) without and with an EMA of the weights, for fp32
and for bf16 moments (the EMA has the moments' type), alternating the four arms ``--repeats`` times, on flat state or
(with ``--compact``) on page pools in slot order, with the card's name and power limit. The EMA adds 2 x its size per
updated element (read and written): 36 B instead of 28 with fp32 moments, 24 B instead of 20 with bf16.

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


def compact_ab(comm, nelem, k, upd_blocks, iters, warmup, repeats, shift=16):
    """Gated AdamW + weight push of one unit on flat state vs the same values in page pools, timed alternately: pages in
    slot order (what a re-shard into an empty pool produces) and in a random slot order (a pool that has been through
    many re-shards). All three must agree bit for bit."""
    upd_blocks = upd_blocks or comm._K.NUM_SMS * 16
    dev = comm.device
    grad = comm.segment("z1_grad")[: nelem * 2].view(torch.bfloat16)
    grad.normal_()
    gate = torch.ones(2, dtype=torch.int32, device=dev)
    npages = (nelem + (1 << shift) - 1) >> shift
    flat = [torch.randn(nelem, device=dev), torch.zeros(nelem, device=dev), torch.zeros(nelem, device=dev)]
    layouts = {}
    for name, table in (("ordered", torch.arange(npages, device=dev)), ("random", torch.randperm(npages, device=dev))):
        idx = (table.long()[:, None] * (1 << shift) + torch.arange(1 << shift, device=dev)).view(-1)[:nelem]
        pool = [torch.zeros(npages << shift, device=dev) for _ in flat]
        for p, x in zip(pool, flat):
            p[idx] = x
        layouts[name] = (table.int(), idx, pool)

    def upd_flat():
        comm.zero1_update_("z1_param", 0, grad.data_ptr(), flat[0].data_ptr(), flat[1].data_ptr(), flat[2].data_ptr(), nelem,
                           HP, gate, k, 0, upd_blocks)

    def upd_paged(layout):
        table, _, pool = layouts[layout]
        return lambda: comm.zero1_update_("z1_param", 0, grad.data_ptr(), pool[0].data_ptr(), pool[1].data_ptr(),
                                          pool[2].data_ptr(), nelem, HP, gate, k, 0, upd_blocks, None, table.data_ptr(), 0,
                                          shift)

    arms = (("flat", upd_flat), ("paged_ordered", upd_paged("ordered")), ("paged_random", upd_paged("random")))
    for _, fn in arms:
        fn()
    torch.cuda.synchronize()
    same = all(torch.equal(p[idx], x) for _, idx, pool in layouts.values() for p, x in zip(pool, flat))
    times = {name: [] for name, _ in arms}
    for _ in range(repeats):
        for name, fn in arms:
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    out = {"paged_equals_flat": same, "timing": "local HBM (virtual ranks), not NVLink"}
    for name, ts in times.items():
        ts = sorted(ts)
        out[f"adamw_allgather_{name}_ms"] = {"median": round(ts[len(ts) // 2], 4), "min": round(ts[0], 4),
                                             "max": round(ts[-1], 4)}
    for name in ("paged_ordered", "paged_random"):
        out[f"{name}_over_flat"] = round(out[f"adamw_allgather_{name}_ms"]["median"] / out["adamw_allgather_flat_ms"]["median"], 4)
    return out


def gpu_info() -> dict:
    """Card name and power limit: part of every absolute number this script prints."""
    import subprocess

    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in out.split(",")[:2]]
    except Exception as e:  # noqa: BLE001 - the timing stands without it, but say why it is missing
        info["power_limit"] = f"unavailable ({e})"
    return info


def clip_ab(comm, nelem, k, rs_blocks, upd_blocks, iters, warmup, repeats, max_norm=1.0):
    """Reduce-scatter + commit + update of one unit without clipping and with it, timed alternately."""
    upd_blocks = upd_blocks or comm._K.NUM_SMS * 16
    dev = comm.device
    grad = comm.segment("z1_grad")[: nelem * 2].view(torch.bfloat16)
    grad.normal_()
    state = [torch.randn(nelem, device=dev), torch.zeros(nelem, device=dev), torch.zeros(nelem, device=dev)]
    gate = torch.zeros(2, dtype=torch.int32, device=dev)
    clip = torch.zeros(2, dtype=torch.float32, device=dev)
    gn = comm.segment("z1_gnorm").data_ptr()
    # only this rank reduces, and only its k holders' copies of slice 0 are non-zero: 1/k keeps the repeated reduce at a
    # fixed point (1/W would decay the gradient to zero, and with it the norm and the clipping)
    scale = 1.0 / min(k, comm.world)

    def step(on):
        def fn():
            comm.zero1_reduce_scatter_("z1_grad", 0, nelem, scale, True, k, rs_blocks, gnorm=gn if on else 0)
            if on:
                comm.zero1_commit_(gate, True, True, gnorm="z1_gnorm", nunits=1, max_norm=max_norm, norm=clip)
            else:
                comm.zero1_commit_(gate, True, True)
            comm.zero1_update_("z1_param", 0, grad.data_ptr(), state[0].data_ptr(), state[1].data_ptr(), state[2].data_ptr(),
                               nelem, HP, gate, k, 0, upd_blocks, coef=clip.data_ptr() + 4 if on else 0)
        return fn

    arms = (("off", step(False)), ("clip", step(True)))
    times = {name: [] for name, _ in arms}
    for _ in range(repeats):
        for name, fn in arms:
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    assert comm.errored() is None
    out = {"timing": "local HBM (virtual ranks), not NVLink", "max_norm": max_norm, "last_norm": float(clip[0]),
           "last_coef": float(clip[1])}
    for name, ts in times.items():
        ts = sorted(ts)
        out[f"rs_commit_update_{name}_ms"] = {"median": round(ts[len(ts) // 2], 4), "min": round(ts[0], 4),
                                              "max": round(ts[-1], 4)}
    out["clip_over_off"] = round(out["rs_commit_update_clip_ms"]["median"] / out["rs_commit_update_off_ms"]["median"], 4)
    return out


def sched_ab(comm, nelem, k, upd_blocks, iters, warmup, repeats):
    """The update of one unit without a schedule and with a 1000-entry rate table and two exempt ranges, alternately."""
    upd_blocks = upd_blocks or comm._K.NUM_SMS * 16
    dev = comm.device
    grad = comm.segment("z1_grad")[: nelem * 2].view(torch.bfloat16)
    grad.normal_()
    gate = torch.ones(2, dtype=torch.int32, device=dev)
    gate[1] = 500
    init = torch.randn(nelem, device=dev)
    table = torch.full((1000,), HP[0], dtype=torch.float32, device=dev)

    def state():
        return [init.clone(), torch.zeros(nelem, device=dev), torch.zeros(nelem, device=dev)]

    def launch(st, **kw):
        return lambda: comm.zero1_update_("z1_param", 0, grad.data_ptr(), st[0].data_ptr(), st[1].data_ptr(),
                                          st[2].data_ptr(), nelem, HP, gate, k, 0, upd_blocks, **kw)

    # bit check: a table of the constant rate and no exemptions is the plain launch
    a, b = state(), state()
    launch(a)()
    launch(b, lr_table=table.data_ptr(), lr_steps=table.numel())()
    torch.cuda.synchronize()
    same = all(torch.equal(x, y) for x, y in zip(a, b))
    nd = [(nelem // 8 // 8 * 8, nelem // 8 // 8 * 8 + 4096), (nelem // 2 // 8 * 8, nelem // 2 // 8 * 8 + 4096)]
    st = state()
    arms = (("off", launch(st)), ("sched", launch(st, lr_table=table.data_ptr(), lr_steps=table.numel(), no_decay=nd)))
    times = {name: [] for name, _ in arms}
    for _ in range(repeats):
        for name, fn in arms:
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    out = {"timing": "local HBM (virtual ranks), not NVLink", "constant_table_equals_off": same, "no_decay_ranges": nd}
    for name, ts in times.items():
        ts = sorted(ts)
        out[f"adamw_allgather_{name}_ms"] = {"median": round(ts[len(ts) // 2], 4), "min": round(ts[0], 4),
                                             "max": round(ts[-1], 4)}
    out["sched_over_off"] = round(out["adamw_allgather_sched_ms"]["median"] / out["adamw_allgather_off_ms"]["median"], 4)
    return out


def moments_ab(comm, nelem, k, upd_blocks, iters, warmup, repeats, paged, shift=16):
    """The update of one unit with fp32 and with bf16 moments, timed alternately, on flat state or on page pools."""
    upd_blocks = upd_blocks or comm._K.NUM_SMS * 16
    dev = comm.device
    grad = comm.segment("z1_grad")[: nelem * 2].view(torch.bfloat16)
    grad.normal_()
    gate = torch.ones(2, dtype=torch.int32, device=dev)
    npages = (nelem + (1 << shift) - 1) >> shift
    n_state = npages << shift if paged else nelem
    table = torch.arange(npages, dtype=torch.int32, device=dev)
    paging = dict(table=table.data_ptr(), page_shift=shift) if paged else {}

    def arm(dtype):
        st = [torch.randn(n_state, device=dev), torch.zeros(n_state, device=dev, dtype=dtype),
              torch.zeros(n_state, device=dev, dtype=dtype)]
        return st, lambda: comm.zero1_update_("z1_param", 0, grad.data_ptr(), st[0].data_ptr(), st[1].data_ptr(),
                                              st[2].data_ptr(), nelem, HP, gate, k, 0, upd_blocks, moment_dtype=dtype,
                                              **paging)

    arms = {"fp32": arm(torch.float32), "bf16": arm(torch.bfloat16)}
    for st, _ in arms.values():
        st[0].copy_(arms["fp32"][0][0])
    for _, fn in arms.values():
        fn()
    torch.cuda.synchronize()
    # from zero moments both launches compute the weights from the same fp32 moments
    same_weights = torch.equal(arms["fp32"][0][0], arms["bf16"][0][0])
    times = {name: [] for name in arms}
    for _ in range(repeats):
        for name, (_, fn) in arms.items():
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    assert comm.errored() is None
    W, kk = comm.world, min(k, comm.world)
    nvec = nelem // 8
    per = (nvec + W - 1) // W
    primary = 8 * min(per, nvec)  # rank 0's primary slice; it also updates the kk - 1 slices it backs up
    updated = sum(8 * (min((s + 1) * per, nvec) - min(s * per, nvec)) for s in {(0 - j) % W for j in range(kk)})
    out = {"timing": "local HBM (virtual ranks), not NVLink", "state": "paged_ordered" if paged else "flat",
           "first_update_weights_equal": same_weights, "elements_updated": updated,
           "pushed_bytes": 2 * primary * (W - kk)}
    for name, ts in times.items():
        ts = sorted(ts)
        per_elem = 2 + 8 + 2 + 4 * (2 if name == "bf16" else 4)
        moved = per_elem * updated + out["pushed_bytes"]
        out[f"adamw_allgather_{name}_moments"] = {
            "ms": {"median": round(ts[len(ts) // 2], 4), "min": round(ts[0], 4), "max": round(ts[-1], 4)},
            "state_bytes_per_element": per_elem, "bytes_moved": moved,
            "gb_per_s_at_median": round(moved / ts[len(ts) // 2] / 1e6, 1)}
    out["bf16_over_fp32"] = round(out["adamw_allgather_bf16_moments"]["ms"]["median"]
                                  / out["adamw_allgather_fp32_moments"]["ms"]["median"], 4)
    return out


def ema_ab(comm, nelem, k, upd_blocks, iters, warmup, repeats, paged, shift=16):
    """The update of one unit without and with an EMA of the weights, for fp32 and for bf16 moments (the EMA takes the
    moments' type), the four arms timed alternately, on flat state or on page pools in slot order. Before timing, one
    launch of each pair from the same state must give the same weights: the EMA does not change the update."""
    from torchft_b200.parallel.zero1 import ema_coefficient

    upd_blocks = upd_blocks or comm._K.NUM_SMS * 16
    dev = comm.device
    grad = comm.segment("z1_grad")[: nelem * 2].view(torch.bfloat16)
    grad.normal_()
    gate = torch.ones(2, dtype=torch.int32, device=dev)
    npages = (nelem + (1 << shift) - 1) >> shift
    n_state = npages << shift if paged else nelem
    table = torch.arange(npages, dtype=torch.int32, device=dev)
    paging = dict(table=table.data_ptr(), page_shift=shift) if paged else {}
    c = ema_coefficient(0.999)
    init = torch.randn(n_state, device=dev)

    def state(dtype):
        return [init.clone(), torch.zeros(n_state, device=dev, dtype=dtype), torch.zeros(n_state, device=dev, dtype=dtype),
                init.to(dtype)]

    def launch(st, dtype, ema):
        kw = dict(ema=st[3].data_ptr(), ema_c=c) if ema else {}
        return lambda: comm.zero1_update_("z1_param", 0, grad.data_ptr(), st[0].data_ptr(), st[1].data_ptr(),
                                          st[2].data_ptr(), nelem, HP, gate, k, 0, upd_blocks, moment_dtype=dtype,
                                          **paging, **kw)

    arms, same = {}, {}
    for name, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        off, on = state(dtype), state(dtype)
        launch(off, dtype, False)()
        launch(on, dtype, True)()
        torch.cuda.synchronize()
        same[name] = torch.equal(off[0], on[0])
        assert same[name], f"{name} moments: the update with an EMA computed other weights than the one without"
        arms[f"{name}_off"], arms[f"{name}_ema"] = launch(off, dtype, False), launch(on, dtype, True)
    times = {name: [] for name in arms}
    for _ in range(repeats):
        for name, fn in arms.items():
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    assert comm.errored() is None
    W, kk = comm.world, min(k, comm.world)
    nvec = nelem // 8
    per = (nvec + W - 1) // W
    primary = 8 * min(per, nvec)
    updated = sum(8 * (min((s + 1) * per, nvec) - min(s * per, nvec)) for s in {(0 - j) % W for j in range(kk)})
    out = {"timing": "local HBM (virtual ranks), not NVLink", "state": "paged_ordered" if paged else "flat",
           "first_update_weights_equal": same, "elements_updated": updated, "pushed_bytes": 2 * primary * (W - kk)}
    for name, ts in times.items():
        ts = sorted(ts)
        msize = 2 if name.startswith("bf16") else 4
        per_elem = 2 + 8 + 2 + 4 * msize + (2 * msize if name.endswith("ema") else 0)  # the EMA is read and written
        moved = per_elem * updated + out["pushed_bytes"]
        out[f"adamw_allgather_{name}"] = {
            "ms": {"median": round(ts[len(ts) // 2], 4), "min": round(ts[0], 4), "max": round(ts[-1], 4)},
            "state_bytes_per_element": per_elem, "bytes_moved": moved,
            "gb_per_s_at_median": round(moved / ts[len(ts) // 2] / 1e6, 1)}
    for name in ("fp32", "bf16"):
        out[f"{name}_ema_over_off"] = round(out[f"adamw_allgather_{name}_ema"]["ms"]["median"]
                                            / out[f"adamw_allgather_{name}_off"]["ms"]["median"], 4)
    return out


def accum_ab(comms, nelem, k, rs_blocks, iters, warmup, repeats):
    """Rank 0's reduce-scatter of one unit in the three accumulation modes, timed alternately: ``off`` (today's launch),
    ``acc`` (a middle micro-batch: fp32 rank sum added into the accumulator) and ``last`` (accumulator + rank sum,
    scaled, rounded to bf16 and pushed to the buddies). Before timing, a first + last pair over the same gradients with
    half the scale must give the ``off`` result bit for bit (2s * scale/2 == s * scale exactly), and slice 0 must equal
    the PyTorch reference bf16(fp32 rank sum * scale). At world 1 there is no ``off`` kernel (the optimizer scales on
    the host), so only the reference is checked."""
    from torchft_b200.parallel.zero1 import ShardLayout, accum_offsets

    comm = comms[0]
    peers = [c.segment("z1_grad")[: nelem * 2].view(torch.bfloat16) for c in comms]
    for p in peers:
        p.normal_()
    L = ShardLayout(((0, nelem),), k)
    _, n = accum_offsets(L, comm.rank, comm.world)
    lo, hi = L.slice_bounds(0, comm.world, comm.rank)
    acc = torch.zeros(n + 8, device=comm.device)
    scale = 1.0 / comm.world
    saved = [p.clone() for p in peers]
    rank_sum = saved[0][lo:hi].float()
    for p in saved[1:]:
        rank_sum = rank_sum + p[lo:hi].float()
    expect = (rank_sum * torch.tensor(scale, dtype=torch.float32, device=comm.device)).bfloat16()

    def launch(mode, sc=scale):
        return lambda: comm.zero1_reduce_scatter_("z1_grad", 0, nelem, sc, True, k, rs_blocks, acc=acc.data_ptr(),
                                                  acc_mode=mode)

    has_off = comm.world > 1
    if has_off:
        launch(0)()
        torch.cuda.synchronize()
        ref = [p.clone() for p in peers]
        for p, x in zip(peers, saved):
            p.copy_(x)
    launch(1, scale / 2)()
    launch(3, scale / 2)()
    torch.cuda.synchronize()
    same = all(torch.equal(p, r) for p, r in zip(peers, ref)) if has_off else None
    matches_ref = torch.equal(peers[0][lo:hi], expect)
    arms = ((("off", launch(0)),) if has_off else ()) + (("acc", launch(2)), ("last", launch(3)))
    times = {name: [] for name, _ in arms}
    for _ in range(repeats):
        for name, fn in arms:
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    assert comm.errored() is None
    out = {"timing": "local HBM (virtual ranks), not NVLink", "accum_equals_off": same, "accum_matches_reference": matches_ref,
           "accum_bytes": 4 * n}
    for name, ts in times.items():
        ts = sorted(ts)
        out[f"reduce_{name}_ms"] = {"median": round(ts[len(ts) // 2], 4), "min": round(ts[0], 4), "max": round(ts[-1], 4)}
    for name in ("acc", "last") if has_off else ():
        out[f"{name}_over_off"] = round(out[f"reduce_{name}_ms"]["median"] / out["reduce_off_ms"]["median"], 4)
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
    ap.add_argument("--compact", action="store_true", help="--virtual: A/B the update on flat vs paged optimizer state")
    ap.add_argument("--clip", action="store_true", help="--virtual: A/B one unit's pipeline without and with gradient clipping")
    ap.add_argument("--accum", action="store_true", help="--virtual: A/B rank 0's reduce in accumulation modes off / acc / last")
    ap.add_argument("--sched", action="store_true", help="--virtual: A/B the update without and with a learning-rate "
                    "table and weight-decay exemptions")
    ap.add_argument("--moments", action="store_true", help="--virtual: A/B the update with fp32 and bf16 moments "
                    "(with --compact: on paged state)")
    ap.add_argument("--ema", action="store_true", help="--virtual: A/B the update without and with an EMA of the weights, "
                    "for fp32 and bf16 moments (with --compact: on paged state)")
    ap.add_argument("--repeats", type=int, default=5, help="--compact / --clip / --accum / --sched / --moments / --ema: "
                    "alternations of the arms")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    nelem = int(a.mb * (1 << 20)) // 2 // 4096 * 4096
    S = nelem * 2

    if a.virtual:
        torch.cuda.set_device(0)
        segments = {"z1_grad": S, "z1_param": S, **({"z1_gnorm": 8} if a.clip else {})}
        comms = SymmetricComm.virtual_world(a.virtual, segments, presignal=True)
        res = {"mode": f"virtual{a.virtual}", "unit_mb": S / 2**20}
        if a.compact or a.clip or a.accum or a.sched or a.moments or a.ema:
            if a.ema:
                res.update(ema_ab(comms[0], nelem, a.replication, a.upd_blocks, a.iters, a.warmup, a.repeats, a.compact))
            elif a.moments:
                res.update(moments_ab(comms[0], nelem, a.replication, a.upd_blocks, a.iters, a.warmup, a.repeats, a.compact))
            elif a.compact:
                res.update(compact_ab(comms[0], nelem, a.replication, a.upd_blocks, a.iters, a.warmup, a.repeats))
            elif a.sched:
                res.update(sched_ab(comms[0], nelem, a.replication, a.upd_blocks, a.iters, a.warmup, a.repeats))
            elif a.accum:
                res.update(accum_ab(comms, nelem, a.replication, a.rs_blocks, a.iters, a.warmup, a.repeats))
            else:
                res.update(clip_ab(comms[0], nelem, a.replication, a.rs_blocks, a.upd_blocks, a.iters, a.warmup, a.repeats))
            res.update(gpu_info())
            print("ZERO1_BENCH " + json.dumps(res), flush=True)
            if a.out:
                os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
                with open(a.out, "w") as f:
                    json.dump(res, f, indent=1)
            return
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
