"""FT-ZeRO-1 durable checkpoints: what a save costs the training step, and how fast snapshot, write and restore run.

    python bench/ckpt_bench.py --model llama3_1b --seq 4096 --batch 1 --steps 4 --saves 3 [--virtual 8]

One trainer at world 1. ``--virtual W`` snapshots only quorum rank 0's share at a world of ``W`` (its primary slices,
about ``14 * numel / W`` bytes), which is what each replica of a ``W``-replica job copies and writes. Measured in one
process, arms alternated:

* ``step_ms.plain``: device-timed steps (CUDA events around the step and its update) after a settled step;
* ``step_ms.after_save``: the same, for the step enqueued right after a save, whose update of each unit waits for that
  unit's snapshot copy while its forward and backward run under the copy;
* ``snapshot``: the device-to-host copy of the share into pinned memory, host-timed to the copy's completion (GB/s);
* ``write_s``: the background write (header, payload, fsync, rename) to a temporary directory;
* ``restore_s``: reading the share back into the device arrays (disk -> pinned bounce buffers -> H2D). The file was
  just written, so it is usually served from the page cache.

Prints one ``CKPT_BENCH {json}`` line with the card's name and power limit. Files go to a temporary directory that is
removed at the end.
"""

from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time
from datetime import timedelta

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _median(xs):
    xs = sorted(xs)
    return round(xs[len(xs) // 2], 2) if xs else None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--virtual", type=int, default=1, help="snapshot quorum rank 0's share at this world")
    ap.add_argument("--steps", type=int, default=4, help="plain timed steps per round")
    ap.add_argument("--saves", type=int, default=3, help="rounds, each ending with one save and its timed next step")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dir", default="", help="parent of the temporary checkpoint directory (default: the system's)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.parallel.trainer import FaultTolerantTrainer
    from torchft_b200.parallel.zero1 import ckpt_read_plan, intersect_ranges, total
    from zero1_bench import gpu_info  # noqa: E402 - bench/ is the script's directory

    if not 1 <= a.virtual <= 8:
        raise SystemExit("--virtual must be in [1, 8]")
    torch.cuda.set_device(0)
    lh = local_lighthouse()
    tr = FaultTolerantTrainer(a.model, loopback(lh.address()), replica_id="ckpt_0", timeout=timedelta(seconds=120))
    z = tr.zopt
    gen = torch.Generator().manual_seed(1234)
    tok = torch.randint(0, tr.cfg.vocab_size, (a.batch, a.seq), generator=gen).to("cuda")
    tgt = torch.randint(0, tr.cfg.vocab_size, (a.batch, a.seq), generator=gen).to("cuda")
    root = tempfile.mkdtemp(prefix="z1ckpt_", dir=a.dir or None)
    cur = torch.cuda.current_stream()

    def timed_step():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(cur)
        tr.step_device(tok, tgt)
        tr.join()
        e1.record(cur)
        e1.synchronize()
        return e0.elapsed_time(e1)

    def settle():
        ms = tr.manager.state_dict()  # resolves the last verdict
        torch.cuda.synchronize()
        return ms

    share = intersect_ranges(z.layout.primary(0, a.virtual), [(0, z.numel)])
    res = {"model": a.model, "seq": a.seq, "batch": a.batch, "virtual_world": a.virtual, "numel": z.numel,
           "share_elements": total(share), "share_bytes": 14 * total(share)}
    try:
        for _ in range(a.warmup):
            tr.step_device(tok, tgt)
        settle()
        plain, after, snap_s, write_s = [], [], [], []
        for _ in range(a.saves):
            for _ in range(a.steps):
                settle()
                plain.append(timed_step())
            ms = settle()
            t0 = time.perf_counter()
            z._save(root, share, 0, a.virtual, ms, tr._opt_events, keep=1)
            after.append(timed_step())  # enqueued while the snapshot copy runs
            z._snap_done.synchronize()
            snap_s.append(time.perf_counter() - t0)
            t1 = time.perf_counter()
            z.wait_checkpoint()
            write_s.append(time.perf_counter() - t1)
        # snapshot alone (nothing else queued), for the copy rate
        ms = settle()
        t0 = time.perf_counter()
        z._save(root, share, 0, a.virtual, ms, tr._opt_events, keep=1)
        z._snap_done.synchronize()
        alone = time.perf_counter() - t0
        z.wait_checkpoint()
        from torchft_b200.checkpointing.sharded import scan

        files = [(h, [tuple(r) for r in h["ranges"]]) for h in scan(root)]
        settle()
        t0 = time.perf_counter()
        z._read_ranges(ckpt_read_plan(share, files), ("param", "master", "m", "v"))
        restore = time.perf_counter() - t0
        gb = 14 * total(share) / 1e9
        res.update({
            "step_ms": {"plain": _median(plain), "after_save": _median(after), "plain_all": [round(x, 2) for x in plain],
                        "after_save_all": [round(x, 2) for x in after]},
            "snapshot": {"alone_s": round(alone, 3), "alone_GBps": round(gb / alone, 2),
                         "under_step_s": _median(snap_s), "under_step_GBps": round(gb / _median(snap_s), 2)},
            "write_s": _median(write_s), "write_GBps": round(gb / _median(write_s), 2),
            "restore_s": round(restore, 3), "restore_GBps": round(gb / restore, 2),
            "staging_gib": round(z.snapshot_bytes() / 2**30, 2)})
    finally:
        shutil.rmtree(root, ignore_errors=True)
    res.update(gpu_info())
    print("CKPT_BENCH " + json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    tr.shutdown()
    lh.shutdown()


if __name__ == "__main__":
    main()
