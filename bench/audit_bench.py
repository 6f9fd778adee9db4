"""The FT-ZeRO-1 replica audit's digest kernel alone, on one rank's share of a Llama-3 model.

At ``--virtual W`` replicas with ``k`` holders per slice one rank digests every bf16 weight of the model and its k/W of
the optimizer state (fp32 master, m and v of the moment type). This times exactly that digest launch with CUDA events
after a warm-up, for flat state and for paged state (page pools in random slot order), with fp32 and bf16 moments. Bytes
read count the weights and the held state once; the fraction is of the H100 SXM data-sheet HBM bandwidth of 3.35 TB/s.
The card's name and power limit are read in the same run.

With ``--trainer-model`` it then times training steps with ``audit_every=1`` against the audit off, in blocks that
alternate within the same two processes (``bench/audit_replica.py``): two FT-ZeRO-1 replicas on a local lighthouse,
k = 2 (two llama3_1b replicas do not fit beside each other on one 80 GB GPU). Both replicas share this one GPU, so the step time includes their time-slicing; what it shows is what the audit
adds to a step, not how it overlaps the forward on a GPU of its own.

    python bench/audit_bench.py [--model llama3_1b] [--virtual 8] [--k 2] [--iters 20] [--ctas-per-sm 3]
                                [--trainer-model llama3_debug --trainer-blocks 4] [--out results.json]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.models.llama import CONFIGS, Llama  # noqa: E402
from torchft_b200.ops import _native  # noqa: E402
from torchft_b200.parallel.zero1 import AUDIT_SEEDS, PAGE_SHIFT  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[torch.cuda.current_device()].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def table(rows, cw):
    out, c = [], 0
    for r in rows:
        out.append(tuple(r) + (c,))
        c += (r[4] + cw - 1) // cw
    return torch.tensor(out, dtype=torch.int64, device="cuda"), len(out), c


def trainer_steps(a: argparse.Namespace) -> dict:
    """Per-step milliseconds with the audit off and on (``audit_every=1``), alternating blocks of 5 steps after 3 warm-up
    steps, median over the blocks and the two replicas."""
    import statistics
    import tempfile

    from torchft_b200.bench_utils import local_lighthouse, loopback

    here = os.path.dirname(os.path.abspath(__file__))
    lh = local_lighthouse(min_replicas=2)
    with tempfile.TemporaryDirectory() as d:
        try:
            procs = [subprocess.Popen([sys.executable, os.path.join(here, "audit_replica.py"), "--lighthouse",
                                       loopback(lh.address()), "--replica", str(r), "--model", a.trainer_model,
                                       "--batch", str(a.trainer_batch), "--seq", str(a.trainer_seq), "--steps", "3", "--bench-blocks",
                                       str(a.trainer_blocks), "--out", os.path.join(d, f"r{r}.json")]) for r in range(2)]
            for p in procs:
                if p.wait(timeout=1200) != 0:
                    raise RuntimeError(f"replica exited with {p.returncode}")
        finally:
            lh.shutdown()
        reps = [json.load(open(os.path.join(d, f"r{r}.json"))) for r in range(2)]
    out = {m: round(statistics.median([x for r in reps for x in r["ms_per_step"][m]]), 2) for m in ("off", "on")}
    out["audits"] = [r["audits"] for r in reps]
    out["divergences"] = [r["divergences"] for r in reps]
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--virtual", type=int, default=8)
    ap.add_argument("--k", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ctas-per-sm", type=int, default=3, help="digest grid (the optimizer launches 3 per SM)")
    ap.add_argument("--trainer-model", default="")
    ap.add_argument("--trainer-blocks", type=int, default=4)
    ap.add_argument("--trainer-seq", type=int, default=128)
    ap.add_argument("--trainer-batch", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    K = _native.load()
    cw = int(K.Z1_DIGEST_CHUNK_WORDS)
    numel = sum(p.numel() for p in Llama(CONFIGS[a.model], device="meta").parameters()) // 8 * 8
    share = (numel * a.k // a.virtual) // 8 * 8  # the state elements one rank holds
    page = 1 << PAGE_SHIFT
    param = torch.empty(numel, dtype=torch.bfloat16, device="cuda").random_()
    slots = torch.zeros(64, dtype=torch.int64, device="cuda")
    results = []
    for mdt in (torch.float32, torch.bfloat16):
        arrays = {"master": torch.empty(share, dtype=torch.float32, device="cuda").random_(),
                  "m": torch.empty(share, dtype=mdt, device="cuda").random_(),
                  "v": torch.empty(share, dtype=mdt, device="cuda").random_()}
        npages = (share + page - 1) // page
        perm = torch.randperm(npages, generator=torch.Generator().manual_seed(0)).to(torch.int32).cuda()
        for paged in (False, True):
            rows = [(param.data_ptr(), 0, 0, 0, numel // 4, AUDIT_SEEDS["weights"], 0)]
            for i, (name, x) in enumerate(arrays.items()):
                es = x.element_size()
                pbs = PAGE_SHIFT + es.bit_length() - 1
                rows.append((x.data_ptr(), perm.data_ptr() if paged else 0, pbs if paged else 0, 0, share * es // 8,
                             AUDIT_SEEDS[name], 1 + i))
            tab, n, chunks = table(rows, cw)
            grid = max(1, min(chunks, K.NUM_SMS * a.ctas_per_sm))
            s = torch.cuda.current_stream().cuda_stream

            def run():
                K.z1_digest(tab.data_ptr(), n, chunks, slots.data_ptr(), grid, s)

            for _ in range(3):
                run()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.iters):
                run()
            t1.record()
            torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / a.iters
            nbytes = 2 * numel + sum(x.element_size() for x in arrays.values()) * share
            r = {"moments": "bf16" if mdt == torch.bfloat16 else "fp32", "state": "paged" if paged else "flat",
                 "bytes": nbytes, "ms": round(ms, 4), "TB/s": round(nbytes / ms / 1e9, 3),
                 "of_3.35TB/s": round(nbytes / ms / 1e9 / (HBM_BYTES_PER_S / 1e12), 3)}
            results.append(r)
            print(f"digest {a.model} W={a.virtual} k={a.k} moments={r['moments']:4s} {r['state']:5s}: "
                  f"{nbytes / 1e9:.2f} GB in {ms:.3f} ms = {r['TB/s']:.2f} TB/s ({100 * r['of_3.35TB/s']:.0f} %)")
        del arrays
    del param
    torch.cuda.empty_cache()
    out = {"card": card(), "model": a.model, "numel": numel, "virtual": a.virtual, "k": a.k,
           "ctas_per_sm": a.ctas_per_sm, "digest": results}
    if a.trainer_model:
        out["trainer"] = trainer_steps(a)
        print(f"trainer {a.trainer_model}, two replicas on one GPU: ms/step audit off {out['trainer']['off']} "
              f"on {out['trainer']['on']}")
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
