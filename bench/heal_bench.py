"""Kill / rejoin benchmark (BASELINE.md config 4): step-time overhead of a replica drop and of a live heal.

Orchestrator (no torchrun): starts a Lighthouse, spawns one trainer process per GPU,
SIGKILLs replica `--victim` when the survivors reach step `--kill-at`, respawns it when
they reach `--rejoin-at`, and collects per-step logs.

    python bench/heal_bench.py --gpus 2 --model llama3_1b --kill-at 6 --rejoin-at 12 --steps 20

Reports: steady step time before the kill, the stall caused by the drop (survivor's
collective times out -> commit fails -> lighthouse drops the dead replica -> remap),
steps lost, the heal transfer size / time / GB/s (NVLink P2P pull by a copy kernel,
vs. the 450 GB/s per-direction NVLink 4 rate of the H100 data sheet), and the step time of the step that carried the heal.
"""

from __future__ import annotations

import argparse
import json
import os
import signal
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def worker(args: argparse.Namespace) -> None:
    import torch
    from datetime import timedelta

    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    torch.cuda.set_device(args.device)
    log = open(args.log, "a", buffering=1)
    t_start = time.time()
    trainer = FaultTolerantTrainer(args.model, args.lighthouse, replica_id=f"replica_{args.replica}",
                                   min_replica_size=1, backend=args.backend, timeout=timedelta(seconds=args.timeout),
                                   device=torch.device("cuda", args.device), init_sync=True)
    cfg = trainer.cfg
    tok = torch.randint(0, cfg.vocab_size, (1, args.seq)).pin_memory()
    tgt = torch.randint(0, cfg.vocab_size, (1, args.seq)).pin_memory()
    log.write(json.dumps({"event": "ready", "replica": args.replica, "t": time.time(), "setup_s": time.time() - t_start}) + "\n")
    while trainer.manager.current_step() < args.steps:
        t0 = time.time()
        before = trainer.manager.current_step()
        loss = trainer.step(tok, tgt)
        torch.cuda.synchronize()
        m = trainer.manager
        tr = m._checkpoint_transport
        rec = {"event": "step", "replica": args.replica, "t": time.time(), "ms": (time.time() - t0) * 1e3,
               "step_before": before, "step_after": m.current_step(), "participants": m.num_participants(),
               "quorum_id": m._quorum_id, "loss": loss, "committed": m.current_step() > before,
               "psum": _checksum(trainer.flat.param)}  # exact checksum of ALL weights
        if getattr(trainer, "zopt", None) is not None:
            rec["z1_pulled_bytes"] = trainer.zopt.pulled_bytes
            rec["z1_lost_elements"] = trainer.zopt.lost_elements
            rec["z1_t"] = trainer.zopt.t
        if getattr(tr, "last_recv_bytes", 0):
            rec["heal_bytes"] = tr.last_recv_bytes
            rec["heal_ms"] = tr.last_recv_ms
            tr.last_recv_bytes = 0
        log.write(json.dumps(rec) + "\n")
    log.write(json.dumps({"event": "done", "replica": args.replica, "t": time.time()}) + "\n")
    trainer.shutdown()


def _checksum(t) -> int:
    """Exact integer checksum of a bf16 buffer, in 256M-element chunks (a one-shot int64 reduction would need 4x the memory)."""
    import torch

    v = t.view(torch.int16)
    return sum(int(v[i: i + (1 << 28)].sum(dtype=torch.int64).item()) for i in range(0, v.numel(), 1 << 28))


def _weights_match(a: list, b: list):
    pa = {e["step_after"]: e["psum"] for e in a if e.get("committed")}
    pb = {e["step_after"]: e["psum"] for e in b if e.get("committed")}
    common = sorted(set(pa) & set(pb))
    if not common:
        return None
    return all(pa[s] == pb[s] for s in common[-3:])


def read_log(path: str) -> list:
    out = []
    try:
        with open(path) as f:
            for line in f:
                line = line.strip()
                if line:
                    out.append(json.loads(line))
    except FileNotFoundError:
        pass
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--role", default="orchestrator")
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--kill-at", type=int, default=6)
    ap.add_argument("--rejoin-at", type=int, default=12)
    ap.add_argument("--victim", type=int, default=1)
    ap.add_argument("--backend", default="b200")
    ap.add_argument("--timeout", type=float, default=5.0)
    ap.add_argument("--heartbeat-timeout-ms", type=int, default=2000)
    ap.add_argument("--out", default="gpurun_out/heal_bench.json")
    ap.add_argument("--replica", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--lighthouse", default="")
    ap.add_argument("--log", default="")
    args = ap.parse_args()
    if args.role == "worker":
        worker(args)
        return

    from torchft_b200.bench_utils import loopback
    from torchft_b200.coordination import LighthouseServer

    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    lh = LighthouseServer(bind="[::]:0", min_replicas=1, join_timeout_ms=3000, heartbeat_timeout_ms=args.heartbeat_timeout_ms)
    addr = loopback(lh.address())
    logs = [os.path.join(os.path.dirname(args.out) or ".", f"heal_replica{r}.jsonl") for r in range(args.gpus)]
    for p in logs:
        if os.path.exists(p):
            os.remove(p)

    def spawn(r: int) -> subprocess.Popen:
        cmd = [sys.executable, os.path.abspath(__file__), "--role", "worker", "--replica", str(r), "--device", str(r),
               "--lighthouse", addr, "--log", logs[r], "--model", args.model, "--seq", str(args.seq), "--steps",
               str(args.steps), "--backend", args.backend, "--timeout", str(args.timeout)]
        return subprocess.Popen(cmd, stdout=open(logs[r] + ".out", "a"), stderr=subprocess.STDOUT)

    procs = {r: spawn(r) for r in range(args.gpus)}
    survivor = 0 if args.victim != 0 else 1
    killed_t = rejoin_t = None
    deadline = time.time() + 1500
    try:
        while time.time() < deadline:
            time.sleep(0.2)
            steps = [e for e in read_log(logs[survivor]) if e["event"] == "step"]
            cur = steps[-1]["step_after"] if steps else 0
            if killed_t is None and cur >= args.kill_at:
                procs[args.victim].send_signal(signal.SIGKILL)
                procs[args.victim].wait()
                killed_t = time.time()
            if killed_t is not None and rejoin_t is None and cur >= args.rejoin_at:
                procs[args.victim] = spawn(args.victim)
                rejoin_t = time.time()
            if all(p.poll() is not None for p in procs.values()):
                break
            if procs[survivor].poll() is not None and procs[survivor].returncode != 0:
                break
    finally:
        for p in procs.values():
            if p.poll() is None:
                p.kill()
        lh.shutdown()

    sv = [e for e in read_log(logs[survivor]) if e["event"] == "step"]
    vc = [e for e in read_log(logs[args.victim]) if e["event"] == "step"]
    steady = sorted(e["ms"] for e in sv if e["participants"] == args.gpus and e["committed"] and e["t"] < (killed_t or 1e18))[2:]
    after_kill = [e for e in sv if killed_t and e["t"] > killed_t]
    failed = [e for e in after_kill if not e["committed"]]
    solo = sorted(e["ms"] for e in after_kill if e["committed"] and e["participants"] == args.gpus - 1)
    heals = [e for e in vc if e.get("heal_bytes")]
    rejoined = [e for e in sv if rejoin_t and e["t"] > rejoin_t and e["participants"] == args.gpus and e["committed"]]
    first_full = rejoined[0] if rejoined else None
    res = {
        "config": vars(args) | {"role": None},
        "survivor_rc": procs[survivor].returncode, "victim_rc": procs[args.victim].returncode,
        "steady_ms_before_kill": round(sum(steady) / max(len(steady), 1), 1) if steady else None,
        "drop": {
            "failed_commits": len(failed),
            "stall_ms_total": round(sum(e["ms"] for e in failed), 1),
            "first_step_after_kill_ms": round(after_kill[0]["ms"], 1) if after_kill else None,
            "solo_step_ms": round(solo[len(solo) // 2], 1) if solo else None,
        },
        "heal": {
            "bytes": heals[0]["heal_bytes"] if heals else None,
            "copy_ms": round(heals[0]["heal_ms"], 2) if heals else None,
            "gbs": round(heals[0]["heal_bytes"] / heals[0]["heal_ms"] / 1e6, 1) if heals else None,
            "frac_of_nvlink": round(heals[0]["heal_bytes"] / heals[0]["heal_ms"] / 1e6 / 450, 3) if heals else None,
            "victim_first_step_ms": round(vc[0]["ms"], 1) if vc else None,
            "survivor_step_ms_during_heal": round(first_full["ms"], 1) if first_full else None,
            "victim_restart_to_ready_s": next((round(e["setup_s"], 1) for e in read_log(logs[args.victim]) if e["event"] == "ready" and rejoin_t and e["t"] > rejoin_t), None),
        },
        "final_steps": {"survivor": sv[-1]["step_after"] if sv else None, "victim": vc[-1]["step_after"] if vc else None},
        # replicas must hold bit-identical weights at equal committed steps (oracle of the
        # reference's integration tests: state_dict equality after injected failures)
        "weights_match_at_common_steps": _weights_match(sv, vc),
        "zero1": {"victim_reshard_pulled_gb": round(max((e.get("z1_pulled_bytes", 0) for e in vc), default=0) / 1e9, 2),
                  "survivor_reshard_pulled_gb": round(max((e.get("z1_pulled_bytes", 0) for e in sv), default=0) / 1e9, 2),
                  "lost_elements": max((e.get("z1_lost_elements", 0) for e in sv + vc), default=0)},
    }
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("HEAL_BENCH " + json.dumps({k: res[k] for k in ("steady_ms_before_kill", "drop", "heal", "final_steps", "survivor_rc", "victim_rc",
                                                               "weights_match_at_common_steps", "zero1")}))


if __name__ == "__main__":
    main()
