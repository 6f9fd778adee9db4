"""Job launch helpers: one torchrun role per replica group.

Parity with the reference's torchx component ``hsdp`` (upstream torchft/torchx.py:17-89):
each replica group is launched as its own ``torchrun`` with ``--master_port=29600+id`` and the
environment ``REPLICA_GROUP_ID`` / ``NUM_REPLICA_GROUPS`` / ``TORCHFT_LIGHTHOUSE``; process
restarts are delegated to torchelastic's ``--max_restarts``. torchx is not available in this
image, so :func:`hsdp` returns a plain, scheduler-agnostic job spec (list of :class:`Role`) and
:func:`launch_local` runs it on the local node (one group per GPU subset).

    python -m torchft_b200.launcher --replicas 4 --workers-per-replica 2 train.py -- --my-arg 1
"""

from __future__ import annotations

import argparse
import os
import signal
import subprocess
import sys
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional


@dataclass
class Role:
    """One launchable unit (a torchrun invocation for one replica group) of a job spec; mirrors ``torchx.specs.Role``."""

    name: str
    entrypoint: str
    args: List[str]
    env: Dict[str, str] = field(default_factory=dict)
    num_replicas: int = 1
    max_retries: int = 0


def hsdp(*script_args: str, replicas: int = 2, workers_per_replica: int = 1, max_restarts: int = 10,
         script: str = "train_ddp.py", env: Optional[Dict[str, str]] = None, lighthouse: Optional[str] = None,
         base_port: int = 29600, gpus_per_node: Optional[int] = None) -> List[Role]:
    """Job spec for fault-tolerant HSDP: ``replicas`` replica groups x ``workers_per_replica`` ranks."""

    env = dict(env or {})
    lighthouse = lighthouse or os.environ.get("TORCHFT_LIGHTHOUSE", "http://127.0.0.1:29510")
    roles = []
    for rid in range(replicas):
        renv = dict(env, REPLICA_GROUP_ID=str(rid), NUM_REPLICA_GROUPS=str(replicas), TORCHFT_LIGHTHOUSE=lighthouse,
                    TORCH_NCCL_ASYNC_ERROR_HANDLING="1")
        if gpus_per_node is not None:
            first = (rid * workers_per_replica) % gpus_per_node
            renv["CUDA_VISIBLE_DEVICES"] = ",".join(str(first + i) for i in range(workers_per_replica))
        roles.append(Role(
            name=f"replica_group_{rid}",
            entrypoint=sys.executable,
            args=["-m", "torch.distributed.run", "--nnodes=1", f"--nproc_per_node={workers_per_replica}",
                  f"--max_restarts={max_restarts}", "--master_addr=127.0.0.1", f"--master_port={base_port + rid}",
                  script, *script_args],
            env=renv, num_replicas=1, max_retries=0))
    return roles


def launch_local(roles: List[Role], poll_s: float = 1.0, relaunch: bool = False) -> int:
    """Run every role as a local subprocess; with ``relaunch`` dead groups are restarted (a poor
    man's scheduler, like the reference's slurm runner loop). Returns the worst exit code."""

    procs: Dict[str, subprocess.Popen] = {}

    def start(r: Role) -> None:
        procs[r.name] = subprocess.Popen([r.entrypoint, *r.args], env=dict(os.environ, **r.env))

    for r in roles:
        start(r)
    worst = 0
    try:
        while procs:
            time.sleep(poll_s)
            for r in roles:
                p = procs.get(r.name)
                if p is None or p.poll() is None:
                    continue
                if p.returncode != 0 and relaunch:
                    start(r)
                else:
                    worst = max(worst, abs(p.returncode))
                    del procs[r.name]
    except KeyboardInterrupt:
        for p in procs.values():
            p.send_signal(signal.SIGINT)
    return worst


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--replicas", type=int, default=2)
    ap.add_argument("--workers-per-replica", type=int, default=1)
    ap.add_argument("--max-restarts", type=int, default=10)
    ap.add_argument("--lighthouse", default=None)
    ap.add_argument("--gpus-per-node", type=int, default=None)
    ap.add_argument("--relaunch", action="store_true")
    ap.add_argument("--dry-run", action="store_true")
    ap.add_argument("script")
    ap.add_argument("script_args", nargs="*")
    a = ap.parse_args()
    roles = hsdp(*a.script_args, replicas=a.replicas, workers_per_replica=a.workers_per_replica,
                 max_restarts=a.max_restarts, script=a.script, lighthouse=a.lighthouse, gpus_per_node=a.gpus_per_node)
    if a.dry_run:
        for r in roles:
            print(r.name, " ".join([r.entrypoint, *r.args]), {k: r.env[k] for k in sorted(r.env)})
        return
    raise SystemExit(launch_local(roles, relaunch=a.relaunch))


if __name__ == "__main__":
    main()
