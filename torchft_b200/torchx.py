"""torchx component: ``torchx run -- -j 4x8 torchft_b200/torchx.py:hsdp --script train.py``.

Parity with the reference's ``torchft/torchx.py:17-89`` + ``.torchxconfig``. The job shape is
computed once by :func:`torchft_b200.launcher.hsdp` (one torchrun role per replica group,
``--master_port=29600+id``, env ``REPLICA_GROUP_ID / NUM_REPLICA_GROUPS / TORCHFT_LIGHTHOUSE``);
this module only converts that scheduler-agnostic spec into ``torchx.specs`` objects. torchx is
not part of this image, so the import is lazy and :func:`hsdp_spec` is available without it.
"""

from __future__ import annotations

import os
from typing import Any, Dict, List, Optional

from torchft_b200.launcher import Role, hsdp as hsdp_spec

__all__ = ["hsdp", "hsdp_spec"]


def hsdp(*script_args: str, replicas: int = 2, workers_per_replica: int = 1, max_restarts: int = 10,
         script: str = "train_ddp.py", env: Optional[Dict[str, str]] = None, image: str = "",
         h: Optional[str] = None, cpu: int = 2, gpu: int = 0, memMB: int = 1024) -> Any:
    """Build a ``torchx.specs.AppDef`` for fault-tolerant HSDP on H100 nodes.

    Args mirror the reference component; ``h`` is a torchx named resource, otherwise
    ``cpu/gpu/memMB`` are used. Raises ``ImportError`` when torchx is not installed.
    """

    try:
        from torchx import specs  # type: ignore[import-not-found]
    except ImportError as e:
        raise ImportError("torchx is not installed; use `python -m torchft_b200.launcher` or hsdp_spec()") from e
    roles: List[Role] = hsdp_spec(*script_args, replicas=replicas, workers_per_replica=workers_per_replica,
                                 max_restarts=max_restarts, script=script, env=env,
                                 lighthouse=os.environ.get("TORCHFT_LIGHTHOUSE"))
    resource = specs.resource(cpu=cpu, gpu=gpu, memMB=memMB, h=h)
    return specs.AppDef(
        name="torchft_b200",
        roles=[specs.Role(name=r.name, image=image, min_replicas=1, num_replicas=1, entrypoint=r.entrypoint,
                          args=r.args, env=r.env, max_retries=r.max_retries, resource=resource) for r in roles])
