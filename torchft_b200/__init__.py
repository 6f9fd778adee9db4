"""torchft_b200 -- per-step fault-tolerant training, built for 8xH100 / NVLink 4 / NVSwitch.

Same capabilities and API surface as meta-pytorch/torchft (Lighthouse quorum
server, Manager, reconfigurable process groups, fault-tolerant DDP/HSDP,
LocalSGD/DiLoCo, live checkpoint recovery), with the control plane in C++ and
the data plane as hand-written sm_90a kernels over NVLink peer memory.
"""

import logging as _logging


def _ensure_native() -> None:
    """A fresh checkout has no ``torchft_b200/_C*.so`` yet and every entry point (``python -m torchft_b200._build``,
    ``__graft_entry__.build()``, plain ``import torchft_b200``) imports this package first: build the C++ control plane on
    first import (g++, ~20 s, one process at a time) instead of failing with ModuleNotFoundError. The CUDA kernels are
    built by ``_build.build_kernels`` / ``ops._native.load`` when they are first needed. ``TORCHFT_B200_NO_AUTOBUILD=1``
    disables this."""
    import importlib
    import importlib.util
    import os

    if importlib.util.find_spec("torchft_b200._C") is not None or os.environ.get("TORCHFT_B200_NO_AUTOBUILD") == "1":
        return
    from torchft_b200 import _build  # no package-level imports in there

    _build.BUILD.mkdir(parents=True, exist_ok=True)
    lock = open(_build.BUILD / ".autobuild.lock", "w")
    try:
        import fcntl

        fcntl.flock(lock, fcntl.LOCK_EX)  # torchrun starts N ranks at once: one builds, the others wait and find it done
        if importlib.util.find_spec("torchft_b200._C") is None:
            _logging.getLogger(__name__).warning("torchft_b200: building the C++ control plane (first import of a fresh checkout)")
            _build.build_control()
            importlib.invalidate_caches()
    finally:
        lock.close()


_ensure_native()

from torchft_b200.data import DistributedSampler  # noqa: E402
from torchft_b200.ddp import DistributedDataParallel, FlatDistributedDataParallel, PureDistributedDataParallel
from torchft_b200.manager import Manager, WorldSizeMode
from torchft_b200.optim import OptimizerWrapper as Optimizer
from torchft_b200.otel import setup_logger as _setup_logger
from torchft_b200.process_group import (
    ManagedProcessGroup,
    ProcessGroupDummy,
    ProcessGroupGloo,
    ProcessGroupNCCL,
    ProcessGroupXCCL,
)
from torchft_b200.baby import ProcessGroupBabyGloo, ProcessGroupBabyNCCL, ProcessGroupBabyXCCL

for _name in ("torchft_quorums", "torchft_commits", "torchft_errors"):
    _setup_logger(_name)


def __getattr__(name: str):  # lazy: needs CUDA at construction time only
    if name == "ProcessGroupB200":
        from torchft_b200.parallel.process_group_b200 import ProcessGroupB200

        return ProcessGroupB200
    raise AttributeError(name)


__all__ = [
    "DistributedDataParallel",
    "FlatDistributedDataParallel",
    "PureDistributedDataParallel",
    "DistributedSampler",
    "Manager",
    "WorldSizeMode",
    "Optimizer",
    "ManagedProcessGroup",
    "ProcessGroupB200",
    "ProcessGroupNCCL",
    "ProcessGroupXCCL",
    "ProcessGroupBabyNCCL",
    "ProcessGroupBabyXCCL",
    "ProcessGroupBabyGloo",
    "ProcessGroupGloo",
    "ProcessGroupDummy",
]
