"""Abstract live-checkpoint transport used to heal a recovering replica.

Same contract as the reference's ``CheckpointTransport``
(upstream torchft/checkpointing/transport.py:14-68): the up-to-date
replica calls :meth:`send_checkpoint` for the ranks assigned to it by the
quorum, the healing replica calls :meth:`recv_checkpoint` with the source's
:meth:`metadata` string, and the source stops serving in
:meth:`disallow_checkpoint` (called from ``Manager.should_commit``) before its
optimizer mutates the state.
"""

from __future__ import annotations

from abc import ABC, abstractmethod
from datetime import timedelta
from typing import Generic, List, TypeVar

T = TypeVar("T")


class CheckpointTransport(Generic[T], ABC):
    """Interface of a live-heal transport (reference: checkpointing/transport.py:14-68): the source calls
    ``send_checkpoint`` / ``disallow_checkpoint``, the healing replica ``recv_checkpoint`` with the source's ``metadata()``."""

    @abstractmethod
    def metadata(self) -> str:
        """Opaque string a remote transport needs to fetch from this one (e.g. a URL)."""

    @abstractmethod
    def send_checkpoint(self, dst_ranks: List[int], step: int, state_dict: T, timeout: timedelta) -> None:
        """Make ``state_dict`` for ``step`` available to ``dst_ranks`` (may be asynchronous)."""

    def disallow_checkpoint(self) -> None:
        """Block until in-flight transfers finish; afterwards the state may be mutated."""

    @abstractmethod
    def recv_checkpoint(self, src_rank: int, metadata: str, step: int, timeout: timedelta) -> T:
        """Fetch the checkpoint for ``step`` from ``src_rank``."""

    def shutdown(self, wait: bool = True) -> None:
        """Release sockets/threads."""


def advertise_host() -> str:
    """Address peers should dial to reach a server of this process.

    ``TORCHFT_ADVERTISE_HOST`` wins; else the hostname when it resolves (the reference uses ``socket.gethostname()``,
    http_transport.py); else the address of the interface that routes off-host, so cross-node peers still get
    something dialable; loopback only as a logged last resort (single-box containers whose hostname does not resolve).
    """
    import logging
    import os
    import socket

    env = os.environ.get("TORCHFT_ADVERTISE_HOST")
    if env:
        return env
    h = socket.gethostname()
    try:
        socket.getaddrinfo(h, None)
        return h
    except OSError:
        pass
    try:
        with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s:
            s.connect(("10.255.255.255", 1))  # no packet is sent; the kernel just picks the outbound interface
            ip = s.getsockname()[0]
        if not ip.startswith("127."):
            return ip
    except OSError:
        pass
    logging.getLogger(__name__).warning("hostname %r does not resolve and no routable interface was found: advertising "
                                        "127.0.0.1 (peers on other hosts cannot reach this transport)", h)
    return "127.0.0.1"
