"""Live checkpoint transports used to heal recovering replicas.

* :class:`P2PTransport` -- native default on a single NVSwitch domain:
  the healer pulls tensors GPU->GPU over NVLink from inside a copy kernel.
* :class:`HTTPTransport` -- TCP fallback / CPU path (reference default).
* :class:`PGTransport` -- over the fault-tolerant process group's send/recv.
* :class:`DurableCheckpointer` -- on-disk checkpoints for whole-job restarts (not part of the reference).
"""

from torchft_b200.checkpointing.transport import CheckpointTransport
from torchft_b200.checkpointing.http_transport import HTTPTransport
from torchft_b200.checkpointing.pg_transport import PGTransport
from torchft_b200.checkpointing.p2p_transport import P2PTransport
from torchft_b200.checkpointing.durable import DurableCheckpointer

__all__ = ["CheckpointTransport", "HTTPTransport", "PGTransport", "P2PTransport", "DurableCheckpointer"]
