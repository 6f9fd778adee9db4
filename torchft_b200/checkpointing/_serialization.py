"""Stream (de)serialisation of arbitrary state_dict pytrees.

Uses ``torch.distributed._serialization``'s zero-copy streaming format when the
installed torch has it and plain ``torch.save``/``torch.load`` otherwise
(reference: upstream torchft/checkpointing/_serialization.py:8-39).
Checkpoints come from a trusted peer of the same job, hence ``weights_only=False``.
"""

from __future__ import annotations

from typing import IO, Any

import torch

try:  # pragma: no cover - depends on torch build
    from torch.distributed._serialization import _streaming_load, _streaming_save

    _HAS_STREAMING = True
except Exception:  # pragma: no cover
    _HAS_STREAMING = False


def streaming_save(obj: Any, f: IO[bytes]) -> None:
    if _HAS_STREAMING:
        _streaming_save(obj, f)
    else:
        torch.save(obj, f)


def streaming_load(f: IO[bytes]) -> Any:
    if _HAS_STREAMING:
        return _streaming_load(f, weights_only=False)
    if not (hasattr(f, "seekable") and f.seekable()):  # torch.load needs a seekable file
        import io

        f = io.BytesIO(f.read())
    return torch.load(f, weights_only=False)
