"""Small device helpers (reference: torchft/utils.py:17-67). CUDA only -- this framework targets H100."""

from __future__ import annotations

from contextlib import nullcontext
from typing import Any, ContextManager, Optional

import torch


def get_stream_context(stream: Optional["torch.cuda.Stream"]) -> ContextManager[Any]:
    """``torch.cuda.stream(stream)`` when there is a device and a stream, else a no-op context."""
    if stream is not None and torch.cuda.is_available():
        return torch.cuda.stream(stream)
    return nullcontext()


def record_event() -> Optional["torch.cuda.Event"]:
    """Record (and return) an event on the current stream; ``None`` on CPU.

    The reference version returns ``None`` unconditionally (SURVEY 7.5 quirk); ours returns the event.
    """
    if torch.cuda.is_available():
        return torch.cuda.current_stream().record_event()
    return None


def synchronize() -> None:
    """Block the host until the CURRENT STREAM has drained (not the whole device)."""
    if torch.cuda.is_available():
        torch.cuda.current_stream().synchronize()


def any_nan(ts: Any) -> bool:
    """True if any tensor in a (nested) list/dict holds a NaN (test helper, reference: _test_utils.py)."""
    if isinstance(ts, torch.Tensor):
        return bool(torch.isnan(ts).any().item())
    if isinstance(ts, dict):
        return any(any_nan(v) for v in ts.values())
    if isinstance(ts, (list, tuple)):
        return any(any_nan(v) for v in ts)
    return False
