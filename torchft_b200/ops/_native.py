"""Loader for the sm_90a data-plane extension ``torchft_b200._K``.

The extension is built in-tree by ``torchft_b200._build`` (see
``__graft_entry__.build``). On a box with a GPU a missing extension is a hard
error -- there is deliberately no eager-PyTorch fallback for the hot ops, so a
silent slow path can never masquerade as the native one.
"""

from __future__ import annotations

import threading
from typing import Any, Optional

import torch

_lock = threading.Lock()
_K: Optional[Any] = None
_err: Optional[BaseException] = None

# kernels launched per wrapper call (for the benchmark's `gpu_launches` claim)
_LAUNCHES_PER_CALL = {
    "allreduce": 1, "allreduce_nvls": 1, "q8_allreduce": 1, "q8_quantize": 1, "q8_dequantize": 1, "q8_reduce": 1,
    "rmsnorm_fwd": 1, "rmsnorm_bwd": 2, "swiglu_fwd": 1, "swiglu_bwd": 1, "rope_qkv": 1, "xent": 1,
    "adamw": 1, "diloco_outer": 1, "heal_copy": 1,
    "q8_reduce_scatter": 1, "q8_slice_reduce": 1, "q8_gather_dequant": 1, "push_exchange": 1, "reduce_scatter": 1, "p2p": 1,
    "zero1_handshake": 1, "zero1_reduce": 1, "zero1_commit": 1, "zero1_update": 1, "z1_digest": 1, "z1_audit_compare": 1,
    "rmsnorm_fwd_fp8": 1, "fp8_rows": 1, "fp8_swiglu": 1, "fp8_cols_t": 2, "embedding_bwd": 2,
}


class _Counting:
    """Thin proxy over the extension module that counts OUR kernel launches."""

    def __init__(self, mod: Any) -> None:
        object.__setattr__(self, "_mod", mod)
        object.__setattr__(self, "launches", 0)
        object.__setattr__(self, "_cache", {})

    def __getattr__(self, name: str) -> Any:
        cache = object.__getattribute__(self, "_cache")
        if name in cache:
            return cache[name]
        attr = getattr(object.__getattribute__(self, "_mod"), name)
        n = _LAUNCHES_PER_CALL.get(name)
        if n is not None:
            inner = attr

            def counted(*a: Any, **k: Any) -> Any:
                object.__setattr__(self, "launches", object.__getattribute__(self, "launches") + n)
                return inner(*a, **k)

            attr = counted
        cache[name] = attr
        return attr


def kernel_launches() -> int:
    """Number of native kernels launched through this process so far."""
    return int(_K.launches) if _K is not None else 0

DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
OP_SUM, OP_MAX, OP_MIN = 0, 1, 2


def load() -> Any:
    """Return the ``_K`` module, building it on first use if the source tree is newer."""
    global _K, _err
    if _K is not None:
        return _K
    with _lock:
        if _K is not None:
            return _K
        try:
            from torchft_b200 import _K as mod  # type: ignore[attr-defined]
        except ImportError as first:
            try:
                from torchft_b200 import _build

                _build.build_kernels()
                from torchft_b200 import _K as mod  # type: ignore[attr-defined,no-redef]
            except Exception as e:  # pragma: no cover - build toolchain missing
                _err = e
                raise ImportError(
                    "torchft_b200._K (sm_90a kernels) is not built and could not be built: "
                    f"{first!r} / {e!r}. Run `python -m torchft_b200._build`."
                ) from e
        _K = _Counting(mod)
        return _K


def available() -> bool:
    """True when the extension imports AND a CUDA device is present."""
    if not torch.cuda.is_available():
        return False
    try:
        load()
        return True
    except ImportError:
        return False


def stream_ptr(stream: Optional[torch.cuda.Stream] = None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


def dtype_code(t: torch.Tensor) -> int:
    try:
        return DTYPE_CODE[t.dtype]
    except KeyError:
        raise TypeError(f"unsupported dtype for native kernels: {t.dtype}") from None
