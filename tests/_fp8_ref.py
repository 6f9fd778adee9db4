"""CPU model of the row-scaled e4m3 quantisation of the fp8 block linears (csrc/kernels/fp8.cuh).

Per row: inputs below 2^-126 are flushed to a zero of their sign (the kernels build with FTZ); the dequantisation scale is
2^e with e = max(-126, ceil(log2(amax / 448))), taken from the bit pattern of amax; the stored byte is RN_e4m3(x * 2^-e),
cast by torch's CPU float8_e4m3fn (round to nearest even; NaN only above 464, which amax * 2^-e <= 448 never reaches).
A row holding an inf or a NaN gets a NaN scale and 0x7F in every byte.
"""

from __future__ import annotations

from typing import Tuple

import torch

E4M3 = torch.float8_e4m3fn
NAN_BYTE = 0x7F


def exponent(amax: torch.Tensor) -> torch.Tensor:
    """e of each finite fp32 amax: amax = 1.f * 2^E, and amax <= 448 * 2^(E-8) = 1.75 * 2^E exactly when f <= 0.75."""
    bits = amax.float().contiguous().view(torch.int32)
    E = (bits >> 23) - 127
    e = E - 8 + ((bits & 0x7FFFFF) > 0x600000).to(torch.int32)
    return e.clamp(min=-126)


def quantize_rows(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 ``[R, C]`` -> (uint8 e4m3 bytes ``[R, C]``, fp32 scale ``[R]``), on the CPU."""
    x = x.detach().cpu().float()
    x = torch.where(x.abs() < 2.0 ** -126, x * 0.0, x)  # FTZ keeps the sign: -tiny * 0 = -0
    bad = ~torch.isfinite(x).all(dim=1)
    amax = torch.where(torch.isfinite(x), x.abs(), 0.0).amax(dim=1) if x.shape[1] else torch.zeros(x.shape[0])
    e = exponent(amax)
    q = (x * torch.exp2(-e.float())[:, None]).to(E4M3).view(torch.uint8).clone()
    q[bad] = NAN_BYTE
    scale = torch.exp2(e.float())
    scale[bad] = float("nan")
    return q, scale


def quantize_cols_t(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 ``W [N, K]`` -> (bytes of W^T ``[K, N]``, fp32 scale ``[K]`` per column of W)."""
    return quantize_rows(w.detach().cpu().t().contiguous())


def dequantize(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """fp64 values of e4m3 bytes ``[R, C]`` with one scale per row."""
    return q.cpu().contiguous().view(E4M3).double() * scale.cpu().double().reshape(-1, 1)
