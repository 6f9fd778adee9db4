"""Can the HBM-bound AdamW update hide under tensor-core GEMMs on one H100?

Times, per "layer" (4 forward-shaped bf16 GEMMs of a Llama-3-8B block at 8192 tokens,
and the AdamW update of that layer's 218 M parameters, 6.1 GB of traffic):
  serial      GEMMs then AdamW on one stream
  overlapped  AdamW on a second stream (optionally narrowed to fewer CTAs / lower priority)
Device-timed with CUDA events over LAYERS layers after warm-up.
"""

from __future__ import annotations

import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torchft_b200.ops import _native  # noqa: E402

LAYERS = 8
T, H, F, QKV = 8192, 4096, 14336, 6144
NP = H * QKV + H * H + 2 * F * H + F * H  # ~218 M


def main() -> None:
    K = _native.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    x = torch.randn(T, H, device=dev, dtype=torch.bfloat16)
    xf = torch.randn(T, F, device=dev, dtype=torch.bfloat16)
    Ws = [torch.randn(n, k, device=dev, dtype=torch.bfloat16) * 0.02 for n, k in ((QKV, H), (H, H), (2 * F, H))]
    Wd = torch.randn(H, F, device=dev, dtype=torch.bfloat16) * 0.02
    p = torch.zeros(LAYERS * NP, device=dev, dtype=torch.bfloat16)
    g = torch.randn(LAYERS * NP, device=dev, dtype=torch.bfloat16)
    master, m, v = (torch.zeros(LAYERS * NP, device=dev, dtype=torch.float32) for _ in range(3))

    def gemms() -> None:
        for W in Ws:
            x @ W.t()
        xf @ Wd.t()

    def adam(layer: int, stream: torch.cuda.Stream, blocks: int) -> None:
        o = layer * NP
        K.adamw(p.data_ptr() + 2 * o, master.data_ptr() + 4 * o, m.data_ptr() + 4 * o, v.data_ptr() + 4 * o,
                g.data_ptr() + 2 * o, NP, 1e-4, 0.9, 0.95, 1e-8, 0.1, 0.1, 0.05, 1.0, 0, stream.cuda_stream, blocks)

    main_s = torch.cuda.current_stream()

    def timed(fn) -> float:
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(3):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / 3

    res = {}

    def only_gemm() -> None:
        for _ in range(LAYERS):
            gemms()

    def only_adam(blocks: int = 0) -> None:
        for layer in range(LAYERS):
            adam(layer, main_s, blocks)

    def serial() -> None:
        for layer in range(LAYERS):
            adam(layer, main_s, 0)
            gemms()

    res["gemm_only_ms"] = timed(only_gemm)
    res["adam_only_ms"] = timed(only_adam)
    for b in (K.NUM_SMS, 2 * K.NUM_SMS, 4 * K.NUM_SMS):
        res[f"adam_only_b{b}_ms"] = timed(lambda: only_adam(b))
    res["serial_ms"] = timed(serial)

    for prio_name, prio in (("lo", 0), ("hi", -1)):
        side = torch.cuda.Stream(priority=prio)
        for blocks in (0, 4 * K.NUM_SMS, 2 * K.NUM_SMS, K.NUM_SMS, K.NUM_SMS // 2):
            def overlapped() -> None:
                # layer i's GEMMs wait only for layer i's update, later updates run underneath
                side.wait_stream(main_s)
                evs = []
                for layer in range(LAYERS):
                    adam(layer, side, blocks)
                    ev = torch.cuda.Event()
                    ev.record(side)
                    evs.append(ev)
                for layer in range(LAYERS):
                    main_s.wait_event(evs[layer])
                    gemms()
                main_s.wait_stream(side)

            res[f"overlap_{prio_name}_b{blocks}_ms"] = timed(overlapped)
    print("OVERLAP_PROBE " + json.dumps({k: round(v, 3) for k, v in res.items()}), flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/overlap_probe.json", "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
