"""The source side of a heal in its own process: builds the seeded state of ``--config``, serves it with
``P2PTransport.send_checkpoint``, prints ``{"metadata", "step"}`` (or ``{"error"}``) as one JSON line, waits for a line on
stdin, then withdraws the checkpoint and exits. It serves from a side stream, as the Manager does. ``source_state`` is
also what the receiving test rebuilds its expected bytes from.

Configurations: ``leaves`` (every dtype the receiver resolves by name, odd shapes and views, host tensors, nested
non-tensor leaves) and ``zero1_vmm`` (the FT-ZeRO-1 heal payload ``{param, t}`` with ``param`` a view of a ``cuMemCreate``
segment, as the symmetric segments are in vmm mode)."""

from __future__ import annotations

import argparse
import json
import os
import sys
from datetime import timedelta

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

STEP = 11
DTYPES = (torch.float32, torch.float64, torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2, torch.int8,
          torch.int16, torch.int32, torch.int64, torch.uint8, torch.bool, torch.complex64)
ZERO1_NUMEL = (32 << 20) + 7  # 64 MiB of bf16 weights and an odd tail: a staging copy long enough to race a fill


def _raw(g, nbytes):
    """``nbytes`` seeded random bytes: as floats they hold NaN payloads, infinities, subnormals and -0.0."""
    return torch.randint(0, 256, (nbytes,), dtype=torch.uint8, generator=g)


def _rand(g, shape, dtype):
    n = 1
    for s in shape:
        n *= s
    if dtype == torch.bool:
        return torch.randint(0, 2, tuple(shape), generator=g).bool()
    size = torch.empty(0, dtype=dtype).element_size()
    return _raw(g, n * size).view(dtype).reshape(shape)


def source_state(config, seed, device, vmm_param=None):
    """The state dict a source with ``seed`` serves (CUDA leaves on ``device``). ``zero1_vmm`` writes the weights into
    ``vmm_param`` when given one."""
    g = torch.Generator().manual_seed(seed)
    dev = torch.device(device)
    if config == "zero1_vmm":
        w = _raw(g, ZERO1_NUMEL * 2).view(torch.bfloat16)
        if vmm_param is None:
            return {"param": w.to(dev), "t": 5}
        vmm_param.copy_(w)
        return {"param": vmm_param, "t": 5}
    assert config == "leaves", config
    sd = {"dtypes": {str(d).replace("torch.", ""): _rand(g, (3, 5, 7), d).to(dev) for d in DTYPES}}
    sd["scalar"] = _rand(g, (), torch.float32).to(dev)
    sd["empty"] = _rand(g, (0, 4), torch.float16).to(dev)
    sd["odd"] = _rand(g, (1, 13, 1), torch.int16).to(dev)
    big = _rand(g, (4099,), torch.uint8).to(dev)
    sd["at_odd_offset"] = {"bytes": big[7:7 + 1001], "half": big[6:6 + 2002].view(torch.float16)}  # offsets 7 and 3
    sd["transposed"] = _rand(g, (37, 41), torch.float32).to(dev).t()
    sd["expanded"] = _rand(g, (1, 5), torch.float64).to(dev).expand(4, 5)
    shared = _rand(g, (1 << 16,), torch.float32).to(dev)
    sd["same_alloc"] = [shared[3:1003], shared[40000:40000 + 777].view(torch.int32)]
    sd["host"] = {"small": _rand(g, (4095,), torch.uint8), "page": _rand(g, (1024,), torch.float32),
                  "small_pinned": _rand(g, (4095,), torch.uint8).pin_memory(),
                  "page_pinned": _rand(g, (2048,), torch.bfloat16).pin_memory()}
    sd["meta"] = {"lr": 0.1, "names": ["a", "b"], "step": 7, "none": None, "pair": (1, 2.5, "x"), "nested": {"k": [3, {"d": 4}]}}
    return sd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="leaves")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    torch.cuda.set_device(args.device)
    from torchft_b200.checkpointing import P2PTransport
    from torchft_b200.ops import _native
    from torchft_b200.parallel.symm_mem import tensor_from_ptr

    K = _native.load()
    seg = None
    timeout = timedelta(seconds=60)
    tr = P2PTransport(timeout)
    try:
        vmm_param = None
        if args.config == "zero1_vmm":
            seg = K.vmm_alloc(ZERO1_NUMEL * 2 + 4096)
            ptr, size = seg[0], seg[1]
            vmm_param = tensor_from_ptr(ptr, size, torch.device("cuda", args.device))[4096:4096 + ZERO1_NUMEL * 2].view(torch.bfloat16)
        sd = source_state(args.config, args.seed, f"cuda:{args.device}", vmm_param)
        torch.cuda.synchronize()
        try:
            # as the Manager serves its state: on a side stream, which does not wait for the legacy default stream
            with torch.cuda.stream(torch.cuda.Stream()):
                tr.send_checkpoint([1], STEP, sd, timeout)
        except Exception as e:  # noqa: BLE001 - the receiving test reports it
            print(json.dumps({"error": f"{type(e).__name__}: {e}"}), flush=True)
            return 1
        print(json.dumps({"metadata": tr.metadata(), "step": STEP}), flush=True)
        sys.stdin.readline()
        tr.disallow_checkpoint()
        return 0
    finally:
        tr.shutdown()
        if seg is not None:
            torch.cuda.synchronize()
            os.close(seg[3])
            K.vmm_unmap(seg[0], seg[1], seg[2])


if __name__ == "__main__":
    sys.exit(main())
