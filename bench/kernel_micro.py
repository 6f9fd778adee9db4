"""Per-kernel timing + roofline fractions for the hand-written sm_90a kernels (1 GPU).

    python bench/kernel_micro.py --out kernel_micro.json
    ncu --set full --clock-control none --import-source on -k regex:adamw -c 2 -o gpurun_out/prof_adamw \
        python bench/kernel_micro.py --only adamw --iters 2

CUDA-event timing, 3+ warm-ups, a >L2 buffer is rewritten between timed iterations;
"frac" = algorithmic bytes / time / the H100 SXM data-sheet HBM3 bandwidth (3 350 GB/s).
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.ops import _native, fused  # noqa: E402
from torchft_b200 import quantization as Q  # noqa: E402


HBM_GBS = 3350.0  # H100 SXM data sheet (HBM3); a power-limited card reaches less


def timeit(fn, iters: int, flush: torch.Tensor) -> float:
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        flush.add_(1.0)  # evict L2 (buffer > 126 MB)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ms.append(s.elapsed_time(e))
    ms.sort()
    return ms[len(ms) // 2]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    K = _native.load()
    dev = torch.device("cuda")
    hbm = HBM_GBS
    flush = torch.zeros(64 << 20, dtype=torch.float32, device=dev)  # 256 MB
    T, H, F, V = 8192, 4096, 14336, 128256
    res = {}

    def want(name: str) -> bool:
        return not args.only or args.only in name or name in args.only

    def record(name, ms, nbytes):
        gbs = nbytes / ms / 1e6
        res[name] = {"ms": round(ms, 4), "algo_gb": round(nbytes / 1e9, 3), "gbs": round(gbs, 1), "frac_of_hbm_datasheet": round(gbs / hbm, 3)}
        print(name, res[name], flush=True)

    sp = lambda: _native.stream_ptr()  # noqa: E731
    if want("rmsnorm"):
        x = torch.randn(T, H, device=dev).bfloat16()
        w = torch.ones(H, device=dev).bfloat16()
        y = torch.empty_like(x)
        rstd = torch.empty(T, device=dev)
        record("rmsnorm_fwd", timeit(lambda: K.rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), T, H, 1e-5, sp()), args.iters, flush), 2 * x.numel() * 2)
        dy = torch.randn_like(x)
        dx = torch.empty_like(x)
        grid = K.rmsnorm_bwd_grid(T)
        part = torch.empty(grid, H, device=dev)
        dw = torch.empty_like(w)
        record("rmsnorm_bwd", timeit(lambda: K.rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), rstd.data_ptr(), dx.data_ptr(), part.data_ptr(), dw.data_ptr(), False, T, H, sp()), args.iters, flush), 3 * x.numel() * 2)
    if want("swiglu"):
        gu = torch.randn(T, 2 * F, device=dev).bfloat16()
        y = torch.empty(T, F, device=dev, dtype=torch.bfloat16)
        record("swiglu_fwd", timeit(lambda: K.swiglu_fwd(gu.data_ptr(), y.data_ptr(), T, F, sp()), args.iters, flush), 3 * T * F * 2)
        dy = torch.randn_like(y)
        dgu = torch.empty_like(gu)
        record("swiglu_bwd", timeit(lambda: K.swiglu_bwd(dy.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, F, sp()), args.iters, flush), 5 * T * F * 2)
    if want("rope"):
        Hq, Hkv, D = 32, 8, 128
        qkv = torch.randn(T, (Hq + 2 * Hkv) * D, device=dev).bfloat16()
        cs = fused.rope_table(T, D, 500000.0, dev)
        q = torch.empty(1, T, Hq, D, device=dev, dtype=torch.bfloat16)
        k = torch.empty(1, T, Hkv, D, device=dev, dtype=torch.bfloat16)
        # forward (dir 0, no v output): q and k rotated out of the packed rows, each element read once and written once
        strides = [*q.stride()[:3], *k.stride()[:3], 0, 0, 0]
        record("rope_qkv_fwd", timeit(lambda: K.rope_qkv(qkv.data_ptr(), qkv.shape[1], q.data_ptr(), k.data_ptr(), 0, strides, cs.data_ptr(), T, T, D, Hq, Hkv, 0, sp()), args.iters, flush), 2 * T * (Hq + Hkv) * D * 2)
    if want("xent"):
        rows = 2048
        logits = torch.randn(rows, V, device=dev).bfloat16()
        tgt = torch.randint(0, V, (rows,), device=dev)
        loss = torch.empty(rows, device=dev)
        record("xent_fwd_bwd", timeit(lambda: K.xent(logits.data_ptr(), tgt.data_ptr(), loss.data_ptr(), rows, V, V, 1.0, -100, sp()), args.iters, flush), 2 * rows * V * 2)
    if want("adamw"):
        n = 1 << 30  # 1 Gi params (8B model = 7.5x this)
        p = torch.zeros(n, device=dev, dtype=torch.bfloat16)
        g = torch.zeros(n, device=dev, dtype=torch.bfloat16)
        master = torch.zeros(n, device=dev)
        m = torch.zeros(n, device=dev)
        v = torch.zeros(n, device=dev)
        record("adamw", timeit(lambda: K.adamw(p.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), g.data_ptr(), n, 1e-3, 0.9, 0.95, 1e-8, 0.1, 0.1, 0.05, 1.0, 0, sp()), args.iters, flush), n * 28)
        for cap in (K.NUM_SMS * c for c in (1, 2, 4, 8, 16)):  # CTA-cap sweep (default = 16 CTAs/SM)
            record(f"adamw_cap{cap}", timeit(lambda: K.adamw(p.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), g.data_ptr(), n, 1e-3, 0.9, 0.95, 1e-8, 0.1, 0.1, 0.05, 1.0, 0, sp(), cap), args.iters, flush), n * 28)
        del p, g, master, m, v
    if want("q8"):
        n = 1 << 28
        x = torch.randn(n, device=dev).bfloat16()
        buf = torch.empty(Q.q8_bytes(n, 8), dtype=torch.uint8, device=dev)
        ng = K.q8_ngroups(n, 8)
        record("q8_quantize_bf16", timeit(lambda: K.q8_quantize(x.data_ptr(), 0, n, ng, 1, buf.data_ptr(), sp()), args.iters, flush), n * 3)
        out = torch.empty_like(x)
        record("q8_dequantize_bf16", timeit(lambda: K.q8_dequantize(buf.data_ptr(), ng, out.data_ptr(), n, 1, sp()), args.iters, flush), n * 3)
    if want("heal_copy"):
        from torchft_b200.checkpointing.p2p_transport import device_copy

        n = 1 << 30
        a = torch.empty(n, dtype=torch.uint8, device=dev)
        b = torch.empty(n, dtype=torch.uint8, device=dev)
        for blocks in (32, 64, K.NUM_SMS):
            record(f"heal_copy_local_b{blocks}", timeit(lambda: device_copy([(a.data_ptr(), b.data_ptr(), n)], blocks=blocks), args.iters, flush), 2 * n)
        del a, b
    if want("diloco_outer"):
        n = 1 << 29
        p = torch.randn(n, device=dev).bfloat16()
        o = torch.randn(n, device=dev).bfloat16()
        g = torch.randn(n, device=dev).bfloat16()
        mom = torch.zeros(n, device=dev)
        record("diloco_outer_bf16", timeit(lambda: K.diloco_outer(p.data_ptr(), o.data_ptr(), g.data_ptr(), mom.data_ptr(), n, 1, 0.7, 0.9, True, 0.25, 0, sp()), args.iters, flush), n * (2 * 5 + 8))
        del p, o, g, mom
    if want("zero1_update"):
        # the FT-ZeRO-1 update kernel at world 1 (= plain gated AdamW through the same code path the trainer uses)
        from datetime import timedelta

        from torchft_b200.parallel.symm_mem import SymmetricComm

        n = 1 << 28
        c = SymmetricComm.virtual_world(1, {"z1_param": n * 2}, dev, timeout=timedelta(seconds=10))[0]
        g = torch.zeros(n, device=dev, dtype=torch.bfloat16)
        master, m, v = (torch.zeros(n, device=dev) for _ in range(3))
        gate = torch.ones(2, dtype=torch.int32, device=dev)
        for cap in (K.NUM_SMS * c for c in (2, 8, 16)):
            record(f"zero1_update_w1_cap{cap}", timeit(lambda: c.zero1_update_("z1_param", 0, g.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), n, (1e-3, 0.9, 0.95, 1e-8, 0.1), gate, 1, 0, cap), args.iters, flush), n * 28)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"hbm_gbs_datasheet": hbm, "kernels": res}, f, indent=1)


if __name__ == "__main__":
    main()
