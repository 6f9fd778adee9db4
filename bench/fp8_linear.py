"""fp8 against bf16 for the block linears' forward and input-gradient GEMMs, per weight shape of Llama-3 1B and 8B.

For each weight W [N, K] at T tokens it times, with CUDA events over many launches after a warm-up:

* bf16: ``x @ W^T`` and ``dy @ W`` (cuBLAS);
* fp8:  the same two GEMMs as rowwise ``torch._scaled_mm`` INCLUDING every quantisation launch the training step makes
  for them: the activation (fp8_rows; in the model wqkv / w13 get it from the fused RMSNorm and w2 from the fused
  SwiGLU, which read more but write the same), W per row, dy per row and W^T per column (fp8_cols_t);

and each quantisation kernel alone. It prints one line per shape and a JSON summary with the card's name and power limit,
read in the same run. Effective TFLOP/s count the 2 x 2 T N K FLOPs of the two GEMMs over the measured time; a
quantisation kernel's GB/s counts the bf16 read and the e4m3 + scale write.

    python bench/fp8_linear.py [--tokens 8192] [--iters 50] [--out results.json]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchft_b200.models.llama import CONFIGS  # noqa: E402
from torchft_b200.ops import fused  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[torch.cuda.current_device()].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, iters: int, warmup: int = 5) -> float:
    """Mean seconds per call of ``fn`` over ``iters`` back-to-back launches, after ``warmup`` calls."""
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def shapes(name: str):
    c = CONFIGS[name]
    qkv = (c.n_heads + 2 * c.n_kv_heads) * c.head_dim
    return {"wqkv": (qkv, c.dim), "wo": (c.dim, c.dim), "w13": (2 * c.ffn_dim, c.dim), "w2": (c.dim, c.ffn_dim)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama3_1b,llama3_8b")
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_linear.py needs a CUDA device")
    T = args.tokens
    gen = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for model in args.models.split(","):
        for wname, (N, K) in shapes(model).items():
            x = torch.randn(T, K, device="cuda", generator=gen).bfloat16()
            W = (torch.randn(N, K, device="cuda", generator=gen) * 0.02).bfloat16()
            dy = (torch.randn(T, N, device="cuda", generator=gen) * 1e-3).bfloat16()
            it = args.iters

            def bf16():
                x @ W.t()
                dy @ W

            def fp8():
                fused._fwd_fp8(fused.fp8_rows(x), W)
                fused._dgrad_fp8(dy, W)

            qa, qw, qd, qt = fused.fp8_rows(x), fused.fp8_rows(W), fused.fp8_rows(dy), fused.fp8_cols_t(W)

            def fp8_gemms():
                fused._mm_fp8(qa, (qw[0].t(), qw[1].view(1, -1)))
                fused._mm_fp8(qd, (qt[0].t(), qt[1]))

            t_bf16, t_fp8, t_mm = timed(bf16, it), timed(fp8, it), timed(fp8_gemms, it)
            q_t = {"x": timed(lambda: fused.fp8_rows(x), it), "W": timed(lambda: fused.fp8_rows(W), it),
                   "dy": timed(lambda: fused.fp8_rows(dy), it), "W^T": timed(lambda: fused.fp8_cols_t(W), it)}
            q_bytes = {"x": 3 * T * K + 4 * T, "W": 3 * N * K + 4 * N, "dy": 3 * T * N + 4 * T,
                       "W^T": 2 * N * K + 3 * N * K + 4 * K}  # fp8_cols_t reads W twice
            flops = 4.0 * T * N * K
            r = {"model": model, "weight": wname, "T": T, "N": N, "K": K,
                 "bf16_ms": t_bf16 * 1e3, "fp8_ms": t_fp8 * 1e3, "fp8_gemm_ms": t_mm * 1e3,
                 "bf16_tflops": flops / t_bf16 / 1e12, "fp8_tflops": flops / t_fp8 / 1e12,
                 "fp8_gemm_tflops": flops / t_mm / 1e12, "speedup": t_bf16 / t_fp8,
                 "quant_us": {k: v * 1e6 for k, v in q_t.items()},
                 "quant_gbps": {k: q_bytes[k] / q_t[k] / 1e9 for k in q_t}}
            rows.append(r)
            print(f"{model:10s} {wname:5s} T={T} N={N:6d} K={K:6d}  bf16 {r['bf16_ms']:7.3f} ms {r['bf16_tflops']:6.1f} TF/s | "
                  f"fp8 {r['fp8_ms']:7.3f} ms {r['fp8_tflops']:6.1f} TF/s (GEMMs alone {r['fp8_gemm_ms']:7.3f} ms "
                  f"{r['fp8_gemm_tflops']:6.1f}) x{r['speedup']:.2f} | quant GB/s "
                  + " ".join(f"{k} {v:.0f}" for k, v in r["quant_gbps"].items()), flush=True)
            del x, W, dy, qa, qw, qd, qt
    out = {"card": card(), "torch": torch.__version__, "rows": rows}
    print(json.dumps({"card": out["card"], "torch": out["torch"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
