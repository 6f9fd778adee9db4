"""Where does a Llama-3 training step go? torch.profiler kernel table for ONE step (1 GPU),
plus an SDPA backend shoot-out at the model's attention shape.

    python bench/step_profile.py --out gpurun_out/step_profile.txt
"""

from __future__ import annotations

import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def attn_shootout(S=8192, Hq=32, Hkv=8, D=128, out=None):
    from torch.nn.attention import SDPBackend, sdpa_kernel

    q = torch.randn(1, Hq, S, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(1, Hkv, S, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(1, Hkv, S, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    flops_fwd = 4 * S * S * Hq * D / 2
    lines = []
    for name, be in (("flash", SDPBackend.FLASH_ATTENTION), ("cudnn", SDPBackend.CUDNN_ATTENTION),
                     ("efficient", SDPBackend.EFFICIENT_ATTENTION), ("default", None)):
        try:
            def run():
                if be is None:
                    o = F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)
                else:
                    with sdpa_kernel(be):
                        o = F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)
                return o
            for _ in range(3):
                o = run()
                o.sum().backward()
            torch.cuda.synchronize()
            s, m, e = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            s.record()
            for _ in range(5):
                o = run()
            m.record()
            g = torch.randn_like(o)
            for _ in range(5):
                o = run()
                o.backward(g)
            e.record()
            torch.cuda.synchronize()
            fwd = s.elapsed_time(m) / 5
            fb = m.elapsed_time(e) / 5
            lines.append(f"sdpa[{name}] fwd {fwd:.3f} ms ({flops_fwd / fwd / 1e9:.0f} TFLOP/s)  fwd+bwd {fb:.3f} ms "
                         f"({3.5 * flops_fwd / fb / 1e9:.0f} TFLOP/s eff)")
        except Exception as ex:  # noqa: BLE001
            lines.append(f"sdpa[{name}] unavailable: {str(ex)[:120]}")
    for l in lines:
        print(l, flush=True)
    if out:
        out.write("\n".join(lines) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama3_1b")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--out", default="gpurun_out/step_profile.txt")
    args = ap.parse_args()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    out = open(args.out, "w")
    attn_shootout(S=args.seq, out=out)

    from torchft_b200.models.llama import CONFIGS, FlatParams, Llama
    from torchft_b200.ops.fused import FlatAdamW

    cfg = CONFIGS[args.model]
    m = Llama(cfg, device="meta")
    flat = FlatParams(m, device=torch.device("cuda"))
    m.init_weights(0)
    opt = FlatAdamW(flat.param, flat.grad)
    opt.direct_grads = True
    tok = torch.randint(0, cfg.vocab_size, (1, args.seq), device="cuda")
    tgt = torch.randint(0, cfg.vocab_size, (1, args.seq), device="cuda")

    def step():
        flat.reset_grads()
        loss = m(tok, tgt)
        loss.backward()
        for p in flat.params:
            flat.adopt_grad(p)
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(3):
        step()
    e.record()
    torch.cuda.synchronize()
    msg = f"plain step (no FT): {s.elapsed_time(e) / 3:.1f} ms"
    print(msg)
    out.write(msg + "\n")
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step()
        torch.cuda.synchronize()
    table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=90)
    out.write(table + "\n")
    print(table[:6000])
    out.close()


if __name__ == "__main__":
    main()
