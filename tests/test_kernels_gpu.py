"""Numerics of the hand-written sm_90a kernels vs plain PyTorch fp32 references."""


import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from torchft_b200.ops import _native

    return _native.load()


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize("rows,H", [(7, 256), (33, 4096), (5, 8192), (3, 16384)])
def test_rmsnorm_fwd_bwd(rows, H):
    from torchft_b200.ops import fused

    torch.manual_seed(0)
    x = torch.randn(rows, H, device="cuda").bfloat16().requires_grad_()
    w = (1 + 0.1 * torch.randn(H, device="cuda")).bfloat16().requires_grad_()
    y = fused.rmsnorm(x, w, 1e-5)
    dy = torch.randn_like(y)
    y.backward(dy)
    xf, wf = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    yf = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    yf.backward(dy.float())
    assert _rel(y, yf) < 1e-2
    assert _rel(x.grad, xf.grad) < 1e-2
    assert _rel(w.grad, wf.grad) < 2e-2


def test_swiglu_fwd_bwd():
    from torchft_b200.ops import fused

    torch.manual_seed(1)
    gu = torch.randn(37, 2 * 192, device="cuda").bfloat16().requires_grad_()
    y = fused.swiglu(gu)
    dy = torch.randn_like(y)
    y.backward(dy)
    g = gu.detach().float().requires_grad_()
    yf = torch.nn.functional.silu(g[:, :192]) * g[:, 192:]
    yf.backward(dy.float())
    assert _rel(y, yf) < 1e-2
    assert _rel(gu.grad, g.grad) < 1e-2


def test_rope_qkv_matches_complex_rotation():
    from torchft_b200.ops import fused

    torch.manual_seed(2)
    B, S, Hq, Hkv, D = 2, 16, 4, 2, 32
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * D, device="cuda").bfloat16().requires_grad_()
    cs = fused.rope_table(S, D, 10000.0, qkv.device)
    q, k, v = fused.rope_qkv(qkv, cs, B, S, Hq, Hkv, D)

    def ref_rot(x):  # x [B,S,H,D] fp32
        xc = torch.view_as_complex(x.reshape(*x.shape[:-1], D // 2, 2))
        f = torch.polar(torch.ones(S, D // 2, device=x.device), torch.outer(
            torch.arange(S, device=x.device).float(),
            1.0 / (10000.0 ** (torch.arange(0, D, 2, device=x.device).float() / D))))
        return torch.view_as_real(xc * f[None, :, None, :]).reshape(x.shape)

    ref = qkv.detach().float().requires_grad_()
    r3 = ref.view(B, S, Hq + 2 * Hkv, D)
    qf, kf, vf = ref_rot(r3[:, :, :Hq]), ref_rot(r3[:, :, Hq:Hq + Hkv]), r3[:, :, Hq + Hkv:]
    assert _rel(q, qf) < 1e-2 and _rel(k, kf) < 1e-2 and _rel(v, vf) < 1e-6
    dq, dk, dv = torch.randn_like(q), torch.randn_like(k), torch.randn_like(v)
    torch.autograd.backward([q, k, v], [dq, dk, dv])
    torch.autograd.backward([qf, kf, vf], [dq.float(), dk.float(), dv.float()])
    assert _rel(qkv.grad, ref.grad) < 1e-2


@pytest.mark.parametrize("D,Hq,Hkv", [(128, 8, 2), (96, 3, 3), (64, 4, 1)])
def test_rope_qkv_backward_takes_sdpa_ordered_gradients(D, Hq, Hkv):
    """dq/dk/dv arrive as [B,H,S,D]-contiguous tensors seen through transpose(1,2) (what SDPA's backward hands over):
    the one-launch backward must read them in place and match the contiguous path bit for bit."""
    from torchft_b200.ops import fused

    torch.manual_seed(12)
    B, S = 2, 24
    cs = fused.rope_table(S, D, 500000.0, torch.device("cuda"))
    base = torch.randn(B * S, (Hq + 2 * Hkv) * D, device="cuda").bfloat16()
    grads = []
    for transposed in (False, True):
        qkv = base.clone().requires_grad_()
        q, k, v = fused.rope_qkv(qkv, cs, B, S, Hq, Hkv, D)
        torch.manual_seed(13)
        gs = []
        for t in (q, k, v):
            g = torch.randn(t.shape, device="cuda").bfloat16()
            gs.append(g.transpose(1, 2).contiguous().transpose(1, 2) if transposed else g)
        assert gs[0].is_contiguous() != transposed
        torch.autograd.backward([q, k, v], gs)
        grads.append(qkv.grad)
    assert torch.equal(grads[0], grads[1])
    # and the raw single-tensor kernel (generic API) agrees with the fused split on q
    K = fused._native.load()
    q2 = torch.empty(B * S, Hq * D, device="cuda", dtype=torch.bfloat16)
    K.rope(base.data_ptr(), q2.data_ptr(), cs.data_ptr(), B * S, S, Hq, D, base.shape[1], Hq * D, 1.0, fused._native.stream_ptr())
    q, _, _ = fused.rope_qkv(base, cs, B, S, Hq, Hkv, D)
    assert torch.equal(q.reshape(B * S, Hq * D), q2)


@pytest.mark.parametrize("tpb,pf,cps", [(128, 0, 4), (128, 1, 2), (256, 1, 3), (512, 0, 8), (512, 1, 1)])
@pytest.mark.parametrize("H", [256, 4096, 5120])
def test_rmsnorm_every_cta_shape_matches_reference(tpb, pf, cps, H):
    from torchft_b200.ops import fused

    K = fused._native.load()
    try:
        K.rmsnorm_tune(0, tpb, pf, cps)
        K.rmsnorm_tune(1, tpb, pf, cps)
        torch.manual_seed(5)
        rows = 777
        x = torch.randn(rows, H, device="cuda").bfloat16().requires_grad_()
        w = (1 + 0.1 * torch.randn(H, device="cuda")).bfloat16().requires_grad_()
        y = fused.rmsnorm(x, w, 1e-5)
        dy = torch.randn_like(y)
        y.backward(dy)
        xf, wf = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
        yf = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
        yf.backward(dy.float())
        assert _rel(y, yf) < 1e-2 and _rel(x.grad, xf.grad) < 1e-2 and _rel(w.grad, wf.grad) < 2e-2
    finally:
        K.rmsnorm_tune(0, 128, 1, 6)
        K.rmsnorm_tune(1, 256, 1, 4)


@pytest.mark.parametrize("T,V", [(64, 1000), (33, 4104), (16, 128256)])
def test_linear_cross_entropy(T, V):
    from torchft_b200.ops import fused

    torch.manual_seed(3)
    H = 128
    h = (torch.randn(T, H, device="cuda") * 0.5).bfloat16().requires_grad_()
    W = (torch.randn(V, H, device="cuda") * 0.05).bfloat16().requires_grad_()
    tgt = torch.randint(0, V, (T,), device="cuda")
    loss = fused.linear_cross_entropy(h, W, tgt, chunk=24, count_valid=False)
    loss.backward()
    hf, Wf = h.detach().float().requires_grad_(), W.detach().float().requires_grad_()
    lf = torch.nn.functional.cross_entropy(hf @ Wf.t(), tgt)
    lf.backward()
    assert abs(loss.item() - lf.item()) < 2e-2 * max(1.0, abs(lf.item()))
    assert _rel(h.grad, hf.grad) < 3e-2
    assert _rel(W.grad, Wf.grad) < 3e-2


def test_cross_entropy_inplace_ignore_index():
    from torchft_b200.ops import fused

    torch.manual_seed(4)
    logits = torch.randn(8, 512, device="cuda").bfloat16()
    tgt = torch.randint(0, 512, (8,), device="cuda")
    tgt[3] = -100
    ref = torch.nn.functional.cross_entropy(logits.float(), tgt, reduction="none", ignore_index=-100)
    losses = fused.cross_entropy_inplace(logits, tgt, 1.0)
    assert torch.allclose(losses, ref, atol=2e-2, rtol=2e-2)
    assert logits[3].abs().max().item() == 0.0


def test_flat_adamw_matches_torch():
    from torchft_b200.ops import fused

    torch.manual_seed(5)
    n = 10007
    p = torch.randn(n, device="cuda").bfloat16()
    g = torch.zeros_like(p)
    opt = fused.FlatAdamW(p, g, lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    ref_p = p.float().clone().requires_grad_()
    ref = torch.optim.AdamW([ref_p], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    gate = torch.ones(1, dtype=torch.int32, device="cuda")
    for step in range(5):
        gr = torch.randn(n, device="cuda").bfloat16()
        g.copy_(gr)
        ref_p.grad = gr.float()
        opt.step(gate=gate)
        ref.step()
    assert _rel(opt.master, ref_p.detach()) < 1e-5
    assert _rel(p, ref_p.detach()) < 5e-3
    before = opt.master.clone()
    gate.zero_()
    opt.step(gate=gate)  # gated off: must be a no-op
    assert torch.equal(before, opt.master)
    ss = opt.grad_sumsq()
    assert abs(ss.item() - g.float().pow(2).sum().item()) < 1e-2 * ss.item()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n", [5, 512, 100003])
def test_q8_roundtrip(K, dtype, n):
    from torchft_b200 import quantization as Q

    torch.manual_seed(6)
    x = (torch.randn(n, device="cuda") * 10).to(dtype)
    buf = Q.quantize_q8(x, world_size=2)
    y = Q.dequantize_q8(buf, n, dtype, world_size=2)
    rel = ((y.float() - x.float()).abs().mean() / x.float().abs().mean()).item()
    assert rel < 0.04


def test_heal_copy(K):
    from torchft_b200.checkpointing.p2p_transport import device_copy

    torch.manual_seed(7)
    srcs = [torch.randn(n, device="cuda") for n in (1, 1000, 1 << 20, 12345)]
    srcs.append(torch.randint(0, 255, (777,), device="cuda", dtype=torch.uint8)[1:])  # unaligned
    dsts = [torch.empty_like(s) for s in srcs]
    device_copy([(s.data_ptr(), d.data_ptr(), s.numel() * s.element_size()) for s, d in zip(srcs, dsts)])
    torch.cuda.synchronize()
    for s, d in zip(srcs, dsts):
        assert torch.equal(s, d)


def test_heal_copy_bulk_tma_variant(K):
    """cp.async.bulk ring (global -> shared -> global, mbarrier-tracked): same bytes as the LSU kernel, incl. odd tails."""
    from torchft_b200.checkpointing.p2p_transport import device_copy

    torch.manual_seed(8)
    sizes = (16, 1000 * 4, (1 << 22) + 16, 12345 * 4, 48 * 1024, 7 << 20)
    srcs = [torch.randint(0, 255, (n,), device="cuda", dtype=torch.uint8) for n in sizes]
    srcs.append(torch.randint(0, 255, (100_003,), device="cuda", dtype=torch.uint8))  # 3-byte tail after the 16 B body
    dsts = [torch.zeros_like(s) for s in srcs]
    for chunk in (1 << 20, 4 << 20):
        for d in dsts:
            d.zero_()
        device_copy([(s.data_ptr(), d.data_ptr(), s.numel()) for s, d in zip(srcs, dsts)], bulk=True, chunk_bytes=chunk)
        torch.cuda.synchronize()
        for s, d in zip(srcs, dsts):
            assert torch.equal(s, d), (s.numel(), chunk)
    # unaligned ranges silently use the LSU kernel
    u = torch.randint(0, 255, (5000,), device="cuda", dtype=torch.uint8)[1:]
    v = torch.zeros(4999, device="cuda", dtype=torch.uint8)
    device_copy([(u.data_ptr(), v.data_ptr(), 4999)], bulk=True)
    torch.cuda.synchronize()
    assert torch.equal(u, v)


def test_llama_tiny_fwd_bwd_matches_reference():
    from torchft_b200.models.llama import CONFIGS, Llama
    from torchft_b200.models.reference import reference_loss

    torch.manual_seed(8)
    cfg = CONFIGS["llama3_tiny"]
    m = Llama(cfg, device="cuda")
    m.init_weights(0)
    tok = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda")
    tgt = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda")
    loss = m(tok, tgt)
    loss.backward()
    ref_loss, ref_grads = reference_loss(m, tok, tgt)
    assert abs(loss.item() - ref_loss) < 3e-2 * max(1.0, abs(ref_loss))
    for name, p in m.named_parameters():
        assert p.grad is not None, name
        r = _rel(p.grad, ref_grads[name])
        assert r < 0.1, (name, r)


def test_direct_wgrad_into_flat_buffer_matches_accumulate_path():
    """reset_grads(): wgrad GEMMs write the flat gradient buffer directly; result == zero+accumulate path."""
    from torchft_b200.models.llama import CONFIGS, FlatParams, Llama

    cfg = CONFIGS["llama3_tiny"]
    tok = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda")
    tgt = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda")
    grads = []
    for direct in (False, True):
        m = Llama(cfg, device="meta")
        flat = FlatParams(m, device=torch.device("cuda"))
        m.init_weights(0)
        flat.grad.fill_(float("nan")) if direct else None  # stale garbage must be fully overwritten
        flat.grad.view(torch.int16).zero_() if not direct else None
        if direct:
            # padding between parameters is never written by producers: it must start (and stay) zero
            flat.grad.zero_()
            for p in flat.params:
                p._flat_grad.fill_(float("nan"))
        flat.reset_grads(zero=not direct)
        m(tok, tgt).backward()
        for p in flat.params:
            flat.adopt_grad(p)
        torch.cuda.synchronize()
        assert not torch.isnan(flat.grad.float()).any()
        grads.append(flat.grad.float().clone())
    rel = (grads[0] - grads[1]).norm() / grads[0].norm()
    assert rel < 1e-2, rel


@pytest.mark.parametrize("world_size", [2, 3, 8])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 0.05), (torch.bfloat16, 0.06), (torch.float16, 0.05)])
@pytest.mark.parametrize("op", ["sum", "avg"])
def test_q8_quantize_reduce_dequantize_all_views(K, world_size, dtype, tol, op):
    """Single-device simulation of the quantised all-reduce over every 2-D view of the inputs
    (strategy of the reference's quantization_test.py:38-106): every "rank" holds the same data,
    so SUM must return world_size * x and AVG x."""
    from torch.distributed import ReduceOp

    from torchft_b200 import _test_utils
    from torchft_b200 import quantization as Q

    torch.manual_seed(11)
    tensors_num, tensor_size = 3, 24
    inp = (torch.rand(tensors_num * tensor_size, device="cuda") * 7.0 + 0.5).to(dtype)
    rop = ReduceOp.SUM if op == "sum" else ReduceOp.AVG
    splits = _test_utils.gen_splits(inp, tensor_size)
    assert len(splits) == 7 ** 3
    for split in splits[:: max(1, len(splits) // 24)]:
        inputs, outputs = inp.clone(), torch.empty_like(inp)
        ins = [c.view(*s) for s, c in zip(split, torch.split(inputs, tensor_size))]
        outs = [c.view(*s) for s, c in zip(split, torch.split(outputs, tensor_size))]
        quant = Q.fused_quantize_into_fp8(ins, world_size)
        final = torch.empty_like(quant)
        for rank in range(world_size):
            copies = [quant.clone() for _ in range(world_size)]  # what rank would have received from every peer
            Q.fused_reduce_fp8(ins, copies, world_size, rank, rop)
            Q.copy_rank_slice(ins, final, copies[rank], world_size, rank)
        Q.fused_dequantize_from_fp8(outs, final, world_size)
        assert not _test_utils.any_nan(outs)
        expect = inputs.float() * (world_size if op == "sum" else 1)
        # reference tolerance: MEAN relative error (e4m3 keeps 3 mantissa bits, so a single element can
        # be off by 2^-4 per quantisation and the pipeline quantises twice)
        err = (outputs.float() - expect).abs() / (expect.abs() + 1e-7)
        assert err.mean().item() < tol and err.max().item() < 0.14, (split, err.mean().item(), err.max().item())


def test_p2p_transport_inplace_targets_matched_by_key_path(K):
    """Heal into a replica whose state_dict is structurally smaller than the sender's (fresh torch optimizer:
    no per-parameter state yet): matching leaves are filled IN PLACE, the rest is allocated."""
    from datetime import timedelta

    from torchft_b200.checkpointing import P2PTransport

    torch.manual_seed(9)
    w_src, m_src = torch.randn(1000, device="cuda"), torch.randn(1000, device="cuda")
    sender_sd = {"model": {"w": w_src}, "optim": {"state": {0: {"exp_avg": m_src, "step": torch.tensor(7.0)}}, "param_groups": [{"lr": 0.1}]}}
    w_dst = torch.zeros(1000, device="cuda")
    fresh_sd = {"model": {"w": w_dst}, "optim": {"state": {}, "param_groups": [{"lr": 0.5}]}}
    t = timedelta(seconds=10)
    src, dst = P2PTransport(t), P2PTransport(t, state_dict=lambda: fresh_sd)
    try:
        src.send_checkpoint([1], 3, sender_sd, t)
        got = dst.recv_checkpoint(0, src.metadata(), 3, t)
        torch.cuda.synchronize()
        assert got["model"]["w"].data_ptr() == w_dst.data_ptr() and torch.equal(w_dst, w_src)
        assert torch.equal(got["optim"]["state"][0]["exp_avg"], m_src)
        assert got["optim"]["state"][0]["exp_avg"].data_ptr() != m_src.data_ptr()
        assert float(got["optim"]["state"][0]["step"]) == 7.0 and got["optim"]["param_groups"][0]["lr"] == 0.1
        src.disallow_checkpoint()
    finally:
        src.shutdown()
        dst.shutdown()


def test_p2p_transport_moves_host_tensors_through_the_gpu_not_through_the_manifest(K):
    """CPU leaves of the source's state (DiLoCo's backup weights with ``backup_device=None``) are staged on the GPU and
    pulled by the same copy kernel; the manifest stays small, and they come back as CPU tensors -- in place when the
    receiver offers a matching CPU target. Round-1 advisor finding: they used to be hex-pickled into the manifest."""
    from datetime import timedelta

    from torchft_b200.checkpointing import P2PTransport

    torch.manual_seed(10)
    backup_src, other_src = torch.randn(300_000), torch.randn(5_000, dtype=torch.float64)  # 1.2 MB and 40 KB on the host
    w_src = torch.randn(1000, device="cuda")
    sender_sd = {"w": w_src, "backup": backup_src, "other": other_src, "tiny": torch.tensor([1.0, 2.0]), "n": 3}
    backup_dst = torch.zeros(300_000)
    fresh_sd = {"w": torch.zeros(1000, device="cuda"), "backup": backup_dst}
    t = timedelta(seconds=10)
    src, dst = P2PTransport(t), P2PTransport(t, state_dict=lambda: fresh_sd)
    try:
        src.send_checkpoint([1], 5, sender_sd, t)
        assert len(src._manifest) < 64 << 10, "host tensors must not be embedded in the manifest"
        got = dst.recv_checkpoint(0, src.metadata(), 5, t)
        torch.cuda.synchronize()
        assert got["backup"] is backup_dst and torch.equal(backup_dst, backup_src)          # in place, on the host
        assert not got["other"].is_cuda and got["other"].dtype == torch.float64 and torch.equal(got["other"], other_src)
        assert torch.equal(got["tiny"], torch.tensor([1.0, 2.0])) and got["n"] == 3 and torch.equal(got["w"], w_src)
        src.disallow_checkpoint()
    finally:
        src.shutdown()
        dst.shutdown()


def _rms(x, g, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * g


@pytest.mark.parametrize("with_res", [False, True])
def test_fused_block_ops_match_fp32_reference(with_res):
    """norm_linear(_res) / linear(res=) / swiglu_linear(res=): forward and every gradient (input, residual stream,
    norm weight, projection weights) against a plain fp32 PyTorch graph of the same sub-block."""
    from torchft_b200.ops import fused

    torch.manual_seed(21)
    T, H, F, eps = 48, 256, 384, 1e-5
    mk = lambda *s, sc=1.0: (torch.randn(*s, device="cuda") * sc).bfloat16().requires_grad_()  # noqa: E731
    x, g = mk(T, H), mk(H, sc=0.2)
    with torch.no_grad():
        g.add_(1.0)
    W13, W2, Wo = mk(2 * F, H, sc=0.05), mk(H, F, sc=0.05), mk(H, H, sc=0.05)
    if with_res:
        xs, gu = fused.norm_linear_res(x, g, W13, eps)
        h = fused.swiglu_linear(gu, W2, res=xs)
        out = fused.linear(h, Wo, res=h)
    else:
        gu = fused.norm_linear(x, g, W13, eps)
        h = x + fused.swiglu_linear(gu, W2)
        out = h + fused.linear(h, Wo)
    dout = torch.randn_like(out)
    out.backward(dout)

    xf, gf, W13f, W2f, Wof = (t.detach().float().requires_grad_() for t in (x, g, W13, W2, Wo))
    guf = _rms(xf, gf, eps) @ W13f.t()
    hf = xf + (torch.nn.functional.silu(guf[:, :F]) * guf[:, F:]) @ W2f.t()
    outf = hf + hf @ Wof.t()
    outf.backward(dout.float())
    assert _rel(out, outf) < 2e-2
    for name, a, b in (("dx", x.grad, xf.grad), ("dg", g.grad, gf.grad), ("dW13", W13.grad, W13f.grad),
                       ("dW2", W2.grad, W2f.grad), ("dWo", Wo.grad, Wof.grad)):
        assert a is not None and _rel(a, b) < 3e-2, (name, _rel(a, b))
