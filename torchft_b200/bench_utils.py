"""Small helpers shared by ``bench.py``, ``__graft_entry__.smoke`` and the GPU tests."""

from __future__ import annotations

from datetime import timedelta
from typing import Any, Dict, Optional

import torch


def local_lighthouse(min_replicas: int = 1, join_timeout_ms: int = 100) -> Any:
    from torchft_b200.coordination import LighthouseServer

    return LighthouseServer(bind="[::]:0", min_replicas=min_replicas, join_timeout_ms=join_timeout_ms)


def loopback(addr: str) -> str:
    """``http://<hostname>:port`` -> ``http://127.0.0.1:port`` (container hostnames may not resolve)."""

    host = addr.split("//")[1].rsplit(":", 1)[0]
    return addr.replace(host, "127.0.0.1")


def ft_smoke_step(model: Optional[Any] = None, cfg: Optional[Any] = None, steps: int = 2, **trainer_kw: Any) -> float:
    """A tiny but COMPLETE fault-tolerant training step on cuda:0: Lighthouse + Manager (C++ control
    plane) + ProcessGroupB200 + fused-kernel Llama forward/backward + device-side commit + gated
    FT-ZeRO-1 AdamW, through the public trainer API including the pinned H2D input copy and the D2H loss read."""
    from torchft_b200.parallel.trainer import FaultTolerantTrainer

    lh = local_lighthouse()
    trainer = None
    try:
        trainer = FaultTolerantTrainer("llama3_debug", loopback(lh.address()), replica_id="smoke_0",
                                       timeout=timedelta(seconds=30), bucket_mb=1.0, **trainer_kw)
        c = trainer.cfg
        tok = torch.randint(0, c.vocab_size, (2, 128)).pin_memory()
        tgt = torch.randint(0, c.vocab_size, (2, 128)).pin_memory()
        loss = 0.0
        for _ in range(steps):
            loss = trainer.step(tok, tgt)
        assert trainer.manager.current_step() == steps, "steps did not commit"
        return loss
    finally:
        if trainer is not None:
            trainer.shutdown()
        lh.shutdown()


def collectives_selfcheck(world: int = 4, nelem: int = 1 << 18, device: Optional[torch.device] = None) -> Dict[str, float]:
    """Run EVERY peer-memory collective kernel once for a ``world``-rank quorum emulated inside this process
    (``SymmetricComm.virtual_world``: one kernel at a time, flags pre-signalled, exact W-rank results) and check
    the numerics against PyTorch. This is what puts the multi-rank kernels in front of single-GPU tooling
    (ncu serialises launches, so really concurrent ranks would dead-wait under it). Returns max abs errors."""
    from torchft_b200.ops import _native
    from torchft_b200.parallel.symm_mem import SymmetricComm
    from torchft_b200.parallel.zero1 import ShardLayout

    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    nb = nelem * 2
    comms = SymmetricComm.virtual_world(world, {"buf": nb, "z1_grad": nb, "z1_param": nb}, dev)
    g = torch.Generator(device=dev).manual_seed(1)
    errs: Dict[str, float] = {}
    raw = [torch.randn(nelem, device=dev, generator=g).bfloat16() for _ in range(world)]
    want = sum(x.float() for x in raw) / world

    def bufs(name: str) -> list:
        return [c.segment(name)[:nb].view(torch.bfloat16) for c in comms]

    # two-shot and one-shot all-reduce (zero-copy symmetric path), and the staged path through the core segment
    for label, plan, n in (("allreduce_twoshot", (1, 8), nelem), ("allreduce_oneshot", (0, 8), 8192)):
        b = bufs("buf")
        for r in range(world):
            b[r].copy_(raw[r])
        # one-shot reduces the whole message in place on every rank, so only the FIRST emulated rank sees pristine
        # inputs; two-shot only ever rewrites slice r and is exact for all ranks
        ranks = range(world) if plan[0] == 1 else range(1)
        for r in ranks:
            c = comms[r]
            c._force_plan = plan
            c.allreduce_(c.segment("buf")[: n * 2].view(torch.bfloat16), scale=1.0 / world)
            c._force_plan = None
        torch.cuda.synchronize()
        errs[label] = max(float((b[r][:n].float() - want[:n]).abs().max()) for r in ranks)
    # fused fp8 delta all-reduce
    a = [torch.randn(nelem, device=dev, generator=g) for _ in range(world)]
    bb = [torch.randn(nelem, device=dev, generator=g) for _ in range(world)]
    outs = [torch.empty(nelem, device=dev) for _ in range(world)]
    for r, c in enumerate(comms):
        c.q8_allreduce_(outs[r], a[r], bb[r], scale=1.0 / world)
    torch.cuda.synchronize()
    # the fp8 kernel quantises INSIDE the launch, so one-rank-at-a-time emulation cannot reproduce the W-rank
    # value (tests/test_collectives_gpu.py checks it with really concurrent ranks); here: it ran and is finite
    errs["q8_allreduce_finite"] = float(all(bool(torch.isfinite(o).all()) for o in outs))
    # FT-ZeRO-1: reduce-scatter, commit verdict, gated AdamW + weight all-gather
    L = ShardLayout(((0, nelem),), 2)
    gr, pr = bufs("z1_grad"), bufs("z1_param")
    init = torch.randn(nelem, device=dev, generator=g).bfloat16()
    master = [init.float() for _ in comms]
    m = [torch.zeros(nelem, device=dev) for _ in comms]
    v = [torch.zeros(nelem, device=dev) for _ in comms]
    gates = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in comms]
    hp = (1e-2, 0.9, 0.95, 1e-8, 0.1)
    for r in range(world):
        gr[r].copy_(raw[r])
        pr[r].copy_(init)
    for c in comms:
        c.zero1_reduce_scatter_("z1_grad", 0, nelem, 1.0 / world, True, 2, 8)
    for r, c in enumerate(comms):
        c.zero1_commit_(gates[r], True, True)
    for r, c in enumerate(comms):
        c.zero1_update_("z1_param", 0, gr[r].data_ptr(), master[r].data_ptr(), m[r].data_ptr(), v[r].data_ptr(), nelem,
                        hp, gates[r], 2, 0, 8)
    torch.cuda.synchronize()
    red = want.bfloat16().float()
    mm = (1 - hp[1]) * red
    vv = (1 - hp[2]) * red * red
    ref_w = init.float() * (1 - hp[0] * hp[4]) - hp[0] / (1 - hp[1]) * mm / ((vv / (1 - hp[2])).sqrt() + hp[3])
    errs["zero1_weights"] = float((pr[0].float() - ref_w).abs().max())
    errs["zero1_replicas_differ"] = float(sum(int(not torch.equal(pr[0], pr[r])) for r in range(1, world)))
    errs["zero1_reduced"] = max(float((gr[r][lo:hi].float() - red[lo:hi]).abs().max())
                                for r in range(world) for lo, hi in L.held(r, world))
    # the same update with bf16 moments: from zero moments the weights are the fp32-moment launch's, and the stored
    # moments are the stochastic rounding of single fp32 products, which the numpy specification reproduces bit for bit
    import numpy as np

    from torchft_b200.parallel.zero1 import bf16_sr

    w_fp32 = pr[0].clone()
    master = [init.float() for _ in comms]
    mb = [torch.zeros(nelem, device=dev, dtype=torch.bfloat16) for _ in comms]
    vb = [torch.zeros(nelem, device=dev, dtype=torch.bfloat16) for _ in comms]
    for r, c in enumerate(comms):
        c.zero1_update_("z1_param", 0, gr[r].data_ptr(), master[r].data_ptr(), mb[r].data_ptr(), vb[r].data_ptr(), nelem,
                        hp, gates[r], 2, 0, 8, moment_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    errs["zero1_bf16_moments_weights_differ"] = float(sum(int(not torch.equal(w_fp32, pr[r])) for r in range(world)))
    g32 = red.cpu().numpy()
    c1, c2 = np.float32(1) - np.float32(hp[1]), np.float32(1) - np.float32(hp[2])
    e = np.arange(nelem, dtype=np.uint64)
    want_m, want_v = bf16_sr(c1 * g32, e, 1, 0), bf16_sr((c2 * g32) * g32, e, 1, 1)
    bits = lambda x: x.view(torch.int16).cpu().numpy().view(np.uint16)  # noqa: E731
    errs["zero1_bf16_moment_bits_differ"] = float(sum(
        int((bits(x[r][lo:hi]) != want[lo:hi]).sum()) for r in range(world) for lo, hi in L.held(r, world)
        for x, want in ((mb, want_m), (vb, want_v))))
    # heal copy (NVLink pull kernel; here between two local buffers)
    from torchft_b200.checkpointing.p2p_transport import device_copy

    src, dst = torch.randn(nelem, device=dev, generator=g), torch.empty(nelem, device=dev)
    device_copy([(src.data_ptr(), dst.data_ptr(), nelem * 4)])
    torch.cuda.synchronize()
    errs["heal_copy"] = float((src - dst).abs().max())
    bad = [c.errored() for c in comms if c.errored() is not None]
    assert not bad, bad
    assert errs["allreduce_twoshot"] < 0.05 and errs["allreduce_oneshot"] < 0.05, errs
    assert errs["q8_allreduce_finite"] == 1.0 and errs["heal_copy"] == 0.0, errs
    assert errs["zero1_reduced"] == 0.0 and errs["zero1_replicas_differ"] == 0 and errs["zero1_weights"] < 2e-2, errs
    assert errs["zero1_bf16_moments_weights_differ"] == 0 and errs["zero1_bf16_moment_bits_differ"] == 0, errs
    assert _native.kernel_launches() > 0
    return errs
