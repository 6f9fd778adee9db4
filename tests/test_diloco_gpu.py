"""DiLoCo on the native data plane: the flat fast path (one fused delta all-reduce + one fused outer-step kernel per sync)
must train exactly like the generic per-parameter path (reference semantics, local_sgd.py:339-384,445-475)."""

from __future__ import annotations

import os
from datetime import timedelta

import pytest
import torch
from torch.distributed import TCPStore

pytestmark = pytest.mark.gpu


def _run(flat: bool, alpha: float, quantize: bool, nesterov: bool):
    from torchft_b200.bench_utils import local_lighthouse, loopback
    from torchft_b200.local_sgd import DiLoCo
    from torchft_b200.manager import Manager
    from torchft_b200.models.llama import CONFIGS, FlatParams, Llama
    from torchft_b200.parallel.process_group_b200 import ProcessGroupB200

    os.environ["TORCHFT_B200_DILOCO_FLAT"] = "1" if flat else "0"
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    lh = local_lighthouse()
    store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
    cfg = CONFIGS["llama3_tiny"]
    model = Llama(cfg, device=dev)  # bf16: the fused model kernels are bf16-only
    FlatParams(model)
    model.init_weights(3)
    pg = ProcessGroupB200(timeout=timedelta(seconds=20), device=dev)
    mgr = Manager(pg=pg, load_state_dict=lambda sd: None, state_dict=lambda: {}, min_replica_size=1, use_async_quorum=False,
                  timeout=timedelta(seconds=20), rank=0, world_size=1, store_addr="127.0.0.1", store_port=store.port,
                  lighthouse_addr=loopback(lh.address()), replica_id=f"diloco_{int(flat)}")
    inner = torch.optim.SGD(model.parameters(), lr=0.05)
    outer = torch.optim.SGD(model.parameters(), lr=0.7, momentum=0.9, nesterov=nesterov)
    try:
        gen = torch.Generator().manual_seed(1)
        with DiLoCo(mgr, [model], inner, outer, sync_every=2, backup_device=dev, should_quantize=quantize,
                    fragment_update_alpha=alpha) as d:
            assert (d._fragments[0]._flat_grad is not None) == flat
            for _ in range(8):
                tok = torch.randint(0, cfg.vocab_size, (2, 32), generator=gen).to(dev)
                tgt = torch.randint(0, cfg.vocab_size, (2, 32), generator=gen).to(dev)
                inner.zero_grad()
                model(tok, tgt).backward()
                inner.step()
            assert mgr.current_step() == 4
            frag = d._fragments[0]
            params = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).clone()
            orig = torch.cat([frag.original_parameters[n].reshape(-1) for n in frag._names]).clone()
        return params, orig
    finally:
        mgr.shutdown(wait=False)
        pg.shutdown()
        lh.shutdown()
        os.environ.pop("TORCHFT_B200_DILOCO_FLAT", None)


@pytest.mark.parametrize("alpha,quantize,nesterov", [(0.0, False, True), (0.3, True, True), (0.0, True, False)])
def test_flat_diloco_matches_generic_path(alpha, quantize, nesterov):
    pg_, og_ = _run(False, alpha, quantize, nesterov)
    pf_, of_ = _run(True, alpha, quantize, nesterov)
    # bf16 weights; the generic path keeps its momentum in bf16 (torch SGD), the fused kernel in fp32
    for got, want in ((pf_, pg_), (of_, og_)):
        diff = (got.float() - want.float()).abs()
        assert float(diff.max()) <= 2e-2 and float(diff.mean()) <= 2e-3, (float(diff.max()), float(diff.mean()))
