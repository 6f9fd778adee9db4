"""Golden-history regression for (Streaming) DiLoCo.

Re-runs the reference's deterministic mocked-update scenario (constant gradient 2, inner lr 1,
outer lr 2, two 1x1 fragments, sync_every 6, with/without sync delay, alpha in {0, .5, 1};
upstream torchft/diloco_regression_test.py) on OUR DiLoCo + Manager + Lighthouse + Gloo and
compares the complete per-step parameter history and the global-parameter history with the JSON
histories upstream torchft checked in (its `test_fixtures/*.json`, stored here as
`tests/golden/diloco/mocked_updates_<index>.json` -- data, not code). Matching them pins
down the fragment schedule, pseudo-gradient sign, restore/merge order and alpha mixing exactly.
"""

import copy
import json
import os
import threading
from concurrent.futures import ThreadPoolExecutor
from datetime import timedelta
from typing import Any, Dict

import pytest
import torch
from torch import nn, optim
from torch.distributed import TCPStore

from torchft_b200.coordination import LighthouseServer
from torchft_b200.local_sgd import DiLoCo
from torchft_b200.manager import Manager
from torchft_b200.process_group import ProcessGroupGloo

FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "diloco")
CASES = [(0, 0.0), (0, 0.5), (0, 1.0), (1, 0.0), (1, 0.5), (1, 1.0)]  # fixture index = position


class MockLinear(nn.Module):
    def __init__(self) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.ones(1, 1))


class MockModel(nn.Module):
    def __init__(self, n: int) -> None:
        super().__init__()
        self.layers = nn.ModuleList(MockLinear() for _ in range(n))


class MockOptimizer(optim.Optimizer):
    def __init__(self, params, lr: float) -> None:
        super().__init__(params, dict(lr=lr))

    def step(self, closure=None):  # type: ignore[override]
        for g in self.param_groups:
            for p in g["params"]:
                if p.grad is not None:
                    p.data.add_(p.grad.data, alpha=-g["lr"])


def _replica(rid: int, lh_addr: str, delay: int, alpha: float, barrier: threading.Barrier) -> Dict[str, Any]:
    store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
    model = MockModel(2)
    inner = MockOptimizer(model.parameters(), lr=1)
    outers = [MockOptimizer(model.layers[i].parameters(), lr=2) for i in range(2)]
    pg = ProcessGroupGloo(timeout=timedelta(seconds=10))
    manager = Manager(pg=pg, min_replica_size=2, use_async_quorum=False,
                      load_state_dict=lambda sd: model.load_state_dict(sd), state_dict=lambda: model.state_dict(),
                      replica_id=str(rid), store_addr="127.0.0.1", store_port=store.port, rank=0, world_size=1,
                      lighthouse_addr=lh_addr, timeout=timedelta(seconds=10), quorum_timeout=timedelta(seconds=10),
                      connect_timeout=timedelta(seconds=10))
    history: Dict[str, Any] = {"history": {}, "global_parameter_history": {}}
    try:
        with DiLoCo(manager, [l for l in model.layers], inner, outers, backup_device=torch.device("cpu"), pin_memory=False,
                    sync_every=6, fragment_sync_delay=delay, fragment_update_alpha=alpha):
            # same preamble as the reference scenario: two committed (empty) steps before training
            manager.start_quorum()
            manager.wait_quorum()
            barrier.wait()
            assert manager.should_commit()
            assert manager.should_commit()
            local_step, seen = 0, set()
            while True:
                history["history"][str(local_step)] = {n: p.data.clone().tolist() for n, p in model.named_parameters()}
                cur = manager.current_step()
                if cur == 7:
                    break
                if cur not in seen:
                    user = copy.deepcopy(manager._manager_state_dict())["user"]
                    history["global_parameter_history"][str(local_step)] = {
                        f"layers.{i}.weight": user[f"StreamingDiLoCoFragment_{i}"]["original_parameters"]["weight"].tolist()
                        for i in range(2)}
                    seen.add(cur)
                for layer in model.layers:
                    layer.weight.grad = torch.ones_like(layer.weight) * 2
                inner.step()
                local_step += 1
        return history
    finally:
        manager.shutdown(wait=False)
        pg.shutdown()


@pytest.mark.parametrize("index", range(len(CASES)))
def test_diloco_matches_reference_history(index):
    delay, alpha = CASES[index]
    with open(os.path.join(FIXTURES, f"mocked_updates_{index}.json")) as f:
        expected = json.load(f)
    lh = LighthouseServer(bind="[::]:0", min_replicas=2)
    barrier = threading.Barrier(2)
    try:
        with ThreadPoolExecutor(max_workers=2) as ex:
            futs = [ex.submit(_replica, r, lh.address(), delay, alpha, barrier) for r in range(2)]
            got = [f.result(timeout=120) for f in futs]
    finally:
        lh.shutdown()
    for r in range(2):
        exp = expected[r][0]
        for section in ("history", "global_parameter_history"):
            assert set(got[r][section]) == set(exp[section]), (section, sorted(got[r][section]), sorted(exp[section]))
            for step, params in exp[section].items():
                for name, val in params.items():
                    torch.testing.assert_close(torch.tensor(got[r][section][step][name]), torch.tensor(val), rtol=1e-5, atol=1e-5,
                                               msg=lambda m: f"replica {r} {section}[{step}][{name}]: {m}")
